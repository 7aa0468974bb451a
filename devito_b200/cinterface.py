"""`Operator.cinterface()` for operators that run on the CUDA path.

The reference writes `<name>.c` / `<name>.h` for every Operator: the generated kernel and a header
with its flat C signature plus the public `struct dataobj` / `struct profiler`
(devito/operator/operator.py:871-902; tests/test_cinterface.py:9-41). Here the kernel is pre-built
(libb200stencil.so), so `<name>.c` is the thin adapter a C/C++ host links instead of the reference's
generated file: the SAME symbol with the SAME kind of signature —

    int Forward(struct dataobj *restrict damp_vec, ..., struct dataobj *restrict u_vec,
                const float vp, const int x_M, const int x_m, ..., const float dt,
                const int p_rec_M, ..., const int time_M, const int time_m,
                const int deviceid, const int devicerm, struct profiler *timers)

— which packs its arguments into `struct b2_iso_args` / `struct b2_tti_args` (include/b200stencil.h)
(or `struct b2_sa_args`) and calls `b2_iso_forward` / `b2_tti_forward` (or `b2_sa_forward`). Functions and Constants come first in alphabetical
order, then bounds, `dt`, sparse point ranges and time bounds, like the parameter order of the
reference's printed samples (`damp_vec, dt, m_vec, ..., u_vec, x_M, x_m, ..., timers`;
devito/ir/iet/utils.py:105-147). The finite-difference weights are literals in the file, as they are
in the reference's generated code.
"""
import os
import tempfile

import numpy as np

__all__ = ['generate', 'jit_dir']

_DATAOBJ = """struct dataobj
{
  void *restrict data;
  int *size;
  unsigned long nbytes;
  unsigned long *npsize;
  unsigned long *dsize;
  int *hsize;
  int *hofs;
  int *oofs;
  void *dmap;
} ;
"""

_PROFILER = """struct profiler
{
  double section0;
  double section1;
  double section2;
} ;
"""


def jit_dir():
    """Where the generated files go (the reference uses its JIT cache directory,
    devito/arch/compiler.py `get_jit_dir`)."""
    d = os.environ.get('DEVITO_B200_JITDIR') or os.path.join(
        tempfile.gettempdir(), f'devito-b200-jitcache-uid{os.getuid()}')
    os.makedirs(d, exist_ok=True)
    return d


def _flit(x):
    return '%.9ef' % float(np.float32(x))


def _warray(name, w):
    vals = ', '.join(_flit(v) for v in w)
    return f"  static const float {name}[{len(w)}] = {{{vals}}};"


class _Param:
    """One formal parameter of the generated function."""

    def __init__(self, key, ctype, name):
        self.key, self.ctype, self.name = key, ctype, name

    @property
    def decl(self):
        sep = '' if self.ctype.endswith('*') else ' '
        return f"{self.ctype}{sep}{self.name}"


def _sparse_params(sf, ndim):
    names = [f'{sf.name}_vec', f'{sf.name}_gp_vec'] + [f'{sf.name}_w{"xyz"[d]}_vec' for d in range(ndim)]
    keys = [sf.name, sf.name + '_gp'] + [f'{sf.name}_w{"xyz"[d]}' for d in range(ndim)]
    return [_Param(k, 'struct dataobj *restrict', n) for k, n in zip(keys, names)]


def _sparse_block(sf, ndim, var):
    ws = [f'(struct b2_dataobj *){sf.name}_w{"xyz"[d]}_vec' for d in range(ndim)] + ['0'] * (3 - ndim)
    return (f"  struct b2_sparse {var} = {{(struct b2_dataobj *){sf.name}_vec, "
            f"(struct b2_dataobj *){sf.name}_gp_vec, {{{', '.join(ws)}}}, "
            f"p_{sf.name}_m, p_{sf.name}_M, {sf.r}}};")


def signature(plan, name, distributed=False):
    """Formal parameters of the adapter, in the reference's order."""
    grid = plan['grid']
    nd = grid.dim
    head = []          # Functions and Constants, sorted by name
    u = plan['u']
    head.append(_Param(u.name, 'struct dataobj *restrict', f'{u.name}_vec'))
    if plan['kind'] == 'tti':
        v = plan['v']
        head.append(_Param(v.name, 'struct dataobj *restrict', f'{v.name}_vec'))
    if plan.get('damp') is not None:
        d = plan['damp']
        head.append(_Param(d.name, 'struct dataobj *restrict', f'{d.name}_vec'))
    if plan['kind'] == 'iso':
        kind, obj = plan['m_role']
        if kind.endswith('_f'):
            head.append(_Param(obj.name, 'struct dataobj *restrict', f'{obj.name}_vec'))
        elif kind.endswith('_c'):
            head.append(_Param(obj.name, 'const float', obj.name))
        for key in ('grad', 'usave', 'born_U', 'born_dm', 'snap'):
            f = plan.get(key)
            if f is not None:
                head.append(_Param(f.name, 'struct dataobj *restrict', f'{f.name}_vec'))
    elif plan['kind'] == 'sa':
        for kind, obj in (plan['b_role'], plan['vp_role']):
            if kind == 'f':
                head.append(_Param(obj.name, 'struct dataobj *restrict', f'{obj.name}_vec'))
            elif kind == 'c':
                head.append(_Param(obj.name, 'const float', obj.name))
    else:
        for n, c in plan['consts'].items():
            if getattr(c, 'is_Function', False) or hasattr(c, 'space_order'):
                head.append(_Param(n, 'struct dataobj *restrict', f'{n}_vec'))
            else:
                head.append(_Param(n, 'const float', n))
        for key in ('born_du', 'born_dv', 'born_dm', 'grad', 'usave', 'vsave'):
            f = plan.get(key)
            if f is not None:
                head.append(_Param(f.name, 'struct dataobj *restrict', f'{f.name}_vec'))
    for sf in (plan['src'], plan['rec']):
        if sf is not None:
            head.extend(_sparse_params(sf, nd))
    head.sort(key=lambda p: p.key)
    tail = []
    for d in grid.dimensions:
        tail.append(_Param(d.max_name, 'const int', d.max_name))
        tail.append(_Param(d.min_name, 'const int', d.min_name))
    tail.append(_Param('dt', 'const float', 'dt'))
    for sf in sorted((s for s in (plan['src'], plan['rec']) if s is not None), key=lambda s: s.name):
        tail.append(_Param(f'p_{sf.name}_M', 'const int', f'p_{sf.name}_M'))
        tail.append(_Param(f'p_{sf.name}_m', 'const int', f'p_{sf.name}_m'))
    tail.append(_Param('time_M', 'const int', 'time_M'))
    tail.append(_Param('time_m', 'const int', 'time_m'))
    tail.append(_Param('deviceid', 'const int', 'deviceid'))
    tail.append(_Param('devicerm', 'const int', 'devicerm'))
    if distributed:
        tail.append(_Param('halo', 'struct b2_halo_ctx *', 'halo'))
    tail.append(_Param('timers', 'struct profiler *', 'timers'))
    return head + tail


def _prototype(name, params):
    return f"int {name}({', '.join(p.decl for p in params)})"


def _bounds(plan, lines):
    names = [d.name for d in plan['grid'].dimensions]
    slots = ['x', 'y', 'z']
    for slot, n in zip(slots, names):
        lines.append(f"  a.{slot}_m = {n}_m;")
        lines.append(f"  a.{slot}_M = {n}_M;")
    lines.append("  a.time_m = time_m;")
    lines.append("  a.time_M = time_M;")


def _tail(plan, entry, lines, distributed):
    if plan['src'] is not None:
        lines.append("  a.src = &src_s;")
    if plan['rec'] is not None:
        lines.append("  a.rec = &rec_s;")
    lines.append(f"  a.rec_toff = {int(plan['rec_toff'])};")
    lines.append("  a.deviceid = deviceid;")
    if distributed:
        lines.append("  a.halo = halo;")
    lines.append("  a.timers = &prof;")
    lines.append("  /* devicerm: arrays whose `dmap` is NULL are staged to the device and released inside the")
    lines.append("     call (== devicerm=1); arrays with `dmap` set stay resident whatever its value */")
    lines.append("  (void)devicerm;")
    lines.append(f"  const int rc = {entry}(&a);")
    lines.append("  if (timers)")
    lines.append("  {")
    lines.append("    timers->section0 += prof.section0;")
    lines.append("    timers->section1 += prof.section1;")
    lines.append("    timers->section2 += prof.section2;")
    lines.append("  }")
    lines.append("  return rc;")


def _iso_body(plan, distributed):
    nd = plan['grid'].dim
    R = plan['R']
    L = []
    for d in range(nd):
        L.append(_warray(f'w_{"xyz"[d]}', plan['w'][d][:R + 1]))
    if plan['src'] is not None:
        L.append(_sparse_block(plan['src'], nd, 'src_s'))
    if plan['rec'] is not None:
        L.append(_sparse_block(plan['rec'], nd, 'rec_s'))
    L.append("  struct b2_profiler prof = {0.0, 0.0, 0.0, 0.0};")
    L.append("  struct b2_iso_args a;")
    L.append("  memset(&a, 0, sizeof(a));")
    L.append(f"  a.ndim = {nd};")
    L.append(f"  a.space_order = {plan['so']};")
    L.append(f"  a.radius = {R};")
    for d in range(nd):
        L.append(f"  a.w[{d}] = w_{'xyz'[d]};")
    L.append(f"  a.u = (struct b2_dataobj *){plan['u'].name}_vec;")
    if plan.get('damp') is not None:
        L.append(f"  a.damp = (struct b2_dataobj *){plan['damp'].name}_vec;")
    kind, obj = plan['m_role']
    if kind == 'one':
        L.append("  a.param_kind = B2_PARAM_SCALAR;")
        L.append("  a.vp = 1.0f;")
    elif kind == 'vp_c':
        L.append("  a.param_kind = B2_PARAM_SCALAR;")
        L.append(f"  a.vp = {obj.name};")
    elif kind == 'm_c':
        L.append("  a.param_kind = B2_PARAM_SCALAR;")
        L.append(f"  a.vp = 1.0f/sqrtf({obj.name});")
    else:
        L.append(f"  a.param_kind = {'B2_PARAM_VP' if kind == 'vp_f' else 'B2_PARAM_M'};")
        L.append(f"  a.param = (struct b2_dataobj *){obj.name}_vec;")
        L.append("  a.vp = 1.0f;")
    L.append("  a.dt = dt;")
    _bounds(plan, L)
    L.append(f"  a.adjoint = {1 if plan.get('adjoint') else 0};")
    if plan.get('snap') is not None:
        L.append(f"  a.snap = (struct b2_dataobj *){plan['snap'].name}_vec;")
        L.append(f"  a.snap_factor = {int(plan['snap_factor'])};")
        L.append(f"  a.snap_toff = {int(plan['snap_toff'])};")
    if plan.get('born_U') is not None:
        L.append(f"  a.born_U = (struct b2_dataobj *){plan['born_U'].name}_vec;")
        L.append(f"  a.born_dm = (struct b2_dataobj *){plan['born_dm'].name}_vec;")
    if plan.get('free_surface'):
        L.append("  a.free_surface = 1;")
    if plan.get('ot4'):
        L.append("  a.ot4 = 1;")
    if plan.get('grad') is not None:
        L.append(f"  a.grad = (struct b2_dataobj *){plan['grad'].name}_vec;")
        L.append(f"  a.usave = (struct b2_dataobj *){plan['usave'].name}_vec;")
    _tail(plan, 'b2_iso_forward', L, distributed)
    return L


def _tti_body(plan, distributed):
    R = plan['R']
    L = []
    for d in range(3):
        L.append(_warray(f'w2_{"xyz"[d]}', plan['w2'][d][:R + 1]))
    for d in range(3):
        L.append(_warray(f'w1_{"xyz"[d]}', plan['w1'][d][:R]))
    if plan['src'] is not None:
        L.append(_sparse_block(plan['src'], 3, 'src_s'))
    if plan['rec'] is not None:
        L.append(_sparse_block(plan['rec'], 3, 'rec_s'))
    L.append("  struct b2_profiler prof = {0.0, 0.0, 0.0, 0.0};")
    L.append("  struct b2_tti_args a;")
    L.append("  memset(&a, 0, sizeof(a));")
    L.append(f"  a.space_order = {plan['so']};")
    L.append(f"  a.radius = {R};")
    for d in range(3):
        L.append(f"  a.w2[{d}] = w2_{'xyz'[d]};")
        L.append(f"  a.w1[{d}] = w1_{'xyz'[d]};")
    L.append(f"  a.u = (struct b2_dataobj *){plan['u'].name}_vec;")
    L.append(f"  a.v = (struct b2_dataobj *){plan['v'].name}_vec;")
    if plan.get('damp') is not None:
        L.append(f"  a.damp = (struct b2_dataobj *){plan['damp'].name}_vec;")
    for n in ('vp', 'epsilon', 'delta', 'theta', 'phi'):
        c = plan['consts'].get(n)
        if c is None:
            L.append(f"  a.{n} = 0.0f;")
        elif hasattr(c, 'space_order'):
            L.append(f"  a.{n}_arr = (struct b2_dataobj *){n}_vec;")
            L.append(f"  a.{n} = {'1.0f' if n == 'vp' else '0.0f'};")
        else:
            L.append(f"  a.{n} = {n};")
    L.append("  a.dt = dt;")
    _bounds(plan, L)
    if plan.get('born_du') is not None:
        L.append(f"  a.born_du = (struct b2_dataobj *){plan['born_du'].name}_vec;")
        L.append(f"  a.born_dv = (struct b2_dataobj *){plan['born_dv'].name}_vec;")
        L.append(f"  a.born_dm = (struct b2_dataobj *){plan['born_dm'].name}_vec;")
    if plan.get('adjoint'):
        L.append("  a.adjoint = 1;")
    if plan.get('grad') is not None:
        L.append(f"  a.grad = (struct b2_dataobj *){plan['grad'].name}_vec;")
        L.append(f"  a.usave = (struct b2_dataobj *){plan['usave'].name}_vec;")
        L.append(f"  a.vsave = (struct b2_dataobj *){plan['vsave'].name}_vec;")
    _tail(plan, 'b2_tti_forward', L, distributed)
    return L


def _sa_body(plan, distributed):
    nd = plan['grid'].dim
    L = []
    for d in range(nd):
        L.append(_warray(f'c_{"xyz"[d]}', plan['c'][d]))
    if plan['src'] is not None:
        L.append(_sparse_block(plan['src'], nd, 'src_s'))
    if plan['rec'] is not None:
        L.append(_sparse_block(plan['rec'], nd, 'rec_s'))
    L.append("  struct b2_profiler prof = {0.0, 0.0, 0.0, 0.0};")
    L.append("  struct b2_sa_args a;")
    L.append("  memset(&a, 0, sizeof(a));")
    L.append(f"  a.ndim = {nd};")
    L.append(f"  a.space_order = {plan['so']};")
    L.append(f"  a.radius = {plan['R']};")
    for d in range(nd):
        L.append(f"  a.c[{d}] = c_{'xyz'[d]};")
    L.append(f"  a.u = (struct b2_dataobj *){plan['u'].name}_vec;")
    for key, (kind, obj) in (('b', plan['b_role']), ('vp', plan['vp_role'])):
        if kind == 'f':
            L.append(f"  a.{key} = (struct b2_dataobj *){obj.name}_vec;")
            L.append(f"  a.{key}_value = 1.0f;")
        elif kind == 'c':
            L.append(f"  a.{key}_value = {obj.name};")
        else:
            L.append(f"  a.{key}_value = {_flit(obj)};")
    if plan.get('damp') is not None:
        L.append(f"  a.damp = (struct b2_dataobj *){plan['damp'].name}_vec;")
    L.append("  a.dt = dt;")
    _bounds(plan, L)
    L.append(f"  a.adjoint = {1 if plan.get('adjoint') else 0};")
    _tail(plan, 'b2_sa_forward', L, distributed)
    return L


def generate(plan, name, distributed=False):
    """(ccode, hcode) strings for a recognised operator."""
    params = signature(plan, name, distributed)
    proto = _prototype(name, params)
    guard = ''.join(ch if ch.isalnum() else '_' for ch in name).upper() + '_H'
    h = [f"#ifndef {guard}", f"#define {guard}", "",
         "/* Interface of the operator `%s`, executed by libb200stencil.so (sm_90a). The two structs"
         % name,
         "   are the reference's public ones (devito/types/dense.py:737-746, devito/types/misc.py:41-68). */",
         "",
         "#ifdef __cplusplus", 'extern "C" {', "#define restrict __restrict__", "#endif", "",
         _DATAOBJ, _PROFILER]
    if distributed:
        h.append("struct b2_halo_ctx;\n")
    h += [proto + ";", "", "#ifdef __cplusplus", "#undef restrict", "}", "#endif", "", f"#endif /* {guard} */", ""]
    body = {'iso': _iso_body, 'tti': _tti_body, 'sa': _sa_body}[plan['kind']](plan, distributed)
    c = ['#include <math.h>', '#include <string.h>', f'#include "{name}.h"', '#include "b200stencil.h"', "",
         "/* `struct dataobj` and `struct b2_dataobj` have the same members in the same order */",
         "typedef char dataobj_layout_check[(sizeof(struct dataobj) == sizeof(struct b2_dataobj)) ? 1 : -1];",
         "", proto, "{"] + body + ["}", ""]
    return '\n'.join(c), '\n'.join(h)
