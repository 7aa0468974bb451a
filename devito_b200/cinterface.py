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

from .operator import wave_entry

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


def _is_array(obj):
    return hasattr(obj, 'space_order')


def signature(plan, name, distributed=False):
    """Formal parameters of the adapter, in the reference's order."""
    entry = wave_entry(plan)
    nd = plan['grid'].dim
    head = []          # Functions and Constants, sorted by name
    for obj in [s.obj for s in entry.arrays] + [prm.obj for prm in entry.params]:
        if _is_array(obj):
            head.append(_Param(obj.name, 'struct dataobj *restrict', f'{obj.name}_vec'))
        elif obj is not None:
            head.append(_Param(obj.name, 'const float', obj.name))
    for sf in (plan['src'], plan['rec']):
        if sf is not None:
            head.extend(_sparse_params(sf, nd))
    head.sort(key=lambda p: p.key)
    tail = []
    for d in plan['grid'].dimensions:
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


def _body(plan, distributed):
    """Fill `struct b2_<kind>_args` from the flat parameters and call the entry point."""
    entry = wave_entry(plan)
    nd = plan['grid'].dim
    L = []
    for member, w in entry.weights:
        for d in range(nd):
            L.append(_warray(f'{member}_{"xyz"[d]}', w[d]))
    if plan['src'] is not None:
        L.append(_sparse_block(plan['src'], nd, 'src_s'))
    if plan['rec'] is not None:
        L.append(_sparse_block(plan['rec'], nd, 'rec_s'))
    L.append("  struct b2_profiler prof = {0.0, 0.0, 0.0, 0.0};")
    L.append(f"  struct b2_{plan['kind']}_args a;")
    L.append("  memset(&a, 0, sizeof(a));")
    for k, v in entry.flags.items():
        L.append(f"  a.{k} = {_flit(v) if isinstance(v, float) else int(v)};")
    for member, _ in entry.weights:
        for d in range(nd):
            L.append(f"  a.{member}[{d}] = {member}_{'xyz'[d]};")
    for s in entry.arrays:
        L.append(f"  a.{s.member} = (struct b2_dataobj *){s.obj.name}_vec;")
    for prm in entry.params:
        obj = prm.obj
        if _is_array(obj):
            L.append(f"  a.{prm.member} = (struct b2_dataobj *){obj.name}_vec;")
            L.append(f"  a.{prm.scalar} = {prm.unit:.1f}f;")
        elif obj is not None:
            L.append(f"  a.{prm.scalar} = {f'1.0f/sqrtf({obj.name})' if prm.slowness else obj.name};")
        else:
            L.append(f"  a.{prm.scalar} = {prm.unit:.1f}f;")
        if prm.member == 'param':
            kind = 'B2_PARAM_SCALAR' if not _is_array(obj) else 'B2_PARAM_M' if prm.slowness else 'B2_PARAM_VP'
            L.append(f"  a.param_kind = {kind};")
    L.append("  a.dt = dt;")
    for slot, d in zip('xyz', plan['grid'].dimensions):
        L.append(f"  a.{slot}_m = {d.name}_m;")
        L.append(f"  a.{slot}_M = {d.name}_M;")
    L.append("  a.time_m = time_m;")
    L.append("  a.time_M = time_M;")
    if plan['src'] is not None:
        L.append("  a.src = &src_s;")
    if plan['rec'] is not None:
        L.append("  a.rec = &rec_s;")
    L.append("  a.deviceid = deviceid;")
    if distributed:
        L.append("  a.halo = halo;")
    L.append("  a.timers = &prof;")
    L.append("  /* devicerm: arrays whose `dmap` is NULL are staged to the device and released inside the")
    L.append("     call (== devicerm=1); arrays with `dmap` set stay resident whatever its value */")
    L.append("  (void)devicerm;")
    L.append(f"  const int rc = {entry.symbol}(&a);")
    L.append("  if (timers)")
    L.append("  {")
    L.append("    timers->section0 += prof.section0;")
    L.append("    timers->section1 += prof.section1;")
    L.append("    timers->section2 += prof.section2;")
    L.append("  }")
    L.append("  return rc;")
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
    body = _body(plan, distributed)
    c = ['#include <math.h>', '#include <string.h>', f'#include "{name}.h"', '#include "b200stencil.h"', "",
         "/* `struct dataobj` and `struct b2_dataobj` have the same members in the same order */",
         "typedef char dataobj_layout_check[(sizeof(struct dataobj) == sizeof(struct b2_dataobj)) ? 1 : -1];",
         "", proto, "{"] + body + ["}", ""]
    return '\n'.join(c), '\n'.join(h)
