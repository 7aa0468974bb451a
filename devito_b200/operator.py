"""`Operator`: same construction/apply contract as the reference, different engine.

Reference contract kept (devito/operator/operator.py): `Operator(exprs, subs=, name=, opt=,
platform=, language=, compiler=)` (:168), `op.apply(**overrides)` / `op(**overrides)` (:906,
:956), `op.arguments(**kw)` (:796), `op.cfunction` (:857), the returned
`PerformanceSummary` (operator/profiling.py:432), non-zero return code -> `ExecutionError`
(:734-772), unknown kwargs -> `InvalidArgument` (:588-592).

What is replaced: the reference lowers the expressions through its compiler
(`_lower`, :283-315) and JIT-compiles C.  Here `Operator.__init__` runs a *semantic pattern
recogniser*: the time-update equations are decomposed into their linear stencil
(`symbolics.linear_terms`), and that stencil is compared — numerically, at random parameter
values — with the stencil the hand-written CUDA kernels implement (isotropic acoustic:
examples/seismic/acoustic/operators.py:71-150; TTI centred: examples/seismic/tti/
operators.py:186-247, 431-480).  On a match the operator becomes a thin marshalling layer
over the C ABI in include/b200stencil.h (one FFI crossing per `apply`, like the reference's
`cfunction(*arg_values)`, :1032).  Everything else (set-up operators) goes to the NumPy
interpreter.  The recognised path NEVER falls back to the CPU.
"""
import ctypes
import itertools
import os
import time as _time
from collections import OrderedDict
from typing import NamedTuple

import numpy as np

from .symbolics import (Number, Add, Mul, Pow, Call, as_expr, linear_terms, NonLinear, fd_weights,
                        fd_offsets, _py_funcs)
from .types import Function, TimeFunction, Constant
from .sparse import Injection, Interpolation, SparseTimeFunction
from .equation import Eq, FreeSurface
from .interpreter import Interpreter, _subsampled
from .parameters import configuration
from .exceptions import InvalidArgument, ExecutionError, InvalidOperator
from .logger import perf, warning
from .tools import flatten
from . import _lib as L_
from . import distributed

__all__ = ['Operator', 'PerformanceSummary']

B2_PARAM_SCALAR, B2_PARAM_VP, B2_PARAM_M = 0, 1, 2


# ---------------------------------------------------------------------------------------------
# performance summary (devito/operator/profiling.py:432-527)
# ---------------------------------------------------------------------------------------------
class PerfEntry:
    def __init__(self, time, gflopss=None, gpointss=None, oi=None, ops=None, itershapes=None):
        self.time = time
        self.gflopss = gflopss
        self.gpointss = gpointss
        self.oi = oi
        self.ops = ops
        self.itershapes = itershapes

    def __repr__(self):
        return f"PerfEntry(time={self.time}, gpointss={self.gpointss})"


class PerformanceSummary(OrderedDict):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.globals = {}

    @property
    def timings(self):
        return OrderedDict((k, v.time) for k, v in self.items())

    @property
    def gflopss(self):
        return OrderedDict((k, v.gflopss) for k, v in self.items())

    @property
    def gpointss(self):
        return OrderedDict((k, v.gpointss) for k, v in self.items())

    @property
    def oi(self):
        return OrderedDict((k, v.oi) for k, v in self.items())

    @property
    def time(self):
        return sum(v.time for v in self.values())


# ---------------------------------------------------------------------------------------------
# scalar evaluation of coefficient expressions (for the recogniser)
# ---------------------------------------------------------------------------------------------
def eval_scalar(expr, leaf):
    if isinstance(expr, Number):
        return float(expr.value)
    if expr.is_Access or expr.is_Symbol:
        return leaf(expr)
    if isinstance(expr, Add):
        return sum(eval_scalar(a, leaf) for a in expr.args)
    if isinstance(expr, Mul):
        out = 1.0
        for a in expr.args:
            out *= eval_scalar(a, leaf)
        return out
    if isinstance(expr, Pow):
        return eval_scalar(expr.base, leaf) ** eval_scalar(expr.exponent, leaf)
    if isinstance(expr, Call):
        return float(_py_funcs[expr.name](eval_scalar(expr.arg, leaf)))
    if expr.is_Derivative:
        return eval_scalar(expr.evaluate, leaf)
    raise TypeError(type(expr).__name__)


def _space_offsets(acc, space_dims):
    """Integer (time_shift, (dx, dy, dz)) of an access, or None if not a plain shifted access."""
    f = acc.function
    tshift = 0
    offs = []
    for idx, d in zip(acc.index_objs, f.dimensions):
        if idx.absolute is not None or idx.shift.denominator != 1:
            return None
        if d.is_Time:
            tshift = int(idx.shift)
        else:
            if idx.base is not d and idx.base != d:
                return None
            offs.append(int(idx.shift))
    return tshift, tuple(offs)


def second_derivative_weights(space_order, h):
    """w[k]/h^2, k = 0..so/2 (symmetric). Reference: `u.laplace` -> per-dim
    finite_diff_weights(2, range(-so/2, so/2+1), 0), each evalf(9) (finite_difference.py:185-187)."""
    R = space_order // 2
    w = fd_weights(2, list(range(-R, R + 1)), 0)
    return [w[R + k] / (float(h) ** 2) for k in range(R + 1)]


def sa_weights(R, h):
    """c_k / h, k = 1..R: the weights of `f.dx(x0=x+h/2)` at fd_order 2R (offsets -R+1 .. R about x + h/2) at
    offset +k; the weight at offset -k+1 is -c_k (examples/seismic/self_adjoint/operators.py:50-62)."""
    from fractions import Fraction
    w = fd_weights(1, list(range(-R + 1, R + 1)), Fraction(1, 2))
    return [w[R - 1 + k] / float(h) for k in range(1, R + 1)]


def half_node_first_derivative_weights(space_order, h):
    """Weights of `f.dx(fd_order=so/2, x0=x+h/2)` for offsets (-R/2+1 .. R/2), R = so/2
    (devito/finite_differences/tools.py:289-297; tti/operators.py:88-102)."""
    R = space_order // 2
    offs = fd_offsets(R, 0.5) if False else list(range(-R // 2 + 1, R // 2 + 1))
    from fractions import Fraction
    w = fd_weights(1, offs, Fraction(1, 2))
    return [c / float(h) for c in w]


class _Unrecognised(Exception):
    pass


class _NotVisco(_Unrecognised):
    """Two updates that do not have the shape of the SLS pair (the second reads the first only at the level the
    first writes): left to the TTI and Born recognisers."""


# ---------------------------------------------------------------------------------------------
# the argument block of a wave operator's C entry point
# ---------------------------------------------------------------------------------------------
class Slot(NamedTuple):
    """An array member of the block: the plan's object, whether the call writes it, whether it is re-laid
    out to the wavefield's halo, and what an override must be (a key of `_OVERRIDE_KINDS`)."""
    member: str
    obj: object
    written: bool
    layout: bool
    check: str


class Param(NamedTuple):
    """A parameter passed as the array `member` or as the scalar `scalar`. `obj` is the plan's Function or
    Constant (None: always `unit`); the scalar is `unit` while the array is used. `slowness`: `obj` is
    m = 1/vp^2, passed as the scalar 1/sqrt(m) or as a B2_PARAM_M array. `switch`: an override may turn an
    array into a scalar and back."""
    member: str
    scalar: str
    obj: object
    unit: float
    slowness: bool
    switch: bool


class Entry(NamedTuple):
    """Everything `Operator.apply`, `Operator.parameters`, the C adapter (cinterface.py) and the reference
    plugin (refplugin.py) need to know about the call of a recognised wave operator."""
    symbol: str             # b2_<kind>_forward, taking a struct b2_<kind>_args
    struct: type            # its ctypes mirror
    flags: dict             # members fixed by the plan (integers; f0 of the viscoacoustic update)
    weights: list           # (member, per-dimension weight lists)
    arrays: list            # Slots, in the order they are marshalled
    params: list            # Params
    host_io: tuple          # members that may come with the caller's device buffer (struct b2_iso_args.host_io)


_OVERRIDE_KINDS = {'wavefield': "a float32 TimeFunction of the wavefield's space order on the same grid",
                   'saved': "a float32 saved TimeFunction (save=nt) of the wavefield's space order",
                   'snapshot': "a float32 saved TimeFunction on the same grid",
                   'function': "a float32 Function or an array of its allocated shape"}


def wave_entry(p):
    """The `Entry` of a recognised wave plan (kind 'iso', 'tti' or 'sa')."""
    kind = p['kind']
    slots = [('u', True, False, 'wavefield'), ('v', True, False, 'wavefield'), ('r', True, False, 'wavefield'),
             ('damp', False, True, 'function'),
             ('snap', True, False, 'snapshot'), ('born_U', True, False, 'wavefield'),
             ('born_du', True, False, 'wavefield'), ('born_dv', True, False, 'wavefield'),
             ('born_dm', False, False, 'function'), ('grad', True, False, 'function'),
             ('usave', False, False, 'saved'), ('vsave', False, False, 'saved')]
    arrays = [Slot(m, p[m], w, lay, chk) for m, w, lay, chk in slots if p.get(m) is not None]
    if kind == 'iso':
        role, obj = p['m_role']
        params = [Param('param', 'vp', obj, 1.0, role.startswith('m_'), True)]
    elif kind == 'sa':
        params = [Param(k, k + '_value', p[k + '_role'][1], 1.0, False, True) for k in ('b', 'vp')]
    elif kind == 'visco':
        params = [Param(k, k + '_value', p[k + '_role'][1], 1.0, False, True) for k in ('b', 'vp', 'qp')]
    else:
        params = [Param(n + '_arr', n, p['consts'].get(n), 1.0 if n == 'vp' else 0.0, False, False)
                  for n in ('vp', 'epsilon', 'delta', 'theta', 'phi')]
    flags = {'space_order': p['so'], 'radius': p['R'], 'adjoint': int(bool(p.get('adjoint'))),
             'rec_toff': p['rec_toff'], 'ndim': p['grid'].dim}
    if kind == 'iso':
        flags.update(free_surface=int(bool(p.get('free_surface'))), ot4=int(bool(p.get('ot4'))))
        if p.get('snap') is not None:
            flags.update(snap_factor=p['snap_factor'], snap_toff=p['snap_toff'])
    if kind == 'visco':
        flags.update(f0=float(p['f0']))
    weights = [(k, p[k]) for k in ('w', 'w2', 'w1', 'c') if k in p]
    struct = {'iso': L_.IsoArgs, 'tti': L_.TtiArgs, 'sa': L_.SaArgs, 'visco': L_.ViscoArgs}[kind]
    return Entry(f'b2_{kind}_forward', struct, flags, weights, arrays, params,
                 ('u', 'damp', 'param') if kind == 'iso' else ())


# ---------------------------------------------------------------------------------------------
# the operator
# ---------------------------------------------------------------------------------------------
class Operator:
    _known_opts = ('opt', 'platform', 'language', 'compiler', 'mpi', 'allocator', 'profiling',
                   'autotune', 'deviceid')

    def __init__(self, expressions, subs=None, name='Kernel', **kwargs):
        self.name = name
        self._options = {k: kwargs.get(k) for k in self._known_opts if k in kwargs}
        items = flatten([expressions] if not isinstance(expressions, (list, tuple)) else list(expressions))
        self._items = []
        for it in items:
            if isinstance(it, Eq):
                self._items.append(('eq', it))
            elif isinstance(it, FreeSurface):
                self._items.append(('fs', it))
            elif isinstance(it, Injection):
                self._items.append(('inject', it))
            elif isinstance(it, Interpolation):
                self._items.append(('interp', it))
            else:
                raise InvalidOperator(f"unsupported expression type {type(it).__name__}")
        self._subs = {as_expr(k): v for k, v in (subs or {}).items()}
        self._plan = None
        self._why_not = None
        self._dirn = 1
        try:
            self._plan = self._recognise()
        except _Unrecognised as e:
            self._why_not = str(e)
        if self._plan is None and any(k == 'fs' for k, _ in self._items):
            raise InvalidOperator(f"free-surface operator not recognised by the CUDA path ({self._why_not}); "
                                  "there is no interpreter (CPU) implementation of it")
        if self._plan is None and self._looks_like_wave_propagation():
            # never silent: the CUDA kernels are the product, the interpreter is host plumbing for
            # set-up operators and the reference's CPU-runnable 2-D diffusion case
            warning(f"Operator `{name}` updates a second-order-in-time field but is not one of the schemes "
                    f"the CUDA path implements ({self._why_not}); it will run on the NumPy interpreter")
        self._interp = None if self._plan is not None else Interpreter(self._items, None, self._subs, name=name)
        self._entry = wave_entry(self._plan) if self._plan is not None and self._plan['kind'] != 'linear' else None
        self._profiler_last = None

    def _looks_like_wave_propagation(self):
        for k, o in self._items:
            if k == 'eq' and o.lhs.is_Access and getattr(o.lhs.function, 'is_TimeFunction', False) \
                    and o.lhs.function.time_order == 2:
                return True
        return False

    # ------------------------------------------------------------------------------------------
    # recognition
    # ------------------------------------------------------------------------------------------
    @property
    def backend(self):
        return 'cuda-sm90a' if self._plan is not None else 'numpy-interpreter'

    def _recognise(self):
        try:
            plan = self._recognise_wave()
        except _Unrecognised as wave_why:
            try:
                plan = self._recognise_linear()
            except _Unrecognised as lin_why:
                raise _Unrecognised(f"{wave_why}; as a generic constant-coefficient update: {lin_why}") from None
        self._check_dtypes(plan)
        return plan

    # the plan members that are arrays the library reads or writes
    _ARRAY_MEMBERS = ('u', 'v', 'r', 'damp', 'snap', 'born_U', 'born_du', 'born_dv', 'born_dm', 'grad', 'usave', 'vsave')

    @classmethod
    def _check_dtypes(cls, plan):
        """The kernels read and write float32 only: a plan whose grid, fields, parameter Functions, saved
        fields or sparse traces and coordinates are of another dtype is not theirs to run."""
        objs = [plan[k] for k in cls._ARRAY_MEMBERS if plan.get(k) is not None]
        for k in ('m_role', 'b_role', 'vp_role', 'qp_role'):
            if plan.get(k) is not None:
                objs.append(plan[k][1])
        objs += list(plan.get('consts', {}).values())
        objs = [o for o in objs if isinstance(o, Function)]
        if np.dtype(plan['grid'].dtype) != np.float32:
            raise _Unrecognised(f"the grid is {np.dtype(plan['grid'].dtype).name}; the kernels compute in float32")
        for o in objs:
            if np.dtype(o.dtype) != np.float32:
                raise _Unrecognised(f"`{o.name}` is {np.dtype(o.dtype).name}; the kernels read float32 arrays")
        for sf in (plan.get('src'), plan.get('rec')):
            if sf is None:
                continue
            for what, dt in (('traces', sf.dtype), ('coordinates', sf.coordinates_data.dtype)):
                if np.dtype(dt) != np.float32:
                    raise _Unrecognised(f"the {what} of `{sf.name}` are {np.dtype(dt).name}; the kernels read "
                                        "float32 sparse data")

    def _recognise_linear(self):
        """A single explicit update `f.forward|backward = sum_k c_k f[t + s_k][p + o_k]` whose
        coefficients contain no field (Constants, spacings, dt and numbers only) — e.g. the reference's
        2-D diffusion example, BASELINE config 1 (examples/cfd/example_diffusion.py:120-133). Runs on
        `b2_linear_forward`; the coefficients are evaluated when the operator is applied."""
        if len(self._items) != 1 or self._items[0][0] != 'eq' or self._items[0][1].is_Increment:
            raise _Unrecognised("not a single plain equation")
        e = self._items[0][1]
        lhs = e.lhs
        if not (lhs.is_Access and getattr(lhs.function, 'is_TimeFunction', False)):
            raise _Unrecognised("lhs is not a TimeFunction")
        f = lhs.function
        grid = f.grid
        if grid is None or not f.is_buffered or grid.dim not in (1, 2, 3) or grid.distributor.is_parallel:
            raise _Unrecognised("needs a buffered TimeFunction on a non-decomposed 1-D/2-D/3-D grid")
        kl = _space_offsets(lhs, None)
        if kl is None or kl[0] not in (1, -1) or any(kl[1]):
            raise _Unrecognised("lhs is not `f.forward` / `f.backward`")
        terms = self._coeffs(e.rhs, [f])
        taps = []
        for acc, coef in terms.items():
            k = _space_offsets(acc, None)
            if k is None:
                raise _Unrecognised("non-affine access")
            if any(abs(o) > f.space_order for o in k[1]):
                raise _Unrecognised("stencil reaches beyond the halo")
            for n in coef.preorder():
                if n.is_Access:
                    raise _Unrecognised("position-dependent coefficient")
            taps.append((k[0], k[1], coef))
        if not taps or len(taps) > L_.MAX_TAPS or len({t for t, _, _ in taps}) > 4:
            raise _Unrecognised("unsupported number of taps / time levels")
        # the slot rule (as in b2_linear_forward): no level read may share the written slot modulo time_size,
        # or a point would read a cell another point of the same step is writing
        if any((t - kl[0]) % f.time_size == 0 for t, _, _ in taps):
            raise _Unrecognised("a level read shares the written time slot (implicit, or aliased modulo time_size)")
        taps.sort(key=lambda t: (t[0], t[1]))
        # iteration box: the equation's SubDomain (rectangular) or the whole grid
        box = []
        sd = e.subdomain.dimensions if e.subdomain is not None else grid.dimensions
        for d, n in zip(sd, grid.shape):
            box.append(d.bounds(0, n - 1) if d.is_Sub else (0, n - 1))
        tmin = min(t for t, _, _ in taps)
        tmax = max(t for t, _, _ in taps)
        return {'kind': 'linear', 'u': f, 'grid': grid, 'so': f.space_order, 'R': 0, 'taps': taps,
                'wshift': kl[0], 'box': box, 'dt': grid.stepping_dim.spacing, 'src': None, 'rec': None,
                'rec_toff': 0, 'tlo': min(tmin, kl[0], 0), 'thi': max(tmax, kl[0], 0)}

    def _recognise_wave(self):
        eqs = [o for k, o in self._items if k == 'eq']
        injs = [o for k, o in self._items if k == 'inject']
        itps = [o for k, o in self._items if k == 'interp']
        fss = [o for k, o in self._items if k == 'fs']
        incs = [e for e in eqs if e.is_Increment]
        eqs = [e for e in eqs if not e.is_Increment]
        if not eqs:
            raise _Unrecognised("no plain time-update equations")
        # `Eq(usave, u)` with usave saved on a ConditionalDimension: time-subsampled snapshots
        snaps = [e for e in eqs if self._is_snapshot_eq(e)]
        eqs = [e for e in eqs if not self._is_snapshot_eq(e)]
        if not eqs:
            raise _Unrecognised("no plain time-update equations")
        updates = []
        for e in eqs:
            lhs = e.lhs
            if not (lhs.is_Access and getattr(lhs.function, 'is_TimeFunction', False)):
                raise _Unrecognised("lhs is not a TimeFunction")
            f = lhs.function
            so = _space_offsets(lhs, None)
            if so is None or so[0] not in (1, -1) or any(so[1]):
                raise _Unrecognised("lhs is not `f.forward` / `f.backward`")
            self._dirn = so[0]
            if f.time_order != 2:
                raise _Unrecognised("time_order != 2")
            if e.subdomain is not None and any(d.is_Sub for d in e.subdomain.dimensions):
                if not self._covered_by_free_surface(e, fss):
                    raise _Unrecognised("restricted subdomain")
            updates.append((f, e))
        if len(injs) > 1 or len(itps) > 1:
            raise _Unrecognised("more than one injection/interpolation")
        if incs and len(updates) not in (1, 2):
            raise _Unrecognised("increments are only supported next to a single acoustic update or a TTI pair")
        if len(incs) > 1:
            raise _Unrecognised("more than one increment")
        if fss and (len(updates) != 1 or len(fss) != 1 or fss[0].field is not updates[0][0]):
            raise _Unrecognised("a free surface is only on the fast path for the single-field acoustic update")
        if len(updates) == 1:
            try:
                plan = self._recognise_iso(updates[0], injs, itps)
            except _Unrecognised as iso_why:
                if incs or fss or snaps:
                    raise
                try:
                    return self._recognise_sa(updates[0], injs, itps)
                except _Unrecognised as sa_why:
                    raise _Unrecognised(f"{iso_why}; as the self-adjoint update: {sa_why}") from None
            if incs:
                if plan['grid'].dim != 3:
                    raise _Unrecognised("imaging condition is 3-D only")
                plan['grad'] = incs[0].lhs.function
                (plan['usave'],) = self._imaging(plan, incs[0], [plan['u']], 7)
            plan['free_surface'] = bool(fss)
            if fss and plan.get('ot4'):
                raise _Unrecognised("a free surface under the OT4 kernel is not on the fast path yet")
            if snaps:
                self._attach_snapshot(plan, snaps)
            if fss and not self._covered_by_free_surface(updates[0][1], fss):
                raise _Unrecognised("free-surface rows and the update's subdomain do not tile the grid")
            return plan
        if snaps:
            raise _Unrecognised("snapshots are on the fast path next to the single-field acoustic update only")
        if len(updates) == 2 and not incs:
            try:
                return self._recognise_visco(updates, injs, itps)
            except _NotVisco:
                pass            # not the shape of the SLS pair: the TTI / Born recognisers below decide
            except _Unrecognised as visco_why:
                raise _Unrecognised(f"as the SLS viscoacoustic pair: {visco_why}") from None
        if len(updates) == 2 and (self._dirn != 1 or incs):
            if any(_space_offsets(e.lhs, None)[0] != -1 for _, e in updates):
                raise _Unrecognised("the TTI imaging condition needs the backward (adjoint) pair")
            plan = self._recognise_tti_adjoint(updates, injs, itps)
            if incs:
                saved = self._imaging(plan, incs[0], [plan['u'], plan['v']], 17)
                if any(s.grid is not plan['grid'] for s in saved):
                    raise _Unrecognised("the forward wavefields must be saved (save=nt) and read at (time, x, y, z)")
                plan['grad'] = incs[0].lhs.function
                plan['usave'], plan['vsave'] = saved
            return plan
        if len(updates) == 2:
            try:
                return self._recognise_tti(updates, injs, itps)
            except _Unrecognised as tti_why:
                try:
                    return self._recognise_born(updates, injs, itps)
                except _Unrecognised as born_why:
                    raise _Unrecognised(f"neither TTI ({tti_why}) nor Born ({born_why})") from None
        if len(updates) == 4:
            if any(_space_offsets(e.lhs, None)[0] != 1 for _, e in updates):
                raise _Unrecognised("TTI Born is on the fast path forward in time only")
            return self._recognise_tti_born(updates, injs, itps)
        raise _Unrecognised("unsupported number of update equations")

    @staticmethod
    def _is_snapshot_eq(e):
        f = e.lhs.function if e.lhs.is_Access else None
        return (f is not None and getattr(f, 'is_TimeFunction', False) and not f.is_buffered and
                getattr(f.time_dim, 'is_Conditional', False))

    def _attach_snapshot(self, plan, snaps):
        """`Eq(usave, u)` / `Eq(usave, u.forward)`, usave = TimeFunction(save=nsnaps, time_dim=
        ConditionalDimension(parent=time, factor=f)) — examples/seismic/tutorials/08_snapshotting.ipynb:
        455-505: every f-th step the wavefield is copied into usave[time / f]."""
        if len(snaps) != 1 or plan.get('adjoint'):
            raise _Unrecognised("one snapshot equation, forward time stepping only")
        e = snaps[0]
        us, u = e.lhs.function, plan['u']
        tdim = us.time_dim
        if tdim.condition is not None or not tdim.factor or int(tdim.factor) < 1 or \
                tdim.parent is not plan['grid'].time_dim:
            raise _Unrecognised("snapshots need a ConditionalDimension(parent=grid.time_dim, factor=n)")
        kl = _space_offsets(e.lhs, None)
        rhs = e.rhs.evaluate if hasattr(e.rhs, 'evaluate') else e.rhs
        if not (rhs.is_Access and rhs.function is u):
            raise _Unrecognised("a snapshot must copy the wavefield itself")
        kr = _space_offsets(rhs, None)
        if kl is None or kr is None or kl[0] != 0 or any(kl[1]) or any(kr[1]) or kr[0] not in (0, 1):
            raise _Unrecognised("a snapshot must be `Eq(usave, u)` or `Eq(usave, u.forward)` at the same point")
        if us.grid is not plan['grid'] or e.subdomain is not None:
            raise _Unrecognised("snapshots cover the whole grid")
        plan['snap'] = us
        plan['snap_factor'] = int(tdim.factor)
        plan['snap_toff'] = int(kr[0])

    @staticmethod
    def _covered_by_free_surface(eq, fss):
        """The reference pairs the update on `physdomain` = z in [so, z_M] (examples/seismic/model.py:
        67-79) with the free-surface rows `fsdomain` = z in [0, so) (model.py:82-98): together they tile
        the grid. True iff `eq`'s subdomain and the FreeSurface's subdomain are that pair (any equal
        thickness), restricted on the LAST dimension only, and the FreeSurface mirrors this very update."""
        if len(fss) != 1:
            return False
        fs = fss[0]
        if fs.eq is not eq and (fs.eq.lhs != eq.lhs or fs.eq.rhs is not eq.rhs):
            return False
        if eq.subdomain is None or fs.subdomain is None:
            return False
        pd, fd = eq.subdomain.dimensions, fs.subdomain.dimensions
        if len(pd) != len(fd) or any(d.is_Sub for d in pd[:-1]) or any(d.is_Sub for d in fd[:-1]):
            return False
        zp, zf = pd[-1], fd[-1]
        if not (zp.is_Sub and zf.is_Sub and zp.parent is zf.parent):
            return False
        return (zp.kind == 'middle' and zf.kind == 'left' and zp.thickness[1] == 0 and
                zp.thickness[0] == zf.thickness[0] and zf.thickness[0] >= eq.lhs.function.space_order // 2)

    def _coeffs(self, rhs, fields):
        rhs = rhs.evaluate
        if self._subs:
            rhs = rhs.subs(self._subs)
        fset = {id(f) for f in fields}
        try:
            terms, rest = linear_terms(rhs, lambda a: id(a.function) in fset)
        except NonLinear as e:
            raise _Unrecognised(f"update is not linear in the wavefield: {e}") from None
        if not (rest.is_Number and float(rest.value) == 0.0):
            raise _Unrecognised("update has a source term that is not a sparse injection")
        return terms

    def _taps(self, rhs, fields, tags=None):
        """{tap: coefficient} of an update linear in `fields`. A tap is the access's (time_shift, offsets), led by
        the entry of `tags` that belongs to the field read when `tags` (one per field) is given."""
        tag = {id(f): t for f, t in zip(fields, tags or ())}
        out = {}
        for acc, coef in self._coeffs(rhs, fields).items():
            k = _space_offsets(acc, None)
            if k is None:
                raise _Unrecognised("non-affine wavefield access")
            out[(tag[id(acc.function)],) + k if tags else k] = coef
        return out

    @staticmethod
    def _leaves(exprs):
        """Non-wavefield leaves of the coefficient expressions."""
        funcs, consts, syms = {}, {}, {}
        for ex in exprs:
            for n in ex.preorder():
                if n.is_Access:
                    funcs[id(n.function)] = n
                elif n.is_Constant:
                    consts[id(n)] = n
                elif n.is_Symbol and not n.is_Dimension:
                    syms[n.name] = n
        return list(funcs.values()), list(consts.values()), list(syms.values())

    def _probe_env(self, rng, funcs, consts, syms, grid, fixed=None):
        vals = {}
        for a in funcs:
            vals[('f', id(a.function))] = rng.uniform(0.5, 2.0)
        for c in consts:
            vals[('c', id(c))] = rng.uniform(0.1, 0.9)
        for s in syms:
            vals[('s', s.name)] = rng.uniform(0.5, 2.0)
        for sp, v in grid.spacing_map.items():
            vals[('s', sp.name)] = float(v)
        vals.update(fixed or {})

        def leaf(n):
            if n.is_Access:
                return vals[('f', id(n.function))]
            if n.is_Constant:
                return vals[('c', id(n))]
            return vals[('s', n.name)]
        return vals, leaf

    def _spacing_values(self, grid):
        out = []
        for d, h in zip(grid.dimensions, grid.spacing):
            v = self._subs.get(d.spacing)
            out.append(float(v if v is not None else h))
        return out

    def _recognise_iso(self, update, injs, itps):
        u, eq = update
        grid = u.grid
        nd = grid.dim
        if nd not in (2, 3):
            raise _Unrecognised("only 2-D/3-D grids")
        so = u.space_order
        if so % 2 or so < 2 or so // 2 > 8:
            raise _Unrecognised(f"space_order {so} unsupported")
        R = so // 2
        # the stencil support must be exactly the (2R*nd + 1)-point star at t plus the centre at t-1
        keyed = self._taps(eq.rhs, [u])
        zero = (0,) * nd
        star = {(0, zero)}
        for d in range(nd):
            for k in range(1, R + 1):
                for s in (-k, k):
                    o = [0] * nd
                    o[d] = s
                    star.add((0, tuple(o)))
        dirn = self._dirn
        if set(keyed) != star | {(-dirn, zero)}:
            if set(keyed) > star | {(-dirn, zero)}:
                plan = self._recognise_ot4(u, keyed, star, R)
                funcs, consts, syms = self._leaves(keyed.values())
                self._attach_sparse(plan, injs, itps, [u], funcs, consts, syms, plan['m_role'])
                return plan
            raise _Unrecognised("stencil support is not the isotropic star")
        funcs, consts, syms = self._leaves(keyed.values())
        for a in funcs:
            k = _space_offsets(a, None)
            if getattr(a.function, 'is_TimeFunction', False) or k is None or any(k[1]):
                raise _Unrecognised("parameter field accessed off-centre")
        dtsym = grid.stepping_dim.spacing
        hs = self._spacing_values(grid)
        w = [second_derivative_weights(so, h) for h in hs]
        rng = np.random.default_rng(1234)
        roles = None
        for probe in range(3):
            vals, leaf = self._probe_env(rng, funcs, consts, syms, grid)
            dt = vals.get(('s', dtsym.name))
            if dt is None:
                raise _Unrecognised("no time spacing in the update")
            c = {k: eval_scalar(v, leaf) for k, v in keyed.items()}
            o1 = [0] * nd
            o1[-1] = 1
            cz = c[(0, tuple(o1))]
            if cz == 0:
                raise _Unrecognised("degenerate stencil")
            den = w[-1][1] / cz
            m_eff = -c[(-dirn, zero)] * dt * dt * den
            d_eff = (den - m_eff / (dt * dt)) * dt
            if roles is None:
                roles = self._iso_roles(m_eff, d_eff, den, vals, funcs, consts)
            # verify the full stencil against the kernel's formula
            m_role, d_role = roles
            m_chk = self._role_value(m_role, vals)
            d_chk = self._role_value(d_role, vals) if d_role is not None else 0.0
            den_chk = m_chk / (dt * dt) + d_chk / dt
            pred = {(-dirn, zero): -m_chk / (dt * dt) / den_chk,
                    (0, zero): (2 * m_chk / (dt * dt) + d_chk / dt + sum(wd[0] for wd in w)) / den_chk}
            for d in range(nd):
                for k in range(1, R + 1):
                    for s in (-k, k):
                        o = [0] * nd
                        o[d] = s
                        pred[(0, tuple(o))] = w[d][k] / den_chk
            for k, v in pred.items():
                if abs(c[k] - v) > 1e-9 * max(1.0, abs(v)):
                    raise _Unrecognised(f"coefficient mismatch at {k}: {c[k]} vs {v}")
        m_role, d_role = roles
        plan = {'kind': 'iso', 'u': u, 'grid': grid, 'so': so, 'R': R, 'w': w,
                'm_role': m_role, 'damp': d_role[1] if d_role is not None else None,
                'dt': dtsym, 'src': None, 'rec': None, 'rec_toff': 0, 'adjoint': dirn == -1}
        self._attach_sparse(plan, injs, itps, [u], funcs, consts, syms, m_role)
        return plan

    def _recognise_sa(self, update, injs, itps):
        """The reference's self-adjoint variable-density visco-acoustic update (examples/seismic/self_adjoint/
        operators.py:4-65 `iso_stencil`): u_next = dt^2 vp^2/b * sum_d (b u.d(x0=d+h/2)).d(x0=d-h/2)
        + (2 - dt w) u + (dt w - 1) u_prev. The radius and weights follow from the support; the roles of the
        parameter leaves (b, vp, w) are tried in turn, and each candidate is checked by comparing EVERY stencil
        coefficient with `predict_sa` at probe values that vary linearly in space, a different gradient per
        Function and axis, so that where b is sampled (node, half node, output point) changes the prediction."""
        u, eq = update
        grid = u.grid
        nd = grid.dim
        if nd not in (2, 3):
            raise _Unrecognised("only 2-D/3-D grids")
        so = u.space_order
        keyed = self._taps(eq.rhs, [u])
        dirn = self._dirn
        zero = (0,) * nd
        R, leaves, c, fcands, cands, probes = self._nested_front(
            [k[1] for k in keyed], keyed.values(), grid, so, 2468)
        star = {(0, zero), (-dirn, zero)}
        for d in range(nd):
            for s in range(1 - 2 * R, 2 * R):
                o = [0] * nd
                o[d] = s
                star.add((0, tuple(o)))
        if set(keyed) != star:
            raise _Unrecognised("stencil support is not the star of radius 2R-1 plus the centre of the other level")

        def match(roles, w_role):
            b, vp = (x[1] for x in roles)
            for value, leaf, dt in probes:
                pred = predict_sa(c, R, nd, lambda off: value(b, off), value(vp, zero),
                                  value(w_role[1], zero) if w_role else 0.0, dt, dirn)
                if not self._nested_matches([(keyed, pred)], leaf):
                    return None
            return roles + (w_role,)
        found = self._find_roles(cands, fcands, 2, match)
        if found is None:
            raise _Unrecognised("coefficients are not those of the self-adjoint update for any roles of "
                                "b, vp and w/Q")
        b_role, vp_role, w_role = found
        plan = {'kind': 'sa', 'u': u, 'grid': grid, 'so': so, 'R': R, 'c': c,
                'b_role': b_role, 'vp_role': vp_role, 'damp': w_role[1] if w_role else None,
                'dt': grid.stepping_dim.spacing, 'src': None, 'rec': None, 'rec_toff': 0, 'adjoint': dirn == -1}
        self._attach_sa_sparse(plan, injs, itps, *leaves)
        return plan

    def _nested_front(self, offsets, exprs, grid, so, seed):
        """What recognising the self-adjoint update and the SLS pair shares, both applying the nested operator L:
        L's radius R from the reach of the wavefield's tap `offsets`; the leaves of the coefficient expressions
        `exprs`, which read no other wavefield, dt and no unknown symbol; L's weights c; the candidates for the
        parameter roles (the Functions, then all); and three probes drawn from `seed`."""
        reach = max((max(abs(o) for o in off) for off in offsets), default=0)
        if reach % 2 == 0:
            raise _Unrecognised("support is not that of nested half-node first derivatives")
        R = (reach + 1) // 2
        if 2 * R > so or R > 8:
            raise _Unrecognised(f"radius {2 * R - 1} does not fit the halo of space_order {so}")
        funcs, consts, syms = self._leaves(exprs)
        for a in funcs:
            if getattr(a.function, 'is_TimeFunction', False):
                raise _Unrecognised("another wavefield in the coefficients")
        dtsym = grid.stepping_dim.spacing
        if dtsym.name not in {s.name for s in syms}:
            raise _Unrecognised("no time spacing in the update")
        known = {dtsym.name} | {sp.name for sp in grid.spacing_map}
        for sym in syms:
            if sym.name not in known:
                raise _Unrecognised(f"unknown symbol {sym.name} in the update")
        c = [sa_weights(R, h) for h in self._spacing_values(grid)]
        fcands = [('f', a.function) for a in funcs]
        cands = fcands + [('c', cst) for cst in consts]
        rng = np.random.default_rng(seed)
        probes = [self._sa_probe(rng, cands, grid) for _ in range(3)]
        return R, (funcs, consts, syms), c, fcands, cands, probes

    @staticmethod
    def _find_roles(cands, fcands, n, match):
        """The first result of `match(roles, damping role)` that is not None: `roles` are n distinct candidates in
        the order of `itertools.permutations`, the damping role is a Function of `fcands` outside them or None, and
        every candidate has a role."""
        every = {id(x[1]) for x in cands}
        for roles in itertools.permutations(cands, n):
            for d_role in [x for x in fcands if all(x is not y for y in roles)] + [None]:
                if {id(x[1]) for x in roles + (d_role,) if x is not None} == every:
                    found = match(roles, d_role)
                    if found is not None:
                        return found
        return None

    @staticmethod
    def _nested_matches(pairs, leaf):
        """Whether, for each (keyed coefficient expressions, predicted coefficients) of `pairs`, the taps are the
        predicted ones and each coefficient evaluated at `leaf` is within 1e-9 times the largest predicted one."""
        for keyed, pred in pairs:
            got = {k: eval_scalar(v, leaf) for k, v in keyed.items()}
            scale = max(abs(v) for v in pred.values())
            if set(got) != set(pred) or not all(abs(got[k] - pred[k]) <= 1e-9 * scale for k in pred):
                return False
        return True

    def _sa_probe(self, rng, cands, grid):
        """Probe values: a Function is base + grad . offset (linear in space), a Constant one number."""
        vals = {}
        for kind, obj in cands:
            if kind == 'f':
                vals[id(obj)] = (rng.uniform(1.0, 2.0), rng.uniform(-0.05, 0.05, size=grid.dim))
            else:
                vals[id(obj)] = (rng.uniform(0.5, 2.0), np.zeros(grid.dim))
        dt = rng.uniform(0.5, 2.0)
        spc = {sp.name: float(v) for sp, v in grid.spacing_map.items()}
        spc[grid.stepping_dim.spacing.name] = dt

        def value(obj, off):
            base, g = vals[id(obj)]
            return base + float(np.dot(g, off))

        def leaf(n):
            if n.is_Access:
                k = _space_offsets(n, None)
                return value(n.function, k[1] if k is not None else (0,) * grid.dim)
            if n.is_Constant:
                return value(n, (0,) * grid.dim)
            return spc[n.name]           # _nested_front refused every other symbol
        return value, leaf, dt

    def _attach_sa_sparse(self, plan, injs, itps, funcs, consts, syms, scale=None, what="src*dt^2*vp^2/b"):
        """Injection `src * dt^2 * vp^2 / b` into the level written (operators.py:101, :149), checked at random
        values; receivers / the adjoint source as for the acoustic update."""
        grid, dtsym = plan['grid'], plan['dt']
        if injs:
            sf, ((ex, (f2, c2, s2)),) = self._injection(injs[0], [plan['u']])
            if dtsym.name not in {s.name for s in s2}:
                raise _Unrecognised("injected expression has no time spacing")
            for sym in s2:
                if sym.name != dtsym.name and sym.name not in {sp.name for sp in grid.spacing_map}:
                    raise _Unrecognised(f"unknown symbol {sym.name} in the injected expression")
            rng = np.random.default_rng(8642)
            roles = [plan['b_role'], plan['vp_role']]
            known = {id(o) for _, o in roles} | {id(sf)}
            if any(id(acc.function) not in known for acc in f2) or any(id(cc) not in known for cc in c2):
                raise _Unrecognised("injected expression has parameters other than vp and b")
            for _ in range(2):
                vals = {i: rng.uniform(0.5, 2.0) for i in known}
                dt = rng.uniform(0.5, 2.0)
                spc = {sp.name: float(v) for sp, v in grid.spacing_map.items()}

                def leaf(n):
                    if n.is_Access:
                        return vals[id(n.function)]
                    if n.is_Constant:
                        return vals[id(n)]
                    return dt if n.name == dtsym.name else spc[n.name]
                vp_, b_ = vals[id(plan['vp_role'][1])], vals[id(plan['b_role'][1])]
                want = vals[id(sf)] * dt * dt * (vp_ ** 2 / b_ if scale is None else scale(vp_, b_))
                if abs(eval_scalar(ex, leaf) - want) > 1e-9 * abs(want):
                    raise _Unrecognised(f"injected expression is not {what}")
            plan['src'] = sf
        if itps:
            self._attach_sparse(plan, [], itps, [plan['u']], funcs, consts, syms, None)

    def _recognise_visco(self, updates, injs, itps):
        """The reference's second-order SLS viscoacoustic pair (examples/seismic/viscoacoustic/operators.py:124-192,
        kernel='sls', time_order=2): r.forward|backward, then p.forward|backward reading r at the level just written.
        The radius and weights follow from the support of p; the roles of the parameter leaves (b, vp, qp and the
        damping mask) are tried in turn, f0 is solved from the coefficient of r[t], and each candidate is checked by
        comparing EVERY coefficient of both equations with `predict_visco` at probe values that vary linearly in
        space (`_sa_probe`), so that where b, rho and tt are sampled changes the prediction."""
        (r, e1), (p, e2) = updates
        dirn = self._dirn
        reads = lambda e, f: [k for k in (_space_offsets(a, None) for a in e.rhs.evaluate.preorder()
                                          if a.is_Access and a.function is f) if k is not None]
        r_in_p = reads(e2, r)
        if not r_in_p or any(k[0] != dirn for k in r_in_p) or any(k[0] == dirn for k in reads(e1, p)):
            raise _NotVisco("the second update does not read the first at the level just written")
        grid = p.grid
        nd = grid.dim
        if nd not in (2, 3):
            raise _Unrecognised("only 2-D/3-D grids")
        so = p.space_order
        if r.space_order != so or r.grid is not grid or r.time_size != p.time_size:
            raise _Unrecognised("p and r differ in space order, grid or time slots")
        keyed = [self._taps(e.rhs, [p, r], ('p', 'r')) for e in (e1, e2)]
        R, leaves, c, fcands, cands, probes = self._nested_front(
            [k[2] for k in keyed[1] if k[0] == 'p'], list(keyed[0].values()) + list(keyed[1].values()), grid, so, 1357)
        at = lambda value, role: (lambda off: value(role[1], off)) if role else (lambda off: 1.0)

        def match(roles, d_role):
            f0 = self._visco_f0(keyed, probes[0], roles, d_role, nd, dirn)
            if f0 is None:
                return None
            for value, leaf, dt in probes:
                pred = predict_visco(c, R, nd, *(at(value, x) for x in roles), at(value, d_role), f0, dt, dirn)
                if not self._nested_matches(zip(keyed, pred), leaf):
                    return None
            return roles + (d_role, f0)
        found = self._find_roles(cands, fcands, 3, match)
        if found is None:
            raise _Unrecognised("coefficients are not those of the SLS update for any roles of b, vp, qp and damp")
        b_role, vp_role, qp_role, d_role, f0 = found
        plan = {'kind': 'visco', 'u': p, 'r': r, 'grid': grid, 'so': so, 'R': R, 'c': c, 'b_role': b_role,
                'vp_role': vp_role, 'qp_role': qp_role, 'damp': d_role[1] if d_role else None,
                'f0': float(np.float32(f0)), 'dt': grid.stepping_dim.spacing, 'src': None, 'rec': None,
                'rec_toff': 0, 'adjoint': dirn == -1}
        self._attach_sa_sparse(plan, injs, itps, *leaves, scale=lambda vp, b: vp * vp, what="src*dt^2/m")
        return plan

    @staticmethod
    def _visco_f0(keyed, probe, roles, d_role, nd, dirn):
        """f0 from the coefficient damp (1 - dt/t_s) of r[t] in the memory-variable update, or None."""
        value, leaf, dt = probe
        zero = (0,) * nd
        coef = keyed[0].get(('r', 0, zero))
        damp = value(d_role[1], zero) if d_role else 1.0
        if coef is None:
            return None
        den = 1.0 - eval_scalar(coef, leaf) / damp
        qp = value(roles[2][1], zero)
        if den <= 0 or qp <= 0:
            return None
        t_s = dt / den
        f0 = (np.sqrt(1.0 + 1.0 / qp ** 2) - 1.0 / qp) / t_s
        return f0 if np.isfinite(f0) and f0 > 0 else None

    def _recognise_ot4(self, u, keyed, star, R):
        """The reference's 4th-order-in-time acoustic update (examples/seismic/acoustic/operators.py:
        50-68, kernel='OT4'):  H = lap(u) + dt^2/12 * lap( lap(u)/m ), the inner Laplacian and 1/m
        sampled at the shifted point. The candidate roles of the parameter leaves are tried in turn;
        each is checked by comparing EVERY stencil coefficient with the prediction at random parameter
        values that also carry a random spatial gradient (so the sampling position of 1/m is checked)."""
        grid = u.grid
        nd = grid.dim
        dirn = self._dirn
        zero = (0,) * nd
        if 2 * R > u.space_order:
            raise _Unrecognised("OT4 needs a halo of 2*radius points")
        funcs, consts, syms = self._leaves(keyed.values())
        for a in funcs:
            if getattr(a.function, 'is_TimeFunction', False) or _space_offsets(a, None) is None:
                raise _Unrecognised("non-affine parameter access")
        dtsym = grid.stepping_dim.spacing
        hs = self._spacing_values(grid)
        w = [second_derivative_weights(u.space_order, h) for h in hs]
        spv = {sp.name: float(v) for sp, v in grid.spacing_map.items()}
        fobjs = [a.function for a in funcs]
        m_cands = [('vp_f', f) for f in fobjs] + [('m_f', f) for f in fobjs] + \
                  [('vp_c', c) for c in consts] + [('m_c', c) for c in consts] + [('one', None)]
        d_cands = [None] + [('damp_f', f) for f in fobjs]

        def unit(d, o):
            v = [0] * nd
            v[d] = o
            return tuple(v)

        def mismatch(m_role, d_role, seed):
            rng = np.random.default_rng(seed)
            base = {id(f): rng.uniform(0.6, 1.6) for f in fobjs}
            gradv = {id(f): rng.uniform(-0.02, 0.02, size=nd) for f in fobjs}
            cval = {id(c): rng.uniform(0.6, 1.6) for c in consts}
            dt = rng.uniform(0.5, 2.0)

            def fval(f, off):
                return float(base[id(f)] + np.dot(gradv[id(f)], off))

            def leaf(n):
                if n.is_Access:
                    return fval(n.function, _space_offsets(n, None)[1])
                if n.is_Constant:
                    return cval[id(n)]
                if n.name == dtsym.name:
                    return dt
                if n.name in spv:
                    return spv[n.name]
                raise _Unrecognised(f"unknown symbol {n.name} in the update")

            def m_at(off):
                kind, obj = m_role
                if kind == 'vp_f':
                    return 1.0 / fval(obj, off) ** 2
                if kind == 'm_f':
                    return fval(obj, off)
                if kind == 'vp_c':
                    return 1.0 / cval[id(obj)] ** 2
                if kind == 'm_c':
                    return cval[id(obj)]
                return 1.0
            dval = fval(d_role[1], zero) if d_role is not None else 0.0
            m0 = m_at(zero)
            den = m0 / dt ** 2 + dval / dt
            lap = {zero: sum(wd[0] for wd in w)}
            for d in range(nd):
                for k in range(1, R + 1):
                    for sgn in (-k, k):
                        lap[unit(d, sgn)] = w[d][k]
            H = dict(lap)
            for q, wq in lap.items():                       # outer Laplacian tap at q
                for o, wo in lap.items():                   # inner Laplacian tap about q
                    key = tuple(a + b for a, b in zip(q, o))
                    H[key] = H.get(key, 0.0) + dt ** 2 / 12.0 * wq / m_at(q) * wo
            pred = {(0, k): v / den for k, v in H.items()}
            pred[(0, zero)] += (2 * m0 / dt ** 2 + dval / dt) / den
            pred[(-dirn, zero)] = -m0 / dt ** 2 / den
            for k in set(pred) | set(keyed):
                got = eval_scalar(keyed[k], leaf) if k in keyed else 0.0
                want = pred.get(k, 0.0)
                if abs(got - want) > 1e-8 * max(1.0, abs(want)):
                    return f"coefficient mismatch at {k}: {got} vs {want}"
            return None

        why = "no parameter leaves"
        for m_role in m_cands:
            for d_role in d_cands:
                if d_role is not None and m_role[1] is d_role[1]:
                    continue
                why = mismatch(m_role, d_role, 2024) or mismatch(m_role, d_role, 4048)
                if why is None:
                    return {'kind': 'iso', 'u': u, 'grid': grid, 'so': u.space_order, 'R': R, 'w': w,
                            'm_role': m_role, 'damp': d_role[1] if d_role is not None else None,
                            'dt': dtsym, 'src': None, 'rec': None, 'rec_toff': 0, 'adjoint': dirn == -1,
                            'ot4': True}
        raise _Unrecognised(f"not the OT4 acoustic update ({why})")

    @staticmethod
    def _role_value(role, vals):
        kind, obj = role
        if kind == 'vp_f':
            v = vals[('f', id(obj))]
            return 1.0 / (v * v)
        if kind == 'vp_c':
            v = vals[('c', id(obj))]
            return 1.0 / (v * v)
        if kind == 'm_f':
            return vals[('f', id(obj))]
        if kind == 'm_c':
            return vals[('c', id(obj))]
        if kind == 'damp_f':
            return vals[('f', id(obj))]
        if kind == 'one':
            return 1.0
        raise KeyError(kind)

    def _iso_roles(self, m_eff, d_eff, den, vals, funcs, consts):
        def close(a, b):
            return abs(a - b) <= 1e-9 * max(1.0, abs(b))
        m_role = None
        for a in funcs:
            v = vals[('f', id(a.function))]
            if close(m_eff, 1.0 / (v * v)):
                m_role = ('vp_f', a.function)
            elif close(m_eff, v):
                m_role = ('m_f', a.function)
        for cst in consts:
            v = vals[('c', id(cst))]
            if close(m_eff, 1.0 / (v * v)):
                m_role = ('vp_c', cst)
            elif close(m_eff, v):
                m_role = ('m_c', cst)
        if m_role is None and close(m_eff, 1.0):
            m_role = ('one', None)
        if m_role is None:
            raise _Unrecognised("cannot identify the squared-slowness parameter")
        d_role = None
        if abs(d_eff) > 1e-9 * abs(den):
            for a in funcs:
                if close(d_eff, vals[('f', id(a.function))]):
                    d_role = ('damp_f', a.function)
            if d_role is None:
                raise _Unrecognised("cannot identify the damping field")
        return m_role, d_role

    @staticmethod
    def _check_radius(sf, fields):
        """devito/operations/interpolators.py:28-37 `check_radius`: the support of a sparse point reaches
        `r` cells beyond the domain, so it must fit in the halo of every field it touches."""
        so = min(f.space_order for f in fields)
        if so < sf.r:
            raise ValueError(f"Space order {so} too small for interpolation r {sf.r}")

    def _injection(self, inj, fields):
        """The checks every injection passes, whatever value it injects: a SparseTimeFunction with linear or sinc
        interpolation that fits the halo, injected once into each of `fields` at the level written, each expression
        containing the source. Returns the source and, per target, the evaluated expression and its leaves."""
        sf = inj.sfunction
        if not isinstance(sf, SparseTimeFunction) or sf.interpolation not in ('linear', 'sinc'):
            raise _Unrecognised("unsupported sparse function for injection")
        self._check_radius(sf, fields)
        if sorted(id(a.function) for a in inj.fields) != sorted(id(f) for f in fields):
            raise _Unrecognised("injection targets differ from the updated fields")
        targets = []
        for a, ex in zip(inj.fields, inj.exprs):
            k = _space_offsets(a, None)
            if k is None or k[0] != self._dirn or any(k[1]):
                raise _Unrecognised("injection must target the updated time level")
            ex = ex.evaluate.subs(self._subs) if self._subs else ex.evaluate
            leaves = self._leaves([ex])
            if not any(acc.function is sf for acc in leaves[0]):
                raise _Unrecognised("injected expression does not contain the source")
            targets.append((ex, leaves))
        return sf, targets

    def _attach_sparse(self, plan, injs, itps, fields, funcs, consts, syms, m_role):
        grid = plan['grid']
        dtsym = plan['dt']
        rng = np.random.default_rng(4321)
        if injs:
            sf, targets = self._injection(injs[0], fields)
            for ex, (f2, c2, s2) in targets:
                literal = dtsym.name not in {s.name for s in s2}
                lits = []
                for probe in range(2):
                    # the update's leaves are in scope too, so that the role of m always has a value
                    # (an expression without m must then fail the comparison, not the lookup)
                    vals, leaf = self._probe_env(rng, list(funcs) + f2, list(consts) + c2, list(syms) + s2, grid)
                    srcv = vals[('f', id(sf))]
                    dt = vals.get(('s', dtsym.name))
                    got = eval_scalar(ex, leaf)
                    if literal:
                        # `src * dt**2 / m` with a literal dt (tests/test_gpu_openacc.py:205-251): the literal is
                        # got * m / src, which must not depend on the probe
                        lits.append(got * self._role_value(m_role, vals) / srcv)
                        continue
                    want = srcv * dt * dt / self._role_value(m_role, vals)
                    if abs(got - want) > 1e-9 * max(1.0, abs(want)):
                        raise _Unrecognised("injected expression is not src*dt^2/m")
                if literal:
                    if abs(lits[1] - lits[0]) > 1e-9 * max(abs(lits[0]), 1e-30) or not lits[0] > 0:
                        raise _Unrecognised("injected expression with a literal dt is not src*lit/m")
                    plan['inject_literal'] = True
                    plan['inject_dt2'] = lits[0]
            plan['src'] = sf
        if itps:
            itp = itps[0]
            sf = itp.sfunction
            if not isinstance(sf, SparseTimeFunction) or sf.interpolation not in ('linear', 'sinc'):
                raise _Unrecognised("unsupported sparse function for interpolation")
            self._check_radius(sf, fields)
            if itp.increment:
                raise _Unrecognised("incremental interpolation")
            ex = itp.expr.evaluate
            accs = [n for n in ex.preorder() if n.is_Access]
            if {id(a.function) for a in accs} != {id(f) for f in fields} or len(accs) != len(fields):
                raise _Unrecognised("interpolated expression is not the (sum of the) wavefield(s)")
            toffs = set()
            for a in accs:
                k = _space_offsets(a, None)
                if k is None or any(k[1]) or k[0] not in (0, self._dirn):
                    raise _Unrecognised("interpolated access must be f or the updated time level")
                toffs.add(k[0])
            if len(toffs) != 1:
                raise _Unrecognised("mixed time offsets in the interpolated expression")
            # must be a plain sum with unit coefficients
            vals = {id(a.function): float(i + 2) for i, a in enumerate(accs)}
            got = eval_scalar(ex, lambda n: vals[id(n.function)])
            if abs(got - sum(vals.values())) > 1e-12:
                raise _Unrecognised("interpolated expression is not a plain sum")
            plan['rec'] = sf
            plan['rec_toff'] = 1 if toffs.pop() != 0 else 0

    def _recognise_born(self, updates, injs, itps):
        """The reference's linearised-modelling operator (examples/seismic/acoustic/operators.py:
        235-277): `eqn1 = iso_stencil(u)`, `eqn2 = iso_stencil(U, q=-dm*u.dt2)`, the source injected
        into `u.forward`, the receivers sampling `U`. eqn2 must be eqn1's stencil applied to U plus
        `-dm (u[t+1] - 2u[t] + u[t-1]) / dt^2` divided by the same denominator."""
        fields = [f for f, _ in updates]

        def depends_on(eq, f):
            return any(n.is_Access and n.function is f for n in eq.rhs.evaluate.preorder())
        first = [(f, e) for (f, e) in updates if not any(depends_on(e, g) for g in fields if g is not f)]
        if len(first) != 1:
            raise _Unrecognised("no update that is independent of the other field")
        (u, equ) = first[0]
        (U, eqU) = [(f, e) for (f, e) in updates if f is not u][0]
        if U.grid is not u.grid or U.space_order != u.space_order or u.grid.dim != 3:
            raise _Unrecognised("Born needs two 3-D wavefields of the same space order")
        # the background update alone is the plain acoustic operator (it also fixes the parameter roles)
        plan = self._recognise_iso((u, equ), [], [])
        if plan.get('ot4') or plan.get('adjoint'):
            raise _Unrecognised("Born is on the fast path for the forward OT2 update only")
        grid = plan['grid']
        tU = self._taps(eqU.rhs, [u, U], ('u', 'U'))
        ku = self._taps(equ.rhs, [u])
        kU = {k[1:]: coef for k, coef in tU.items() if k[0] == 'U'}
        kq = {k[1:]: coef for k, coef in tU.items() if k[0] == 'u'}
        zero = (0, 0, 0)
        if set(kU) != set(ku) or set(kq) != {(1, zero), (0, zero), (-1, zero)}:
            raise _Unrecognised("second update is not the background stencil plus a centred u.dt2 term")
        funcs, consts, syms = self._leaves(list(kU.values()) + list(kq.values()))
        known = {id(plan['damp'])} if plan.get('damp') is not None else set()
        if plan['m_role'][1] is not None:
            known.add(id(plan['m_role'][1]))
        extra = [a for a in funcs if id(a.function) not in known]
        if len(extra) != 1 or getattr(extra[0].function, 'is_TimeFunction', False):
            raise _Unrecognised("cannot identify the model perturbation dm")
        dm = extra[0].function
        kd = _space_offsets(extra[0], None)
        if kd is None or any(kd[1]):
            raise _Unrecognised("dm accessed off-centre")
        dtsym = plan['dt']
        rng = np.random.default_rng(515)
        for probe in range(2):
            vals, leaf = self._probe_env(rng, funcs, consts, syms, grid)
            dt = vals[('s', dtsym.name)]
            m_val = self._role_value(plan['m_role'], vals)
            d_val = vals[('f', id(plan['damp']))] if plan.get('damp') is not None else 0.0
            den = m_val / dt ** 2 + d_val / dt
            dmv = vals[('f', id(dm))]
            for k, coef in kU.items():
                if abs(eval_scalar(coef, leaf) - eval_scalar(ku[k], leaf)) > 1e-9 * max(1.0, abs(eval_scalar(ku[k], leaf))):
                    raise _Unrecognised(f"U is not updated with the background stencil (tap {k})")
            want = {(1, zero): -dmv / dt ** 2 / den, (0, zero): 2 * dmv / dt ** 2 / den, (-1, zero): -dmv / dt ** 2 / den}
            for k, wv in want.items():
                if abs(eval_scalar(kq[k], leaf) - wv) > 1e-9 * max(1.0, abs(wv)):
                    raise _Unrecognised("the source of the second update is not -dm * u.dt2")
        # sparse terms: the source drives u, the receivers sample U
        fu, cu, su = self._leaves(ku.values())
        self._attach_sparse(plan, injs, [], [u], fu, cu, su, plan['m_role'])
        self._attach_sparse(plan, [], itps, [U], fu, cu, su, plan['m_role'])
        plan['born_U'] = U
        plan['born_dm'] = dm
        return plan

    def _imaging(self, plan, inc, fields, seed):
        """`Inc(g, -sum_i s_i * f_i.dt2)` next to the adjoint update of `fields`, each s_i a forward wavefield saved
        (save=nt) and read at (time, x, y, z): the reference's Gradient operator (examples/seismic/acoustic/
        operators.py:190-232) for one field, its `GradientTTI` (tti/operators.py `JacobianAdjOperator`) for the TTI
        pair. The coefficients are checked at values drawn from `seed`. Returns the s_i, in the order of `fields`."""
        grid = plan['grid']
        form = ' + '.join(f'saved * {f.name}.dt2' for f in fields)
        lhs = inc.lhs
        if not (lhs.is_Access and isinstance(lhs.function, Function) and not lhs.function.is_TimeFunction):
            raise _Unrecognised("increment target is not a Function")
        if lhs.function.grid is not grid:
            raise _Unrecognised("increment target lives on another grid")
        k = _space_offsets(lhs, None)
        if k is None or any(k[1]):
            raise _Unrecognised("increment target accessed off-centre")
        rhs = inc.rhs.evaluate
        if self._subs:
            rhs = rhs.subs(self._subs)
        ids = {id(f) for f in fields}
        try:
            terms, rest = linear_terms(rhs, lambda a: id(a.function) in ids)
        except NonLinear as e:
            raise _Unrecognised(f"increment is not linear in the adjoint wavefields: {e}") from None
        if not (rest.is_Number and float(rest.value) == 0.0):
            raise _Unrecognised("increment has terms without the adjoint wavefields")
        keyed = {id(f): {} for f in fields}
        for acc, coef in terms.items():
            kk = _space_offsets(acc, None)
            if kk is None or any(kk[1]):
                raise _Unrecognised("increment reads an adjoint wavefield off-centre")
            keyed[id(acc.function)][kk[0]] = coef
        saved = []
        for f in fields:
            if set(keyed[id(f)]) != {-1, 0, 1}:
                raise _Unrecognised(f"increment is not -({form})")
            funcs, consts, _ = self._leaves(keyed[id(f)].values())
            sv = [a for a in funcs if getattr(a.function, 'is_TimeFunction', False)]
            if len(sv) != 1 or len(funcs) != 1 or consts:
                raise _Unrecognised(f"each term of the increment must multiply {f.name}.dt2 by one saved wavefield")
            us = sv[0]
            ku = _space_offsets(us, None)
            if us.function.is_buffered or ku is None or ku[0] != 0 or any(ku[1]) or \
                    us.function.space_order != plan['u'].space_order:
                raise _Unrecognised("the forward wavefield must be saved (save=nt) and read at (time, x, y, z)")
            saved.append(us.function)
        if len({id(s) for s in saved}) != len(saved):
            raise _Unrecognised("the terms of the increment must use distinct saved wavefields")
        rng = np.random.default_rng(seed)
        dtname = plan['dt'].name
        for probe in range(2):
            # saved field i is drawn in [0.5 + 2i, 2 + 2i], so a term that multiplies the wrong field cannot match
            val = {id(s): rng.uniform(0.5 + 2 * i, 2.0 + 2 * i) for i, s in enumerate(saved)}
            dt = rng.uniform(0.5, 2.0)

            def leaf(n):
                if n.is_Access:
                    return val[id(n.function)]
                if n.name == dtname:
                    return dt
                raise _Unrecognised(f"unknown symbol {n.name} in the increment")
            for f, s in zip(fields, saved):
                c = {t: eval_scalar(e, leaf) for t, e in keyed[id(f)].items()}
                s_ = val[id(s)]
                want = {-1: -s_ / dt ** 2, 0: 2 * s_ / dt ** 2, 1: -s_ / dt ** 2}
                for t in want:
                    if abs(c[t] - want[t]) > 1e-9 * abs(want[t]):
                        raise _Unrecognised(f"increment is not -({form})")
        return saved

    # -- TTI -------------------------------------------------------------------------------------
    _TTI_PARAMS = ('vp', 'epsilon', 'delta', 'theta', 'phi')

    def _recognise_tti_adjoint(self, updates, injs, itps):
        """The reference's centred-TTI adjoint `AdjointTTI` (tti/operators.py `AdjointOperator`, `kernel_centered(...,
        forward=False)`): (p.backward, r.backward) from H0 = Gh(e2 p + sd r), Hz = Gzz(sd p + r), e2 and sd sampled at
        every tap point, with the backward damping; the receivers injected into both fields at the level written."""
        return self._recognise_tti(updates, injs, itps, adjoint=True)

    def _recognise_tti(self, updates, injs, itps, adjoint=False):
        (u, equ), (v, eqv) = updates
        grid = u.grid
        nd = grid.dim
        if nd not in (2, 3) or v.grid is not grid:
            raise _Unrecognised("TTI fast path needs a 2-D or 3-D grid shared by both fields")
        so = u.space_order
        if so != v.space_order or so % 4 or so // 2 > 8:
            raise _Unrecognised(f"TTI needs space_order multiple of 4 (got {so})")
        R = so // 2
        ku, kv = (self._taps(e.rhs, [u, v], ('u', 'v')) for e in (equ, eqv))
        funcs, consts, syms = self._leaves(list(ku.values()) + list(kv.values()))
        pnames = self._TTI_PARAMS
        byname = {c.name: c for c in consts if c.name in pnames}
        damp = None
        for a in funcs:
            f = a.function
            if getattr(f, 'is_TimeFunction', False):
                raise _Unrecognised("unexpected time-varying coefficient")
            if f.name in pnames:
                if f.space_order != so:
                    raise _Unrecognised("array-valued TTI parameters must share the wavefield's space_order")
                byname[f.name] = f
            elif damp is None or damp is f:
                damp = f
            else:
                raise _Unrecognised(f"unknown coefficient field {f.name}")
        if any(n not in byname for n in ('vp', 'epsilon', 'delta', 'theta')):
            raise _Unrecognised("TTI fast path needs vp/epsilon/delta/theta[/phi] (Constants or Functions)")
        if nd == 2 and 'phi' in byname:
            raise _Unrecognised("a 2-D TTI update has no azimuth phi")
        for n in (c for c in consts if c.name not in pnames):
            raise _Unrecognised(f"unknown Constant {n.name} in the TTI update")
        # every access of damp must be at the centre
        for ex in list(ku.values()) + list(kv.values()):
            for n in ex.preorder():
                if n.is_Access and n.function is damp:
                    k = _space_offsets(n, None)
                    if k is None or any(k[1]):
                        raise _Unrecognised("damp accessed off-centre")
        dtsym = grid.stepping_dim.spacing
        hs = self._spacing_values(grid)
        w2 = [second_derivative_weights(so, h) for h in hs]
        w1 = [half_node_first_derivative_weights(so, h) for h in hs]
        rng = np.random.default_rng(99)
        for probe in range(2):
            P, leaf, dt, dval, _ = self._tti_probe(rng, byname, damp, grid)
            pu, pv = predict_tti(w2, w1, R, P, dval, dt, adjoint=adjoint, nd=nd)
            for got, pred, nm in ((ku, pu, 'u'), (kv, pv, 'v')):
                keys = set(got) | set(pred)
                for k in keys:
                    g = eval_scalar(got[k], leaf) if k in got else 0.0
                    p = pred.get(k, 0.0)
                    if abs(g - p) > 1e-8 * max(1.0, abs(p)):
                        raise _Unrecognised(f"TTI coefficient mismatch in {nm} at {k}: {g} vs {p}")
        m_role = ('vp_f', byname['vp']) if isinstance(byname['vp'], Function) else ('vp_c', byname['vp'])
        plan = {'kind': 'tti', 'u': u, 'v': v, 'grid': grid, 'so': so, 'R': R, 'w2': w2, 'w1': w1,
                'consts': byname, 'damp': damp, 'dt': dtsym, 'src': None, 'rec': None, 'rec_toff': 0,
                'm_role': m_role, 'adjoint': adjoint}
        self._attach_sparse(plan, injs, itps, [u, v], funcs, consts, syms, plan['m_role'])
        return plan

    def _tti_probe(self, rng, byname, damp, grid, dm=None):
        """Values for one probe of the TTI recognisers. Each parameter gets a random value AND, if `byname` has it
        as a Function, a random spatial gradient, so that the comparison also checks WHERE each factor is sampled
        (the reference samples the rotation factors at the shifted points of the outer derivative,
        tti/operators.py:92-102). dt, then damp and (TTI Born) dm at the centre, are drawn after them.
        Returns `P(name, offset)`, `leaf`, dt and the values of damp (0 without it) and dm."""
        nd = grid.dim
        base = {n: rng.uniform(0.2, 0.8) for n in self._TTI_PARAMS}
        gradv = {n: (rng.uniform(-0.02, 0.02, size=nd) if isinstance(byname.get(n), Function) else np.zeros(nd))
                 for n in self._TTI_PARAMS}
        if 'phi' not in byname:
            base['phi'] = 0.0
        dt = rng.uniform(0.5, 2.0)
        dval = rng.uniform(0.5, 2.0) if damp is not None else 0.0
        dmv = rng.uniform(0.5, 2.0) if dm is not None else None
        spv = {sp.name: float(v) for sp, v in grid.spacing_map.items()}
        dtname = grid.stepping_dim.spacing.name

        def P(name, off):
            return float(base[name] + np.dot(gradv[name], off))

        def leaf(n):
            if n.is_Access:
                f = n.function
                if f is damp:
                    return dval
                if f is dm:
                    return dmv
                k = _space_offsets(n, None)
                if k is None:
                    raise _Unrecognised("non-affine parameter access")
                return P(f.name, k[1])
            if n.is_Constant:
                return P(n.name, (0,) * nd)
            if n.name == dtname:
                return dt
            if n.name in spv:
                return spv[n.name]
            raise _Unrecognised(f"unknown symbol {n.name}")
        return P, leaf, dt, dval, dmv

    def _recognise_tti_born(self, updates, injs, itps):
        """The reference's centred-TTI linearised-modelling operator `BornTTI` (examples/seismic/tti/operators.py:
        532-586): `kernel_centered(model, u0, v0)`, the source injected into (u0.forward, v0.forward),
        `kernel_centered(model, du, dv, qu=-dm*u0.dt2, qv=-dm*v0.dt2)`, the receivers sampling du + dv. The
        linearised equations must be the background ones applied to (du, dv) plus `-dm * u0.dt2` (du) and
        `-dm * v0.dt2` (dv) over the same denominator, with the same parameter objects."""
        fields = [f for f, _ in updates]

        def reads(eq):
            return {id(n.function) for n in eq.rhs.evaluate.preorder() if n.is_Access} & {id(f) for f in fields}
        rd = {id(f): reads(e) for f, e in updates}
        pairs = [(i, j) for i in range(4) for j in range(i + 1, 4)
                 if rd[id(fields[i])] | rd[id(fields[j])] <= {id(fields[i]), id(fields[j])}]
        if len(pairs) != 1:
            raise _Unrecognised("TTI Born: no unique background pair that reads no other field")
        bg = [updates[k] for k in pairs[0]]
        lin = [x for k, x in enumerate(updates) if k not in pairs[0]]
        plan = self._recognise_tti(bg, [], [])
        u0, v0 = plan['u'], plan['v']
        grid, so, damp, consts = plan['grid'], plan['so'], plan['damp'], plan['consts']
        for f, _ in lin:
            if f.grid is not grid or f.space_order != so:
                raise _Unrecognised("TTI Born: the linearised fields need the background grid and space order")
        ku0, kv0 = (self._taps(e.rhs, [u0, v0], (0, 1)) for _, e in bg)
        # split each linearised equation into taps on the linearised pair (tagged 'a', 'b') and on the background
        # pair (0, 1)
        (fa, ea), (fb, eb) = lin
        ta, tb = (self._taps(e.rhs, [fa, fb, u0, v0], ('a', 'b', 0, 1)) for e in (ea, eb))

        def split(keyed, du):
            own = {(int(k[0] != du),) + k[1:]: coef for k, coef in keyed.items() if k[0] in ('a', 'b')}
            ext = {k: coef for k, coef in keyed.items() if k[0] in (0, 1)}
            return own, ext
        # du is the field whose equation carries the background u0 taps; dv the v0 ones
        cand = []
        for du, dv, tdu, tdv, tag in ((fa, fb, ta, tb, 'a'), (fb, fa, tb, ta, 'b')):
            own_u, ext_u = split(tdu, tag)
            own_v, ext_v = split(tdv, tag)
            if set(own_u) == set(ku0) and set(own_v) == set(kv0):
                cand.append((du, dv, own_u, ext_u, own_v, ext_v))
        if not cand:
            raise _Unrecognised("TTI Born: the linearised pair is not updated with the background taps")
        allc = list(ku0.values()) + list(kv0.values())
        for c in cand[0][2:]:
            allc += list(c.values())
        funcs, csts, syms = self._leaves(allc)
        known = {id(c) for c in consts.values()}
        if damp is not None:
            known.add(id(damp))
        for cst in csts:
            if id(cst) not in known:
                raise _Unrecognised(f"TTI Born: Constant {cst.name} is not one of the background parameters")
        extra = {id(a.function): a.function for a in funcs if id(a.function) not in known}
        if len(extra) != 1:
            raise _Unrecognised("TTI Born: cannot identify the model perturbation dm (the linearised pair must use the "
                                "background parameters)")
        dm = next(iter(extra.values()))
        if getattr(dm, 'is_TimeFunction', False) or dm.name in self._TTI_PARAMS:
            raise _Unrecognised("TTI Born: cannot identify the model perturbation dm")
        for ex in allc:
            for n in ex.preorder():
                if n.is_Access and n.function is dm:
                    k = _space_offsets(n, None)
                    if k is None or any(k[1]):
                        raise _Unrecognised("dm accessed off-centre")
        zero = (0,) * grid.dim
        rng = np.random.default_rng(2718)
        errors = []
        for du, dv, own_u, ext_u, own_v, ext_v in cand:
            try:
                for probe in range(2):
                    P, leaf, dt, dval, dmv = self._tti_probe(rng, consts, damp, grid, dm)
                    for got, want in ((own_u, ku0), (own_v, kv0)):
                        for k, c in want.items():
                            w = eval_scalar(c, leaf)
                            if abs(eval_scalar(got[k], leaf) - w) > 1e-9 * max(1.0, abs(w)):
                                raise _Unrecognised(f"the linearised pair is not updated with the background stencil "
                                                    f"(tap {k})")
                    vp = P('vp', zero)
                    den = 1.0 / (vp * vp) / dt ** 2 + dval / dt
                    for ext, src in ((ext_u, 0), (ext_v, 1)):
                        want = {(src, 1, zero): -dmv / dt ** 2 / den, (src, 0, zero): 2 * dmv / dt ** 2 / den,
                                (src, -1, zero): -dmv / dt ** 2 / den}
                        if set(ext) != set(want):
                            raise _Unrecognised("the linearised pair is not driven by a centred u0.dt2 / v0.dt2 term")
                        for k, wv in want.items():
                            if abs(eval_scalar(ext[k], leaf) - wv) > 1e-9 * max(1.0, abs(wv)):
                                raise _Unrecognised("the source of the linearised pair is not -dm * u0.dt2 / "
                                                    "-dm * v0.dt2")
            except _Unrecognised as e:
                errors.append(str(e))
                continue
            fu, cu, su = self._leaves(ku0.values())
            self._attach_sparse(plan, injs, [], [u0, v0], fu, cu, su, plan['m_role'])
            self._attach_sparse(plan, [], itps, [du, dv], fu, cu, su, plan['m_role'])
            plan['born_du'], plan['born_dv'], plan['born_dm'] = du, dv, dm
            return plan
        raise _Unrecognised(f"TTI Born: {errors[0]}")

    # ------------------------------------------------------------------------------------------
    # introspection
    # ------------------------------------------------------------------------------------------
    def __str__(self):
        if self._plan is None:
            return (f"/* Operator `{self.name}`: NumPy interpreter ({len(self._items)} expressions)"
                    f"{' -- not recognised: ' + self._why_not if self._why_not else ''} */")
        p = self._plan
        if p['kind'] == 'linear':
            taps = ', '.join(f"f[t{t:+d}]{list(o)}" for t, o, _ in p['taps'])
            return (f"/* Operator `{self.name}` -> libb200stencil.so::b2_linear_forward (sm_90a)\n"
                    f"   {p['u'].name}[t{p['wshift']:+d}] = sum_k c_k * ({taps}) */")
        head = (f"/* Operator `{self.name}` -> libb200stencil.so::{self._entry.symbol} (sm_90a)\n"
                f"   space_order={p['so']} radius={p['R']} src={p['src'] and p['src'].name} "
                f"rec={p['rec'] and p['rec'].name} rec_toff={p['rec_toff']}"
                f"{' free_surface' if p.get('free_surface') else ''}{' OT4' if p.get('ot4') else ''} */\n")
        # like the reference, `str(op)` is C: here the adapter that `cinterface()` writes
        from . import cinterface as ci
        return head + ci.generate(p, self.name, distributed=p['grid'].distributor.is_parallel)[0]

    ccode = property(__str__)

    @property
    def cfunction(self):
        """The C-ABI entry point this operator calls (devito/operator/operator.py:857-869)."""
        if self._plan is None:
            raise InvalidOperator("interpreted operators have no C entry point")
        return getattr(L_.load_library(), self._entry.symbol if self._entry else 'b2_linear_forward')

    def cinterface(self, force=False):
        """Write `<name>.c` / `<name>.h` under the JIT directory and return `(ccode, hcode)`
        (devito/operator/operator.py:871-902). For an operator on the CUDA path the C file is the
        adapter exporting the reference-style symbol `int <name>(struct dataobj *..., ...)` on top of
        libb200stencil.so — see devito_b200/cinterface.py."""
        from . import cinterface as ci
        if self._plan is None or self._plan['kind'] == 'linear':
            raise InvalidOperator("no C adapter is generated for interpreted / generic-stencil operators")
        dist = self._plan['grid'].distributor.is_parallel
        ccode, hcode = ci.generate(self._plan, self.name, distributed=dist)
        dest = ci.jit_dir()
        for ext, code in (('.c', ccode), ('.h', hcode)):
            path = os.path.join(dest, self.name + ext)
            if force or not os.path.isfile(path):
                with open(path, 'w') as f:
                    f.write(code)
        return ccode, hcode

    @property
    def parameters(self):
        p = self._plan
        if p is None:
            return tuple(self._interp.functions.values())
        if p['kind'] == 'linear':
            cs = {id(n): n for _, _, c in p['taps'] for n in c.preorder() if n.is_Constant}
            return (p['u'],) + tuple(cs.values())
        out = [s.obj for s in self._entry.arrays] + [prm.obj for prm in self._entry.params] + [p['src'], p['rec']]
        return tuple(o for o in out if o is not None)

    # ------------------------------------------------------------------------------------------
    # execution
    # ------------------------------------------------------------------------------------------
    def __call__(self, **kwargs):
        return self.apply(**kwargs)

    def apply(self, **kwargs):
        if self._plan is None:
            return self._apply_interp(**kwargs)
        if self._plan['kind'] == 'linear':
            return self._apply_linear(**kwargs)
        return self._apply_wave(**kwargs)

    def arguments(self, **kwargs):
        if self._plan is None:
            return self._interp_args(dict(kwargs))
        if self._plan['kind'] == 'linear':
            return self._prepare_linear(dict(kwargs))
        return self._prepare(dict(kwargs))[0]

    _prepare_arguments = arguments

    # -- generic -----------------------------------------------------------------------------------
    _ignored_kwargs = ('autotune', 'nthreads', 'nthreads_nonaffine', 'deviceid', 'devicerm',
                       'resident', 'kernel', 'errctl')

    def _interp_args(self, kwargs):
        it = self._interp
        fns = it.functions
        scalars = {}
        bounds = {}
        grid = next((f.grid for f in fns.values() if f.grid is not None), None)
        if grid is not None:
            for sp, v in grid.spacing_map.items():
                scalars[sp.name] = float(kwargs.pop(sp.name, v))
            for d, n in zip(grid.dimensions, grid.shape):
                lo = kwargs.pop(d.min_name, 0)
                hi = kwargs.pop(d.max_name, n - 1)
                bounds[d.name] = (lo, hi)
                scalars[d.min_name] = lo
                scalars[d.max_name] = hi
                scalars[f'{d.name}_size'] = n
        if 'dt' in kwargs:
            scalars['dt'] = float(kwargs.pop('dt'))
        # Constants by name
        for kind, _, obj, lhs, rhs in it.items:
            exprs = [rhs] if kind == 'eq' else (list(obj.exprs) if kind == 'inject' else [obj.expr])
            for ex in exprs:
                for n in ex.preorder():
                    if n.is_Constant and n.name in kwargs:
                        scalars[n.name] = float(kwargs.pop(n.name))
        # time range
        tlo, thi = it.time_shifts()
        sized = [f for f in fns.values() if (getattr(f, 'is_SparseTimeFunction', False))
                 or (getattr(f, 'is_TimeFunction', False) and not f.is_buffered)]
        time_m = kwargs.pop('time_m', None)
        time_M = kwargs.pop('time_M', kwargs.pop('time', kwargs.pop('t', None)))
        if it.has_time:
            if time_m is None:
                time_m = -min(tlo, 0)
            if time_M is None:
                if not sized:
                    raise InvalidArgument("No value found for parameter time_M")
                # a snapshot on a ConditionalDimension(factor=n) bounds time by time_size * n
                nt = min(f.nt if getattr(f, 'is_SparseTimeFunction', False) else
                         f.time_size * (_subsampled(f) or 1) for f in sized)
                time_M = nt - 1 - max(thi, 0)
        else:
            time_m, time_M = 0, 0
        for k in list(kwargs):
            if k in self._ignored_kwargs or k in fns:
                kwargs.pop(k)
        if kwargs and not configuration['ignore-unknowns']:
            raise InvalidArgument(f"Unrecognized argument(s) {sorted(kwargs)} in kwargs")
        return {'time_m': time_m, 'time_M': time_M, 'scalars': scalars, 'bounds': bounds}

    def _apply_interp(self, **kwargs):
        args = self._interp_args(dict(kwargs))
        t0 = _time.perf_counter()
        self._interp.run(args['time_m'], args['time_M'], args['scalars'], args['bounds'])
        el = _time.perf_counter() - t0
        summary = PerformanceSummary()
        summary['section0'] = PerfEntry(el)
        summary.globals['fdlike'] = PerfEntry(el)
        return summary

    # -- CUDA path ---------------------------------------------------------------------------------
    def _resolve(self, kwargs, obj, post=None):
        """User override by name, else the default object. Like the reference
        (devito/types/dense.py:913-926) an override is either an object of the same kind or a bare
        ndarray standing in for the function's allocated data (halo included): the array is then
        used in place — uploaded before the time loop, written back when the call returns."""
        if obj is None:
            return None
        v = kwargs.pop(obj.name, None)
        if v is None:
            return obj
        if isinstance(v, np.ndarray):
            return self._shadow(obj, v, post)
        if isinstance(v, L_.ForeignDataobj):
            return self._foreign(obj, v)
        return v

    @staticmethod
    def _foreign(obj, fo):
        """A `struct dataobj` built by the caller (devito_b200/refplugin.py passes the reference's own)
        stands in for `obj`'s data; the library stages it in and out inside the call."""
        want = tuple(obj.storage.shape)
        got = fo.shape(len(want))
        if got != want:
            raise InvalidArgument(f"Shape {got} of runtime value `{obj.name}` does not match the allocated "
                                  f"shape {want}")
        if fo.obj.dmap or not fo.obj.data:
            raise InvalidArgument(f"runtime struct for `{obj.name}` must describe a host array")
        sh = object.__new__(type(obj))
        sh.__dict__.update(obj.__dict__)
        sh._foreign_obj = fo
        return sh

    @staticmethod
    def _shadow(obj, arr, post):
        from .types import FieldStorage
        want = tuple(obj.storage.shape)
        if tuple(arr.shape) != want:
            raise InvalidArgument(f"Shape {arr.shape} of runtime value `{obj.name}` does not match "
                                  f"the allocated shape {want}")
        if arr.dtype != np.float32 or not arr.flags['C_CONTIGUOUS'] or not arr.flags['WRITEABLE']:
            raise InvalidArgument(f"runtime value `{obj.name}` must be a writeable C-contiguous float32 array")
        sh = object.__new__(type(obj))
        sh.__dict__.update(obj.__dict__)
        st = FieldStorage(want, np.float32)
        st._host = arr
        sh._storage = st
        if post is not None:
            def writeback():
                if not st.host_valid:
                    st.sync_to_host()
                st.dev = None
                st.dev_valid = False
            post.append(writeback)
        return sh

    @staticmethod
    def _override_ok(check, f, so, grid):
        """Whether `f` is what the kernel reads in a slot of this `check` (see `_OVERRIDE_KINDS`)."""
        if np.dtype(f.dtype) != np.float32:
            return False
        if check == 'function':
            return isinstance(f, Function)
        if not isinstance(f, TimeFunction):
            return False
        if check == 'wavefield':
            return f.space_order == so and f.grid.shape == grid.shape
        if check == 'saved':
            return not f.is_buffered and f.space_order == so
        return not f.is_buffered and f.grid.shape == grid.shape

    def _resolve_param(self, kwargs, prm, so):
        """A Function (passed as an array) or a float: the override by name of `prm.obj`, else `prm.obj`
        itself. Without `prm.switch` the override keeps the kind the Operator was built with."""
        obj = prm.obj
        if obj is None:
            return prm.unit
        val = kwargs.pop(obj.name, obj)
        if isinstance(obj, Function):
            if isinstance(val, L_.ForeignDataobj):
                val = self._foreign(obj, val)
            elif isinstance(val, np.ndarray) and val.ndim:
                val = self._shadow(obj, val, None)
        if not prm.switch:
            if isinstance(obj, Function) and (not isinstance(val, Function) or val.space_order != so):
                raise InvalidArgument(f"`{obj.name}` must be overridden by a Function of the same space_order")
            if not isinstance(obj, Function) and isinstance(val, Function):
                raise InvalidArgument(f"array-valued `{obj.name}` needs an Operator built with a Function")
        if isinstance(val, Function):
            if np.dtype(val.dtype) != np.float32:
                raise InvalidArgument(f"the override of `{obj.name}` must be a float32 Function")
            return val
        if isinstance(val, np.ndarray) and val.ndim:
            raise InvalidArgument(f"an array `{obj.name}` must have the allocated shape of a Function")
        return float(val.data if isinstance(val, Constant) else val)

    def _prepare(self, kwargs, omit=()):
        p, entry = self._plan, self._entry
        grid = p['grid']
        args = OrderedDict()
        hold = []          # keep ctypes/ndarray objects alive during the call
        post = args['post'] = []     # run after the C call (write-back of ndarray overrides)
        for s in entry.arrays:
            if s.member in omit:
                continue
            f = args[s.member] = self._resolve(kwargs, s.obj, post)
            if not self._override_ok(s.check, f, p['so'], grid):
                raise InvalidArgument(f"the override of `{s.obj.name}` must be {_OVERRIDE_KINDS[s.check]}")
        args['fields'] = [args[m] for m in ('u', 'v') if m in args]
        if grid.distributor.is_parallel:
            if p['kind'] in ('sa', 'visco'):
                name = {'sa': "self-adjoint", 'visco': "SLS viscoacoustic"}[p['kind']]
                raise InvalidArgument(f"the {name} update does not run on a decomposed grid in this version")
            if p['kind'] == 'tti' and grid.dim == 2:
                raise InvalidArgument("2-D TTI modelling does not run on a decomposed grid in this version")
            if p['kind'] == 'tti' and p.get('adjoint'):
                raise InvalidArgument("the TTI adjoint does not run on a decomposed grid in this version")
            if 'born_du' in args:
                raise InvalidArgument("TTI Born modelling does not run on a decomposed grid in this version")
        args['params'] = [self._resolve_param(kwargs, prm, p['so']) for prm in entry.params]
        # spacing / dt
        dt = kwargs.pop('dt', None)
        if dt is None:
            raise InvalidArgument("No value found for parameter dt")
        args['dt'] = float(np.float32(dt))
        for sp in grid.spacing_symbols:
            if sp.name in kwargs:
                hv = kwargs.pop(sp.name)
                cur = self._spacing_values(grid)[grid.spacing_symbols.index(sp)]
                if abs(float(hv) - cur) > 1e-6 * abs(cur):
                    raise InvalidArgument(f"runtime override of {sp.name} is not supported by the "
                                          "pre-built kernels; rebuild the Operator")
        # bounds
        lo, hi = [], []
        for d, n in zip(grid.dimensions, grid.shape):
            a = kwargs.pop(d.min_name, 0)
            b = kwargs.pop(d.max_name, n - 1)
            if a < 0 or b > n - 1:
                raise InvalidArgument(f"OOB detected due to {d.min_name}={a}, {d.max_name}={b}")
            lo.append(int(a))
            hi.append(int(b))
        args['lo'], args['hi'] = lo, hi
        if p.get('ot4') and (p.get('free_surface') or p.get('grad') is not None):
            raise InvalidArgument("the OT4 kernel is not yet combined with a free surface or the imaging condition")
        if p.get('free_surface') and lo[-1] != 0:
            raise InvalidArgument("a free-surface operator must iterate from the surface row (lower bound 0 "
                                  "on the last dimension)")
        # sparse
        src = self._resolve(kwargs, p['src'], post)
        rec = self._resolve(kwargs, p['rec'], post)
        for sf in (src, rec):
            # a caller-built sparse table (is_foreign) carries its own float32 arrays
            if sf is not None and not getattr(sf, 'is_foreign', False) and \
                    (np.dtype(sf.dtype) != np.float32 or np.dtype(sf.coordinates_data.dtype) != np.float32):
                raise InvalidArgument(f"the override of `{sf.name}` must be a float32 SparseTimeFunction "
                                      "(traces and coordinates)")
        args['src'], args['rec'] = src, rec
        # time range (devito/types/dimension.py:279-331)
        sized = [s for s in (src, rec) if s is not None]
        sized += [f for f in args['fields'] if not f.is_buffered]
        sized += [args[s.member] for s in entry.arrays if s.check == 'saved' and s.member not in omit]
        time_m = kwargs.pop('time_m', None)
        time_M = kwargs.pop('time_M', kwargs.pop('time', None))
        if time_m is None:
            time_m = 1           # u[t-1] is read: lower offset -1
        if time_M is None:
            cands = [(s.nt if getattr(s, 'is_SparseTimeFunction', False) else s.time_size) - 2 for s in sized]
            if args.get('snap') is not None:
                # the sub-sampled dimension bounds its parent: time / factor < nsnaps
                cands.append(args['snap'].time_size * p['snap_factor'] - 1)
            if not cands:
                raise InvalidArgument("No value found for parameter time_M")
            time_M = min(cands)      # u[t+1] is written: upper offset +1
        for s in sized:
            n = s.nt if getattr(s, 'is_SparseTimeFunction', False) else s.time_size - 1
            if time_M >= n or time_m < 0:
                raise InvalidArgument(f"OOB detected due to time_M={time_M}")
        if args.get('snap') is not None:
            need = int(time_M) // p['snap_factor'] + 1
            if need > args['snap'].time_size:
                raise InvalidArgument(f"OOB detected due to time_M={time_M}: {need} snapshots needed, "
                                      f"`{args['snap'].name}` holds {args['snap'].time_size}")
        args['time_m'], args['time_M'] = int(time_m), int(time_M)
        args['resident'] = bool(kwargs.pop('resident', True)) and not bool(kwargs.pop('devicerm', 0))
        args['kernel'] = int(kwargs.pop('kernel', 0))
        args['errctl'] = int(kwargs.pop('errctl', 1 if configuration.get('errctl') == 'max' else 0))
        args['deviceid'] = kwargs.pop('deviceid', None)
        for k in ('autotune', 'nthreads', 'nthreads_nonaffine'):
            kwargs.pop(k, None)
        if kwargs and not configuration['ignore-unknowns']:
            raise InvalidArgument(f"Unrecognized argument(s) {sorted(kwargs)} in kwargs")
        return args, hold

    def _device(self, args):
        import torch
        dev = args.get('deviceid')
        if dev is None or dev < 0:
            dev = configuration['deviceid']
        if dev is None or dev < 0:
            dev = torch.cuda.current_device() if torch.cuda.is_available() else 0
        return int(dev)

    @staticmethod
    def _as_layout(fn, so):
        """Host array of a parameter Function defined with another space_order, re-padded to the
        allocated layout of the wavefield (halo `so`)."""
        src = fn.data_ro_with_halo
        h = fn.space_order
        dom = src[tuple(slice(h, src.shape[i] - h) for i in range(src.ndim))]
        if h >= so:
            d = h - so
            return np.ascontiguousarray(src[tuple(slice(d, src.shape[i] - d) for i in range(src.ndim))])
        out = np.pad(dom, so, mode='edge')
        inner = tuple(slice(so - h, out.shape[i] - (so - h)) for i in range(out.ndim))
        out[inner] = src
        return np.ascontiguousarray(out)

    def _field_obj(self, fn, dev, resident, hold, so=None, written=False, host_io_ok=False, post=None):
        """(b2_dataobj for a dense function: resident (dmap set) or host-staged, whether it is host-staged
        through the caller's device buffer (host_io)). A resident array the call writes is marked written by a hook
        appended to `post`, run once the call has returned, so that a view the caller keeps sees what it wrote."""
        import torch
        fo = getattr(fn, '_foreign_obj', None)
        if fo is not None:
            if so is not None and fn.space_order != so:
                raise InvalidArgument(f"`{fn.name}`: a caller-built struct needs the wavefield's space order {so}")
            if resident:
                raise InvalidArgument("caller-built structs are host arrays: apply with resident=False")
            hold.append(fo)
            return fo, False
        if so is not None and fn.space_order != so:
            host = self._as_layout(fn, so)
            hold.append(host)
            halo = tuple((0, 0) if d.is_Time else (so, so) for d in fn.dimensions)
            if resident:
                t = torch.from_numpy(host).to(f'cuda:{dev}')
                hold.append(t)
                ob = L_.make_dataobj(host=host, dev_ptr=t.data_ptr(), halo=halo)
            else:
                ob = L_.make_dataobj(host=host, halo=halo)
            hold.append(ob)
            return ob, False
        st = fn.storage
        host_io = False
        if resident:
            dist_ = fn.grid.distributor if fn.grid is not None else None
            p2p_field = (written and dist_ is not None and dist_.is_parallel and distributed.p2p_enabled()
                         and getattr(fn, 'is_TimeFunction', False) and getattr(fn, 'is_buffered', False))
            if p2p_field:
                st.raw = True        # plain cudaMalloc: exportable through CUDA IPC
            t = st.to_device(torch.device('cuda', dev))
            if p2p_field and not st.p2p_registered:
                distributed.register_field(st, fn.grid, dev)
            ob = L_.make_dataobj(dev_ptr=t.data_ptr(), shape=st.shape, halo=fn.halo)
            if written:
                post.append(st.mark_device_written)
        else:
            host = st.host if written else st.host_ro
            dist_ = fn.grid.distributor if fn.grid is not None else None
            if (host_io_ok and dist_ is not None and dist_.is_parallel and distributed.p2p_enabled()
                    and (getattr(fn, 'is_buffered', False) or not getattr(fn, 'is_TimeFunction', False))):
                # host-staged apply under decomposition: the library moves host <-> device itself (host_io), through
                # a device buffer that stays registered with the neighbour ranks (peer-memory halo path)
                import torch
                if getattr(fn, 'is_TimeFunction', False):
                    st.raw = True
                t = st.device_scratch(torch.device('cuda', dev))
                if getattr(fn, 'is_TimeFunction', False) and not st.p2p_registered:
                    distributed.register_field(st, fn.grid, dev)
                ob = L_.make_dataobj(host=host, dev_ptr=t.data_ptr(), halo=fn.halo)
                host_io = True
            else:
                ob = L_.make_dataobj(host=host, halo=fn.halo)
        hold.append(ob)
        return ob, host_io

    def _sparse_obj(self, sf, grid, hold, written=False, post=None, trange=None):
        """b2_sparse for a SparseTimeFunction. Under x-slab decomposition every rank holds all
        points (positions are made relative to the local slab; the kernels' bound guards drop
        what lies outside). A *written* function (receivers) is evaluated only for the points
        whose base cell this rank owns and merged with an all-reduce afterwards — the reference
        scatters points to their owner ranks instead (devito/types/sparse.py:608-730)."""
        if sf is None:
            return None
        if getattr(sf, 'is_foreign', False):
            if grid.distributor.is_parallel:
                raise InvalidArgument("caller-built sparse tables are not combined with domain decomposition")
            s = L_.Sparse()
            s.data, s.gp = sf.data.ptr, sf.gp.ptr
            for i, wo in enumerate(sf.ws):
                s.w[i] = wo.ptr
            s.p_m, s.p_M, s.r = sf.p_m, sf.p_M, sf.r
            hold.extend([sf, s])
            return s
        gp, ws = sf.tabulate()
        dist = grid.distributor
        host = sf.storage.host if written else sf.storage.host_ro
        if dist.is_parallel:
            off = dist.offsets
            gp = np.ascontiguousarray((gp - np.asarray(off, dtype=np.int32)[None, :]).astype(np.int32))
            nloc = grid.shape[0]
            if not written:
                # scatter (devito/types/sparse.py:608-730 routes every point to the ranks its support touches):
                # this rank keeps only the points whose (2r)-wide support reaches its own cells; the kernel's
                # guards then deposit into the owned cells only
                r_ = int(sf.r)
                keep = np.nonzero((gp[:, 0] + r_ >= 0) & (gp[:, 0] - r_ + 1 <= nloc - 1))[0]
                if len(keep) == 0:
                    return None
                if len(keep) < gp.shape[0]:
                    gp = np.ascontiguousarray(gp[keep])
                    ws = [np.ascontiguousarray(w[keep]) for w in ws]
                    host = np.ascontiguousarray(host[:, keep])
            if written:
                # a point is evaluated by the rank that owns its base cell (the physical boundary ranks also own
                # what lies beyond the domain on their side)
                lo_ok = (gp[:, 0] >= 0) | dist.is_boundary_left
                hi_ok = (gp[:, 0] < nloc) | dist.is_boundary_right
                mask = lo_ok & hi_ok
                idx = np.nonzero(mask)[0]
                gp = np.ascontiguousarray(gp[idx])
                ws = [np.ascontiguousarray(w[idx]) for w in ws]
                # start from the caller's traces: rows outside [time_m, time_M] are not this call's to touch
                # (restart over time sub-ranges keeps what earlier calls recorded, like the reference)
                local = np.ascontiguousarray(host[:, idx])
                full = host
                t_lo, t_hi = trange if trange is not None else (0, host.shape[0] - 1)
                t_lo, t_hi = max(0, t_lo), min(host.shape[0] - 1, t_hi)

                def merge():
                    import torch
                    import torch.distributed as tdist
                    blk = np.zeros((t_hi - t_lo + 1, full.shape[1]), dtype=full.dtype)
                    blk[:, idx] = local[t_lo:t_hi + 1]
                    t = torch.from_numpy(blk)
                    if tdist.get_backend() == 'nccl':
                        tg = t.cuda()
                        tdist.all_reduce(tg)
                        t.copy_(tg.cpu())
                    else:
                        tdist.all_reduce(t)
                    full[t_lo:t_hi + 1] = blk
                if post is not None:
                    post.append(merge)
                host = local
                if len(idx) == 0:
                    return None
        data = L_.make_dataobj(host=host)
        gpo = L_.make_dataobj(host=gp)
        wos = [L_.make_dataobj(host=w) for w in ws]
        s = L_.Sparse()
        s.data = data.ptr
        s.gp = gpo.ptr
        for i, wo in enumerate(wos):
            s.w[i] = wo.ptr
        s.p_m, s.p_M = 0, host.shape[1] - 1
        s.r = sf.r
        hold.extend([gp, ws, data, gpo, wos, s, host])
        return s

    def _call(self, L, symbol, a, args, dev, post=()):
        """Run entry point `symbol` on the filled argument block `a`, then the post-call hooks."""
        a.deviceid = dev
        timers = L_.Profiler()
        a.timers = ctypes.pointer(timers)
        t0 = _time.perf_counter()
        rc = getattr(L, symbol)(ctypes.byref(a))
        t_wall = _time.perf_counter() - t0
        for fn in list(post) + args['post']:
            fn()
        return self._finish(rc, L, timers, args, t_wall)

    def _finish(self, rc, L, timers, args, t_wall):
        if rc != 0:
            msg = L.b2_last_error().decode()
            if rc == 100:
                raise ExecutionError(f"Operator `{self.name}`: NaN/Inf detected ({msg})")
            raise ExecutionError(f"Operator `{self.name}` failed with code {rc}: {msg}")
        nsteps = args['time_M'] - args['time_m'] + 1
        pts = float(np.prod([h - l + 1 for l, h in zip(args['lo'], args['hi'])])) * nsteps
        summary = PerformanceSummary()
        tot = timers.section0 + timers.section1 + timers.section2
        ops, bpp = self._flops_and_bytes_per_point()
        for nm in ('section0', 'section1', 'section2'):
            t = getattr(timers, nm)
            main = t > 0 and nm == 'section0'
            summary[nm] = PerfEntry(t, gpointss=(pts / t / 1e9 if main else None),
                                    gflopss=(ops * pts / t / 1e9 if main else None),
                                    oi=(ops / bpp if main else None), ops=(ops if main else None))
        summary.globals['fdlike'] = PerfEntry(t_wall, gpointss=pts / t_wall / 1e9 if t_wall > 0 else None)
        summary.globals['fdlike-nosetup'] = PerfEntry(tot, gpointss=pts / tot / 1e9 if tot > 0 else None)
        perf(f"Operator `{self.name}` ran in {t_wall:.4f} s [{pts / max(tot, 1e-12) / 1e9:.2f} GPts/s on device]")
        self._profiler_last = summary
        return summary

    def _flops_and_bytes_per_point(self):
        """Floating-point operations the CUDA kernels execute per grid point and time step (counted on
        the kernels' own formulas, a multiply-add = 2) and the algorithmic HBM bytes per point (SURVEY
        §8d) — what the reference reports as `gflopss` / `oi` from its own op count
        (devito/operator/profiling.py:344-430)."""
        p = self._plan
        if p['kind'] == 'linear':
            return float(2 * len(p['taps'])), 4.0 * (len({t for t, _, _ in p['taps']}) + 1)
        R, nd = p['R'], p['grid'].dim
        if p['kind'] in ('sa', 'visco'):
            # the nested operator: per axis 2R fluxes of R multiply-adds and a multiply, then R outer multiply-adds
            lap = nd * (2 * R * (2 * R + 1) + 2 * R)
            if p['kind'] == 'sa':
                return float(lap + 6), 24.0                 # the update 6
            # the epilogue of b2_visco_point.cuh 16 (forward) or the mix 8 and the update 6 (adjoint); bytes of
            # DESIGN §3.3k
            return (float(lap + 14), 64.0) if p.get('adjoint') else (float(lap + 16), 44.0)
        star = 1 + nd * R * 3                       # centre mul + per tap pair: add, multiply-add
        if p['kind'] == 'iso':
            arr = p['m_role'][0].endswith('_f')
            ops = star + 8
            bpp = 20.0 if arr else 16.0
            if p.get('ot4'):
                ops += 2 * star + 3
                bpp += 8.0
            return float(ops), bpp
        arr = any(hasattr(c, 'space_order') for c in p['consts'].values())
        ops = star + 2 * (6 * R + 5) + 2 * (6 * R + 3) + 16
        return float(ops), (48.0 if arr else 28.0)

    def _w_arrays(self, wlists, hold):
        arr = (ctypes.POINTER(ctypes.c_float) * 3)()
        for i, w in enumerate(wlists):
            a = np.ascontiguousarray(np.asarray(w, dtype=np.float32))
            hold.append(a)
            arr[i] = a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
        return arr

    def _apply_wave(self, **kwargs):
        L = L_.lib()
        hold = []          # alive until the call returns
        a, args, dev, post = self._marshal_wave(kwargs, hold)
        return self._call(L, self._entry.symbol, a, args, dev, post)

    def _marshal_wave(self, kwargs, hold, omit=()):
        """The entry point's argument block for an apply with `kwargs`: (block, prepared arguments, device, post-call
        hooks). `hold` keeps what the block points into alive; the array members in `omit` are left NULL."""
        args, held = self._prepare(dict(kwargs), omit)
        hold.extend(held)
        p, entry = self._plan, self._entry
        grid = p['grid']
        dev = self._device(args)
        res = args['resident']
        a = entry.struct()
        for k, v in entry.flags.items():
            setattr(a, k, v)
        for member, w in entry.weights:
            setattr(a, member, self._w_arrays(w, hold))
        host_io = False
        post = []
        for s in entry.arrays:
            if s.member in omit:
                continue
            ob, hio = self._field_obj(args[s.member], dev, res, hold, so=p['so'] if s.layout else None,
                                      written=s.written, host_io_ok=s.member in entry.host_io, post=post)
            setattr(a, s.member, ob.ptr)
            host_io |= hio
        for prm, val in zip(entry.params, args['params']):
            if isinstance(val, Function):
                ob, hio = self._field_obj(val, dev, res, hold, so=p['so'], host_io_ok=prm.member in entry.host_io)
                setattr(a, prm.member, ob.ptr)
                setattr(a, prm.scalar, prm.unit)
                host_io |= hio
            else:
                setattr(a, prm.scalar, 1.0 / np.sqrt(val) if prm.slowness else val)
            if prm.member == 'param':
                a.param_kind = (B2_PARAM_SCALAR if not isinstance(val, Function) else
                                B2_PARAM_M if prm.slowness else B2_PARAM_VP)
        if entry.host_io:
            a.host_io = int(host_io)
        a.dt = args['dt']
        for ax, lo, hi in zip('xyz', args['lo'], args['hi']):
            setattr(a, ax + '_m', lo)
            setattr(a, ax + '_M', hi)
        a.time_m, a.time_M = args['time_m'], args['time_M']
        s = self._sparse_obj(args['src'], grid, hold)
        r = self._sparse_obj(args['rec'], grid, hold, written=True, post=post,
                             trange=(args['time_m'], args['time_M']))
        a.src = ctypes.pointer(s) if s is not None else None
        a.rec = ctypes.pointer(r) if r is not None else None
        a.errctl = args['errctl']
        a.kernel = args['kernel']
        if grid.distributor.is_parallel:
            a.halo = distributed.halo_context(dev)
        if p.get('inject_literal'):
            # injection used a literal dt**2 (not the `dt` symbol): it must agree with runtime dt
            if abs(p['inject_dt2'] - a.dt * a.dt) > 1e-5 * p['inject_dt2']:
                raise InvalidArgument("literal dt in the injected expression differs from runtime dt")
        return a, args, dev, post

    # -- generic constant-coefficient update ------------------------------------------------------
    def _prepare_linear(self, kwargs):
        p = self._plan
        grid, f0 = p['grid'], p['u']
        args = OrderedDict()
        post = args['post'] = []
        f = self._resolve(kwargs, f0, post)
        if not isinstance(f, TimeFunction) or f.space_order != f0.space_order or f.grid.shape != grid.shape \
                or f.time_size != f0.time_size:
            raise InvalidArgument("incompatible override for the updated field")
        if np.dtype(f.dtype) != np.float32:
            raise InvalidArgument(f"the override of `{f0.name}` must be a float32 TimeFunction")
        args['fields'] = [f]
        # scalar environment of the coefficients: spacings, dt, Constants (overridable by name)
        env = {sp.name: float(v) for sp, v in grid.spacing_map.items()}
        for sp in grid.spacing_symbols:
            if sp.name in kwargs:
                env[sp.name] = float(kwargs.pop(sp.name))
        need_dt = any(n.is_Symbol and n.name == p['dt'].name for _, _, c in p['taps'] for n in c.preorder())
        if 'dt' in kwargs:
            env[p['dt'].name] = float(np.float32(kwargs.pop('dt')))
        elif need_dt:
            raise InvalidArgument("No value found for parameter dt")
        # a Constant may appear in many taps: resolve each one (and its override) once
        nodes = {id(n): n for _, _, c in p['taps'] for n in c.preorder() if n.is_Constant}
        over = {n.name: kwargs.pop(n.name) for n in nodes.values() if n.name in kwargs}
        consts = {}
        for k, n in nodes.items():
            v = over.get(n.name, n)
            consts[k] = float(v.data if isinstance(v, Constant) else v)

        def leaf(n):
            if n.is_Constant:
                return consts[id(n)]
            if n.name in env:
                return env[n.name]
            raise InvalidArgument(f"No value found for parameter {n.name}")
        args['taps'] = [(t, o, float(np.float32(eval_scalar(c, leaf)))) for t, o, c in p['taps']]
        lo, hi = [], []
        for d, n, (bl, bh) in zip(grid.dimensions, grid.shape, p['box']):
            a = kwargs.pop(d.min_name, None)
            b = kwargs.pop(d.max_name, None)
            a = bl if a is None else a
            b = bh if b is None else b
            if a < 0 or b > n - 1:
                raise InvalidArgument(f"OOB detected due to {d.min_name}={a}, {d.max_name}={b}")
            lo.append(int(a))
            hi.append(int(b))
        args['lo'], args['hi'] = lo, hi
        time_m = kwargs.pop('time_m', None)
        time_M = kwargs.pop('time_M', kwargs.pop('time', kwargs.pop(grid.stepping_dim.name, None)))
        if time_m is None:
            time_m = -p['tlo']
        if time_M is None:
            raise InvalidArgument("No value found for parameter time_M")
        if time_m < 0:
            raise InvalidArgument(f"OOB detected due to time_m={time_m}")
        args['time_m'], args['time_M'] = int(time_m), int(time_M)
        args['resident'] = bool(kwargs.pop('resident', True)) and not bool(kwargs.pop('devicerm', 0))
        args['deviceid'] = kwargs.pop('deviceid', None)
        for k in ('autotune', 'nthreads', 'nthreads_nonaffine', 'kernel', 'errctl'):
            kwargs.pop(k, None)
        if kwargs and not configuration['ignore-unknowns']:
            raise InvalidArgument(f"Unrecognized argument(s) {sorted(kwargs)} in kwargs")
        return args

    def _apply_linear(self, **kwargs):
        L = L_.lib()
        args = self._prepare_linear(dict(kwargs))
        p = self._plan
        grid = p['grid']
        nd = grid.dim
        dev = self._device(args)
        hold = []
        a = L_.LinearArgs()
        a.ndim = nd
        post = []
        a.f = self._field_obj(args['fields'][0], dev, args['resident'], hold, written=True, post=post)[0].ptr
        a.halo = p['so']
        taps = (L_.Tap * len(args['taps']))()
        for i, (t, o, c) in enumerate(args['taps']):
            taps[i].tshift = int(t)
            for d in range(nd):
                taps[i].off[d] = int(o[d])
            taps[i].coef = c
        a.ntaps = len(args['taps'])
        a.taps = taps
        a.wshift = p['wshift']
        lo, hi = args['lo'] + [0] * (3 - nd), args['hi'] + [0] * (3 - nd)
        a.x_m, a.x_M, a.y_m, a.y_M, a.z_m, a.z_M = lo[0], hi[0], lo[1], hi[1], lo[2], hi[2]
        a.time_m, a.time_M = args['time_m'], args['time_M']
        return self._call(L, 'b2_linear_forward', a, args, dev, post)


# ---------------------------------------------------------------------------------------------
# the stencil the self-adjoint kernels implement, as linear coefficients (float64) — used only by the recogniser
# ---------------------------------------------------------------------------------------------
def predict_sa(c, R, nd, bval, vp, w, dt, dirn):
    """{(time_shift, offsets): coefficient} of u_next = C sum_d sum_k c_k (F_d(p+(k-1)) - F_d(p-k)) + (2 - dt w) u
    + (dt w - 1) u_prev, F_d(q) = b(q) sum_i c_i (u(q+i) - u(q-i+1)), C = dt^2 vp^2 / b(p). `bval(offset)` is b at
    that offset from the output point; vp and w are their values at the output point."""
    zero = (0,) * nd
    C = dt * dt * vp * vp / bval(zero)
    out = {(0, zero): 2.0 - dt * w, (-dirn, zero): dt * w - 1.0}
    for off, v in nested_taps(c, R, nd, bval).items():
        out[(0, off)] = out.get((0, off), 0.0) + C * v
    return out


# ---------------------------------------------------------------------------------------------
# the SLS viscoacoustic pair as linear coefficients (float64) — used only by the recogniser
# ---------------------------------------------------------------------------------------------
def nested_taps(c, R, nd, bval):
    """{offset: coefficient} of L(f) = sum_d sum_k c_k (F_d(p+(k-1)) - F_d(p-k)), F_d(q) = b(q) sum_i c_i (f(q+i) -
    f(q-i+1)) at the output point; `bval(offset)` is b at that offset from it."""
    out = {}

    def unit(d, o):
        e = [0] * nd
        e[d] = o
        return tuple(e)
    for d in range(nd):
        for j in range(-R, R):
            a = c[d][j] if j >= 0 else -c[d][-j - 1]
            bq = bval(unit(d, j))
            for i in range(1, R + 1):
                for m, sgn in ((j + i, 1.0), (j - i + 1, -1.0)):
                    key = unit(d, m)
                    out[key] = out.get(key, 0.0) + a * bq * sgn * c[d][i - 1]
    return out


def predict_visco(c, R, nd, bval, vpval, qpval, dval, f0, dt, dirn):
    """({(field, time_shift, offsets): coefficient} of the memory-variable update, ... of the pressure update) of the
    reference's sls_2nd_order (tests/visco_ref.py states the scheme). The parameters are callables of the offset from
    the output point; the adjoint applies L to (1+tt) rho p and rho r[t-1], so there tt and rho are taken at the
    nodes."""
    zero = (0,) * nd

    def relax(off):
        q = qpval(off)
        t_s = (np.sqrt(1.0 + 1.0 / q ** 2) - 1.0 / q) / f0
        return t_s, 1.0 / (f0 ** 2 * t_s * t_s) - 1.0
    t_s, tt = relax(zero)
    damp = dval(zero)
    m = 1.0 / vpval(zero) ** 2
    e = (1.0 - damp) / dt
    W = damp / (m / dt ** 2 + e)
    L = nested_taps(c, R, nd, bval)
    eq1 = {('r', 0, zero): damp * (1.0 - dt / t_s)}
    eq2 = {}
    if dirn == 1:
        rho = 1.0 / bval(zero)
        for off, w in L.items():
            eq1[('p', 0, off)] = damp * dt * tt / t_s * rho * w
            eq2[('p', 0, off)] = W * rho * (1.0 + tt) * w
        eq2[('r', 1, zero)] = -W
    else:
        eq1[('p', 0, zero)] = -damp * dt * tt / t_s
        for off, w in L.items():
            rho = 1.0 / bval(off)
            eq2[('p', 0, off)] = W * rho * (1.0 + relax(off)[1]) * w
            eq2[('r', -1, off)] = W * rho * w
    eq2[('p', 0, zero)] = eq2.get(('p', 0, zero), 0.0) + W * (2.0 * m / dt ** 2 + e)
    eq2[('p', -dirn, zero)] = -W * m / dt ** 2
    return eq1, eq2


# ---------------------------------------------------------------------------------------------
# the stencil the TTI kernels implement, as linear coefficients (float64) — used only by the
# recogniser to confirm that a user's equations are this scheme.
# ---------------------------------------------------------------------------------------------
def predict_tti(w2, w1, R, P, damp, dt, adjoint=False, nd=3):
    """`P(name, offset)` -> value of parameter `name` sampled `offset` grid points from the output
    point (constants ignore the offset). `adjoint`: the backward pair of `kernel_centered(..., forward=False)`,
    H0 = Gh(e2 p + sd r), Hz = Gzz(sd p + r) with e2, sd sampled at each tap point, the previous level t+1.
    `nd` = 2: the rotation (sin theta, cos theta) on (x, z) of `Gzz_centered_2d`."""
    h = R // 2
    z3 = (0,) * nd

    def C(off):
        th = P('theta', off)
        st, ct = np.sin(th), np.cos(th)
        if nd == 2:
            return [st, ct]
        ph = P('phi', off)
        return [st * np.cos(ph), st * np.sin(ph), ct]
    e2 = 1 + 2 * P('epsilon', z3)
    sd = np.sqrt(1 + 2 * P('delta', z3))

    def unit(d, o):
        v = [0] * nd
        v[d] = o
        return tuple(v)

    def add(dst, key, val):
        dst[key] = dst.get(key, 0.0) + val

    # Gzz = sum_d D-_d ( C_d(q) * Gz(q) ),  Gz(q) = sum_e C_e(q) D+_e f(q)
    gzz = {}
    for d in range(nd):
        for j in range(R):
            q = unit(d, j - h)
            cq = C(q)
            for e in range(nd):
                for i in range(R):
                    off = tuple(a + b for a, b in zip(q, unit(e, i - h + 1)))
                    add(gzz, off, w1[d][j] * cq[d] * cq[e] * w1[e][i])
    lap = {}
    add(lap, z3, sum(w[0] for w in w2))
    for d in range(nd):
        for k in range(1, R + 1):
            add(lap, unit(d, k), w2[d][k])
            add(lap, unit(d, -k), w2[d][k])
    vp = P('vp', z3)
    m_dt2 = 1.0 / (vp * vp) / (dt * dt)
    den = m_dt2 + damp / dt
    pu, pv = {}, {}
    if adjoint:
        E2 = lambda k: 1 + 2 * P('epsilon', k)
        SD = lambda k: np.sqrt(1 + 2 * P('delta', k))
        gh = dict(lap)
        for k, val in gzz.items():
            add(gh, k, -val)
        for k, val in gh.items():              # H0 = Gh(e2 p + sd r)
            add(pu, ('u', 0) + (k,), E2(k) * val / den)
            add(pu, ('v', 0) + (k,), SD(k) * val / den)
        for k, val in gzz.items():             # Hz = Gzz(sd p + r)
            add(pv, ('u', 0) + (k,), SD(k) * val / den)
            add(pv, ('v', 0) + (k,), val / den)
    else:
        for k, val in lap.items():
            add(pu, ('u', 0) + (k,), e2 * val / den)
            add(pv, ('u', 0) + (k,), sd * val / den)
        for k, val in gzz.items():
            add(pu, ('u', 0) + (k,), -e2 * val / den)
            add(pu, ('v', 0) + (k,), sd * val / den)
            add(pv, ('u', 0) + (k,), -sd * val / den)
            add(pv, ('v', 0) + (k,), val / den)
    prev = 1 if adjoint else -1
    add(pu, ('u', 0, z3), (2 * m_dt2 + damp / dt) / den)
    add(pu, ('u', prev, z3), -m_dt2 / den)
    add(pv, ('v', 0, z3), (2 * m_dt2 + damp / dt) / den)
    add(pv, ('v', prev, z3), -m_dt2 / den)
    pu = {k: v for k, v in pu.items() if abs(v) > 1e-14}
    pv = {k: v for k, v in pv.items() if abs(v) > 1e-14}
    return pu, pv
