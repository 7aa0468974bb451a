"""Reference-side binding: the Operator backend a devito maintainer would add as `devito/core/b200.py`.

    import devito                       # the REAL reference (devito @ 436199c)
    import devito_b200.refplugin        # registers (Hopper, 'advanced', 'cuda')
    configuration['platform'], configuration['language'] = 'hopper', 'cuda'
    # ... examples/seismic run unchanged: the wave propagators execute in libb200stencil.so

The open-source reference has no operator for `(Hopper, 'advanced', 'cuda')`
(devito/operator/registry.py:33-57 raises "Cannot compile an Operator for ..."); this module fills
that slot with `B200CudaOperator`:

* `_build` lowers the expressions with the reference's own CPU pipeline (so `op.parameters`,
  `op.arguments()` and argument checking stay the reference's, devito/operator/operator.py:218-315,
  :608-757), and — next to it — restates the user's equations in `devito_b200`'s expression tree
  and hands them to that package's pattern recogniser. Operators that are not one of the
  propagation schemes of libb200stencil (the set-up operators of examples/seismic: `initdamp`,
  `smooth`, `norm` ...) simply stay CPU operators and JIT-compile with gcc like before.
* `apply` of a recognised operator calls `self.arguments(**kwargs)` — the reference builds its own
  `struct dataobj` for every array (devito/types/dense.py:737-777) and its own coordinate tables
  `src_gp/src_wx/...` (devito/operations/interpolators.py:674-718) — and passes THOSE STRUCTS to
  `b2_iso_forward` / `b2_tti_forward` (include/b200stencil.h). The library stages host arrays in and
  out inside the call, like the reference's device path does around its kernel
  (devito/passes/iet/definitions.py:636-671).

Nothing here is imported by `devito_b200` itself; importing this module needs the unmodified reference
package on `sys.path`.
"""
import ctypes
import os
import time as _time
from fractions import Fraction

import numpy as np
import sympy

import devito
from devito import configuration
from devito.arch.archinfo import Hopper, get_platform
from devito.core.cpu import Cpu64AdvOmpOperator
from devito.data.allocators import default_allocator
from devito.operator.registry import operator_registry
from devito.operations.interpolators import Injection as _RefInjection, Interpolation as _RefInterpolation
from devito.types.basic import AbstractFunction
from devito.types import Eq as _RefEq

import devito_b200 as dv
from devito_b200 import _lib as L_
from devito_b200.equation import FreeSurface
from devito_b200.symbolics import Access, Index, Number, Call, _np_funcs

__all__ = ['B200CudaOperator', 'register', 'activate', 'reference_cpu']

# tests: run recognised operators on the reference's own CPU path (same Operator objects)
_force_cpu = [False]


class reference_cpu:
    """Context manager: inside it every B200CudaOperator applies through the reference's CPU code path."""

    def __enter__(self):
        self._old = _force_cpu[0]
        _force_cpu[0] = True

    def __exit__(self, *a):
        _force_cpu[0] = self._old


class _Unconvertible(Exception):
    pass


# ---------------------------------------------------------------------------------------------
# the user's (reference) expressions restated in devito_b200's tree — for RECOGNITION only;
# no data is copied, the shadow objects never allocate
# ---------------------------------------------------------------------------------------------
class _Shadow:
    def __init__(self):
        self.grids, self.fns, self.consts, self.sparse = {}, {}, {}, {}

    def grid(self, g):
        if id(g) in self.grids:
            return self.grids[id(g)]
        subs = []
        sd = g.subdomains
        if 'physdomain' in sd or 'fsdomain' in sd:
            from devito_b200.seismic.model import PhysicalDomain, FSDomain
            fs = 'fsdomain' in sd
            so = int(getattr(sd['fsdomain'], 'size', 0)) if fs else int(getattr(sd.get('physdomain'), 'so', 0))
            subs.append(PhysicalDomain(so, fs=fs))
            if fs:
                subs.append(FSDomain(so))
        sg = dv.Grid(shape=tuple(g.shape), extent=tuple(float(e) for e in g.extent),
                     origin=tuple(float(o) for o in g.origin), dtype=g.dtype, subdomains=subs)
        if [d.name for d in g.dimensions] != [d.name for d in sg.dimensions]:
            raise _Unconvertible("grid dimensions are not named x, y, z")
        self.grids[id(g)] = sg
        return sg

    def function(self, f):
        if id(f) in self.fns:
            return self.fns[id(f)]
        if f.is_SparseTimeFunction:
            sg = self.grid(f.grid)
            kind = type(f.interpolator).__name__
            interp = {'LinearInterpolator': 'linear', 'SincInterpolator': 'sinc'}.get(kind)
            if interp is None:
                raise _Unconvertible(f"sparse function with {kind}")
            s = dv.SparseTimeFunction(name=f.name, grid=sg, npoint=int(f.npoint), nt=int(f.nt),
                                      interpolation=interp, r=int(f.r))
        elif f.is_TimeFunction:
            sg = self.grid(f.grid)
            s = dv.TimeFunction(name=f.name, grid=sg, time_order=int(f.time_order), space_order=int(f.space_order),
                                save=int(f.save) if isinstance(f.save, (int, np.integer)) else None)
            if f.save is not None and not isinstance(f.save, (int, np.integer)):
                raise _Unconvertible("buffered / conditional saving")
        elif f.is_Function:
            s = dv.Function(name=f.name, grid=self.grid(f.grid), space_order=int(f.space_order))
        else:
            raise _Unconvertible(f"function type {type(f).__name__}")
        if f.is_DiscreteFunction and getattr(f, 'staggered', None) not in (None, ()) and \
                any(v != 0 for v in getattr(f.staggered, '_getters', {}).values() if isinstance(v, int)):
            raise _Unconvertible("staggered function")
        self.fns[id(f)] = s
        return s

    def constant(self, c):
        if id(c) not in self.consts:
            self.consts[id(c)] = dv.Constant(name=c.name, value=float(c.data))
        return self.consts[id(c)]

    # -- expressions -------------------------------------------------------------------------------
    def symbol(self, s, grid):
        for sp in grid.spacing_symbols:
            if sp.name == s.name:
                return sp
        if s.name == grid.stepping_dim.spacing.name:
            return grid.stepping_dim.spacing
        raise _Unconvertible(f"free symbol {s}")

    def access(self, e):
        f = e.function
        sf = self.function(f)
        if all(i == d for i, d in zip(e.indices, f.dimensions)):
            return sf
        idx = []
        for i, d, sd in zip(e.indices, f.dimensions, sf.dimensions):
            off = sympy.sympify(i) - d
            if off == 0:
                idx.append(Index(sd, 0))
                continue
            if d.is_Time or d.is_Stepping:
                sp = d.spacing
            else:
                sp = d.spacing
            k = sympy.nsimplify(sympy.simplify(off / sp), rational=True)
            if not k.is_Rational:
                raise _Unconvertible(f"index {i} of {f.name}")
            idx.append(Index(sd, Fraction(int(k.p), int(k.q))))
        return Access(sf, idx)

    def expr(self, e, grid):
        e = sympy.sympify(e)
        if isinstance(e, AbstractFunction):
            return self.access(e)
        if getattr(e, 'is_Constant', False) and hasattr(e, 'data') and not e.is_Number:
            return self.constant(e)
        if e.is_Number:
            if e.is_Integer:
                return Number(int(e))
            return Number(float(e))
        if e.is_Symbol:
            return self.symbol(e, grid)
        if e.is_Add:
            out = self.expr(e.args[0], grid)
            for a in e.args[1:]:
                out = out + self.expr(a, grid)
            return out
        if e.is_Mul:
            out = self.expr(e.args[0], grid)
            for a in e.args[1:]:
                out = out * self.expr(a, grid)
            return out
        if e.is_Pow:
            return self.expr(e.base, grid) ** self.expr(e.exp, grid)
        name = type(e).__name__
        if name in _np_funcs and len(e.args) == 1:
            return Call(name, self.expr(e.args[0], grid))
        raise _Unconvertible(f"expression node {name}")


def _restate(expressions, kwargs):
    """devito_b200.Operator over the restated equations, or None when they are not on its fast path."""
    sh = _Shadow()
    items, eqs = [], []
    grid = None
    for e in expressions:
        for f in (e.lhs.function,) if isinstance(e, _RefEq) and hasattr(e.lhs, 'function') else ():
            if getattr(f, 'grid', None) is not None:
                grid = grid or f.grid
    if grid is None:
        return None
    sg = sh.grid(grid)
    fs_rows = []
    for e in expressions:
        if isinstance(e, _RefInjection):
            sf = sh.function(e.interpolator.sfunction)
            if isinstance(e.field, (tuple, list, sympy.Tuple)):      # TTI: one source into u and v
                field = [sh.expr(f, sg) for f in e.field]
                ex = ([sh.expr(x, sg) for x in e.expr] if isinstance(e.expr, (tuple, list, sympy.Tuple))
                      else sh.expr(e.expr, sg))
            else:
                field, ex = sh.expr(e.field, sg), sh.expr(e.expr, sg)
            items += sf.inject(field=field, expr=ex)
        elif isinstance(e, _RefInterpolation):
            sf = sh.function(e.interpolator.sfunction)
            items += sf.interpolate(expr=sh.expr(e.expr, sg), increment=bool(e.increment))
        elif isinstance(e, _RefEq):
            sd = e.subdomain
            name = getattr(sd, 'name', None)
            if name == 'fsdomain':
                fs_rows.append(e)           # examples/seismic/acoustic/operators.py:5-47 `freesurface`
                continue
            ssd = sg.subdomains[name] if name in ('physdomain', 'interior') else None
            if sd is not None and ssd is None and name not in (None, 'domain'):
                raise _Unconvertible(f"subdomain {name}")
            cls = dv.Inc if type(e).__name__ == 'Inc' else dv.Eq
            q = cls(sh.expr(e.lhs, sg), sh.expr(e.rhs.evaluate, sg), subdomain=ssd)
            eqs.append((e, q))
            items.append(q)
        else:
            raise _Unconvertible(f"{type(e).__name__} in the operator")
    if fs_rows:
        # the reference's free surface: [mirrored copy of the update on fsdomain, `u.forward[z=0] = 0`]
        if len(fs_rows) != 2 or len(eqs) != 1:
            raise _Unconvertible("free-surface equations next to more than one update")
        mirrored, zero = fs_rows
        ref_update, q = eqs[0]
        if mirrored.lhs != ref_update.lhs or zero.rhs != 0 or zero.lhs.function is not ref_update.lhs.function:
            raise _Unconvertible("unexpected free-surface equations")
        if not mirrored.rhs.has(devito.sign):
            raise _Unconvertible("free-surface equation without mirrored taps")
        items.insert(items.index(q) + 1, FreeSurface(q, sg.subdomains['fsdomain']))
    subs = {}
    for k, v in (kwargs.get('subs') or {}).items():
        subs[sh.symbol(k, sg)] = float(v)
    op = dv.Operator(items, subs=subs, name=kwargs.get('name', 'Kernel'))
    if op.backend != 'cuda-sm90a' or op._plan.get('kind') not in ('iso', 'tti'):
        return None
    return op



# ---------------------------------------------------------------------------------------------
# first-order systems on staggered grids (elastic, staggered TTI ...): tap tables for b2_system_forward
# ---------------------------------------------------------------------------------------------
class _SystemPlan:
    """What `_restate_system` extracts from the reference's evaluated equations."""

    def __init__(self):
        self.fields = []            # reference TimeFunctions, index = field id
        self.scratch = []           # (field id, name) of scratch fields (interpolated expressions)
        self.stages = []            # (out id, out_tshift, [(fid, tshift, off, coef, key|None)], box widening)
        self.coef_exprs = {}        # key -> sympy expression of a coefficient array
        self.injections = []        # (sparse function, [fids], tshift, scale expression)
        self.interpolations = []    # (sparse function, fid, tshift)
        self.grid = None
        self.so = None


def _wave_accesses(expr, fset):
    out = []
    for a in sympy.preorder_traversal(expr):
        if isinstance(a, AbstractFunction) and a.function.name in fset and a not in out:
            out.append(a)
    return out


def _array_offsets(acc):
    """(tshift, array offsets) of an access to a (staggered) TimeFunction: the symbolic offset in units of the
    spacing minus the function's own half-cell stagger must be an integer."""
    f = acc.function
    stag = tuple(getattr(f, 'staggered', None) or (0,) * len(f.dimensions))
    tshift, offs = 0, []
    for i, d, sg in zip(acc.indices, f.dimensions, stag):
        k = sympy.nsimplify(sympy.simplify((sympy.sympify(i) - d) / d.spacing), rational=True)
        if not k.is_Rational:
            raise _Unconvertible(f"index {i} of {f.name}")
        if d.is_Time:
            tshift = int(k)
            continue
        k = k - sympy.Rational(int(sg), 2) if sg else k
        if k.q != 1:
            raise _Unconvertible(f"{f.name}: offset {i} is not on the function's own (staggered) grid")
        offs.append(int(k))
    return tshift, tuple(offs)


def _linear_parts(rhs, fset):
    """rhs = sum_a coef_a * a over the wavefield accesses a; raises when it is not linear / has a rest.
    (The expressions are devito's Differentiable nodes, on which `sympy.diff` stays unevaluated: the
    coefficient of a is rhs[a = 1, others = 0] - rhs[all = 0]; linearity is probed numerically.)"""
    accs = _wave_accesses(rhs, fset)
    dummies = {a: sympy.Dummy(f"w{i}") for i, a in enumerate(accs)}
    e = rhs.xreplace(dummies)
    zero = {d: sympy.Integer(0) for d in dummies.values()}
    rest = e.xreplace(zero)
    parts = []
    for a, dmy in dummies.items():
        one = dict(zero)
        one[dmy] = sympy.Integer(1)
        c = e.xreplace(one) - rest
        parts.append((a, c))
    # numeric probe: every non-wavefield leaf (parameter accesses, SafeInv nodes, symbols) gets a random value
    rng = np.random.default_rng(7)
    vals = {d: rng.uniform(-1.0, 1.0) for d in dummies.values()}

    def num(x):
        if x in vals:
            return vals[x]
        if x.is_Number:
            return float(x)
        if isinstance(x, AbstractFunction) or type(x).__name__ in ('SafeInv', 'cos', 'sin', 'sqrt', 'exp', 'Abs') \
                or x.is_Symbol:
            return vals.setdefault(x, rng.uniform(0.5, 1.5))
        if x.is_Add:
            return sum(num(a) for a in x.args)
        if x.is_Mul:
            out = 1.0
            for a in x.args:
                out *= num(a)
            return out
        if x.is_Pow:
            return num(x.base) ** num(x.exp)
        raise _Unconvertible(f"expression node {type(x).__name__}")
    full = num(e)
    r0 = num(rest)
    lin = r0 + sum(num(c) * vals[dummies[a]] for a, c in parts)
    if abs(full - lin) > 1e-9 * max(1.0, abs(full)):
        raise _Unconvertible("update is not linear in the wavefields")
    if abs(r0) > 1e-12:
        raise _Unconvertible("update has a term without a wavefield")
    return [(a, c) for a, c in parts if c != 0]


def _restate_system(expressions, kwargs):
    """Tap tables for a sequence of explicit updates `f.forward = linear(fields)`; None when the operator has
    no such form (the acoustic / TTI second-order schemes never come here: `_restate` takes them first)."""
    plan = _SystemPlan()
    subs = dict(kwargs.get('subs') or {})
    updates, sparse_ops = [], []
    for e in expressions:
        if isinstance(e, (_RefInjection, _RefInterpolation)):
            sparse_ops.append(e)
        elif isinstance(e, _RefEq):
            if e.subdomain is not None and getattr(e.subdomain, 'name', None) not in ('domain', 'physdomain'):
                raise _Unconvertible(f"subdomain {getattr(e.subdomain, 'name', None)}")
            ev = e.evaluate
            flat = ev._flatten if hasattr(ev, '_flatten') else [ev]
            for q in flat:
                updates.append((q.lhs, q.rhs))
        else:
            raise _Unconvertible(f"{type(e).__name__} in the operator")
    if not updates:
        return None
    for lhs, _ in updates:
        f = getattr(lhs, 'function', None)
        if f is None or not f.is_TimeFunction or f.time_order != 1 or f.save is not None:
            raise _Unconvertible("lhs is not a buffered first-order-in-time TimeFunction")
        if f.name not in [q.name for q in plan.fields]:
            plan.fields.append(f)
    grid = plan.fields[0].grid
    so = plan.fields[0].space_order
    if any(f.grid is not grid or f.space_order != so for f in plan.fields) or grid.dim not in (2, 3):
        raise _Unconvertible("fields on different grids / space orders")
    if 'physdomain' in grid.subdomains and any(getattr(d, 'is_Sub', False) for d in grid.subdomains['physdomain'].dimensions):
        raise _Unconvertible("free-surface model")
    plan.grid, plan.so = grid, so
    plan.values = {str(k): float(v) for k, v in subs.items()}       # spacings substituted by the Operator (`subs=`)
    fset = {f.name for f in plan.fields}           # by name: tensor components are re-created on access
    fid = {f.name: i for i, f in enumerate(plan.fields)}

    def taps_of(rhs):
        taps = []
        for acc, coef in _linear_parts(rhs, fset):
            tshift, offs = _array_offsets(acc)
            if tshift not in (0, 1) or any(abs(o) > so for o in offs):
                raise _Unconvertible("tap outside the supported time levels / halo")
            # coefficient = scalar part (numbers, dt, spacings: evaluated when the operator is applied) x field part
            # (material parameters / damping at shifted positions: tabulated as one array per distinct expression)
            coef = sympy.sympify(coef)
            deps = {n for n in sympy.preorder_traversal(coef)
                    if isinstance(n, AbstractFunction) or type(n).__name__ == 'SafeInv'}
            scal, fieldpart = (coef.as_independent(*deps, as_Add=False) if deps else (coef, sympy.Integer(1)))
            key = None
            if fieldpart != 1:
                key = str(fieldpart)            # (srepr does not print the names of devito Functions: collisions)
                plan.coef_exprs.setdefault(key, fieldpart)
            taps.append((fid[acc.function.name], tshift, offs, scal, key))
        return taps

    for lhs, rhs in updates:
        tshift, offs = _array_offsets(lhs)
        if tshift != 1 or any(offs):
            raise _Unconvertible("lhs is not `f.forward` at the function's own position")
        plan.stages.append((fid[lhs.function.name], 1, taps_of(rhs), 0))
    dt = grid.stepping_dim.spacing
    for e in sparse_ops:
        sf = e.interpolator.sfunction
        if type(e.interpolator).__name__ not in ('LinearInterpolator', 'SincInterpolator'):
            raise _Unconvertible("interpolator")
        if isinstance(e, _RefInjection):
            flds = (list(e.field) if isinstance(e.field, (tuple, list, sympy.Tuple, sympy.MatrixBase)) or
                    getattr(e.field, 'is_Matrix', False) else [e.field])
            exprs = list(e.expr) if isinstance(e.expr, (tuple, list, sympy.Tuple)) else [e.expr] * len(flds)
            if len(flds) > 3 or len({str(sympy.sympify(x)) for x in exprs}) != 1:
                raise _Unconvertible("injection into more than 3 fields / with different expressions")
            ids, shifts = [], set()
            for a in flds:
                if a.function.name not in fset:
                    raise _Unconvertible("injection into a field that is not updated")
                ts, offs = _array_offsets(a)
                if any(offs) or any(getattr(a.function, 'staggered', None) or ()):
                    raise _Unconvertible("injection into a staggered field")
                ids.append(fid[a.function.name])
                shifts.add(ts)
            src_acc = [a for a in sympy.preorder_traversal(sympy.sympify(exprs[0]))
                       if isinstance(a, AbstractFunction) and a.function.name == sf.name]
            if len(shifts) != 1 or len(src_acc) != 1:
                raise _Unconvertible("injection expression")
            scale = sympy.simplify(sympy.sympify(exprs[0]) / src_acc[0])
            pacc = [a for a in sympy.preorder_traversal(scale) if isinstance(a, AbstractFunction)]
            pkind, pfn = 0, None
            if pacc:
                # src * dt * vp**2  /  src * dt / m : the injection kernel's two position-dependent scale modes
                P = pacc[0]
                if len(set(pacc)) != 1 or any(i != d for i, d in zip(P.indices, P.function.dimensions)) or \
                        P.function.space_order != so:
                    raise _Unconvertible("position-dependent injection scale")
                for kind, q in ((1, sympy.simplify(scale / P ** 2)), (2, sympy.simplify(scale * P))):
                    if not any(isinstance(a, AbstractFunction) for a in sympy.preorder_traversal(q)):
                        pkind, pfn, scale = kind, P.function, q
                        break
                else:
                    raise _Unconvertible("position-dependent injection scale")
            plan.injections.append((sf, ids, shifts.pop(), scale, pkind, pfn))
        else:
            if e.increment:
                raise _Unconvertible("incremental interpolation")
            # the interpolated expression is evaluated at the sparse points' (node) position
            # (devito/operations/interpolators.py:527 `expr._eval_at(self.sfunction).evaluate`)
            ex = sympy.sympify(e.expr)
            ex = ex._eval_at(sf) if hasattr(ex, '_eval_at') else ex
            if isinstance(ex, AbstractFunction) and ex.function.name in fset and \
                    not any(getattr(ex.function, 'staggered', None) or ()):
                ts, offs = _array_offsets(ex)
                if any(offs):
                    raise _Unconvertible("interpolation of a shifted field")
                plan.interpolations.append((sf, fid[ex.function.name], ts))
            else:
                # an expression (div(v) ...): an extra stage fills a scratch field that is then sampled
                evx = ex.evaluate
                sid = len(plan.fields) + len(plan.scratch)
                taps = taps_of(evx)
                # the interpolation guard samples cells up to r beyond the domain, where the reference evaluates the
                # expression from the fields' halo: the stage's box is widened by r, which its taps must allow
                r = int(sf.r)
                if any(key is not None for *_, key in taps) or any(abs(o) + r > so for _, _, offs, _, _ in taps
                                                                   for o in offs):
                    raise _Unconvertible(f"{sf.name}: the expression cannot be evaluated {r} cells into the halo")
                plan.scratch.append((sid, f"scratch_{sf.name}"))
                plan.stages.append((sid, 0, taps, r))
                plan.interpolations.append((sf, sid, 0))
    if len(plan.fields) + len(plan.scratch) > 16:
        raise _Unconvertible("too many fields")
    # stages that fill scratch fields read time level t: run them BEFORE the updates overwrite nothing they need
    # (they read tshift 0 only, the updates write tshift 1), order as given is fine
    return plan


def _eval_coef(expr, grid, values):
    """NumPy evaluation of a coefficient expression (material parameters at shifted node positions, SafeInv,
    numbers, dt) over the grid's domain, float32 like the reference's generated code."""
    shape = tuple(grid.shape)

    def rec(e):
        if isinstance(e, AbstractFunction):
            f = e.function
            arr = f.data_with_halo.view(np.ndarray) if hasattr(f, 'data_with_halo') else None
            sl = []
            for i, d, (hl, hr), n in zip(e.indices, f.dimensions, f._size_halo, shape):
                k = sympy.nsimplify(sympy.simplify((sympy.sympify(i) - d) / d.spacing), rational=True)
                if not (k.is_Rational and k.q == 1) or abs(int(k)) > hl:
                    raise _Unconvertible(f"parameter access {e}")
                sl.append(slice(hl + int(k), hl + int(k) + n))
            return np.asarray(arr[tuple(sl)], dtype=np.float32)
        if getattr(e, 'is_Constant', False) and hasattr(e, 'data') and not e.is_Number:
            return np.float32(e.data)
        if e.is_Number:
            return np.float32(float(e))
        if e.is_Symbol:
            if e.name in values:
                return np.float32(values[e.name])
            raise _Unconvertible(f"no value for {e}")
        if e.is_Add:
            out = rec(e.args[0])
            for a in e.args[1:]:
                out = out + rec(a)
            return out
        if e.is_Mul:
            out = rec(e.args[0])
            for a in e.args[1:]:
                out = out * rec(a)
            return out
        if e.is_Pow:
            b, x = rec(e.base), e.exp
            if x == -1:
                return np.float32(1.0) / b
            return np.power(b, np.float32(float(x)))
        if type(e).__name__ in ('cos', 'sin', 'sqrt', 'exp', 'Abs') and len(e.args) == 1:
            fn = {'cos': np.cos, 'sin': np.sin, 'sqrt': np.sqrt, 'exp': np.exp, 'Abs': np.abs}[type(e).__name__]
            return fn(rec(e.args[0])).astype(np.float32)
        if type(e).__name__ == 'SafeInv':
            # devito/passes/iet/misc.py:243-258: (a < eps || b < eps) ? 0 : 1/a with eps = resolution^2
            a, b = rec(e.args[0]), rec(e.args[1])
            eps = np.float32(np.finfo(np.float32).resolution ** 2)
            with np.errstate(divide='ignore'):
                return np.where((a < eps) | (b < eps), np.float32(0.0), np.float32(1.0) / a).astype(np.float32)
        raise _Unconvertible(f"coefficient node {type(e).__name__}")
    out = rec(sympy.sympify(expr))
    return np.ascontiguousarray(np.broadcast_to(out, shape), dtype=np.float32)

# ---------------------------------------------------------------------------------------------
# the Operator
# ---------------------------------------------------------------------------------------------
def _addr(cobj):
    """Address of the struct behind whatever ctypes handle `op.arguments()` holds (byref / pointer)."""
    if hasattr(cobj, '_obj'):
        return ctypes.addressof(cobj._obj)
    if hasattr(cobj, 'contents'):
        return ctypes.addressof(cobj.contents)
    return ctypes.addressof(cobj)


def _coef_resident(arr):
    """A tabulated coefficient array as a device-resident `struct dataobj` (dmap set, no host copy): uploaded once,
    reused by every apply until the fingerprint of its inputs changes."""
    import torch
    dev = dv.configuration['deviceid']
    device = torch.device('cuda', 0 if dev is None or dev < 0 else dev)
    t = torch.from_numpy(np.array(arr, dtype=np.float32, order='C')).to(device)
    torch.cuda.synchronize(device)
    obj = L_.make_dataobj(dev_ptr=t.data_ptr(), shape=arr.shape)
    obj._keep = t
    return obj


class B200CudaOperator(Cpu64AdvOmpOperator):
    """`(Hopper, 'advanced', 'cuda')`: wave propagators run in libb200stencil.so, everything else
    stays on the reference's CPU path."""

    @classmethod
    def _normalize_kwargs(cls, **kwargs):
        # the CPU lowering (argument machinery, set-up operators) is OpenMP C on the host cores
        kwargs = dict(kwargs)
        kwargs['options'] = dict(kwargs['options'], openmp=True)
        kwargs['b200_target'] = (kwargs['platform'], kwargs['language'])
        kwargs['platform'] = get_platform()
        kwargs['language'] = 'openmp'
        kwargs['compiler'] = configuration['compiler'].__new_with__(platform=kwargs['platform'], language='openmp',
                                                                    mpi=configuration['mpi'])
        kwargs['allocator'] = default_allocator(f"{kwargs['compiler'].__class__.__name__}.openmp.{kwargs['platform']}")
        return super()._normalize_kwargs(**kwargs)

    @classmethod
    def _build(cls, expressions, **kwargs):
        kwargs.pop('b200_target', None)
        op = super()._build(expressions, **kwargs)
        op._b200_sys = None
        try:
            op._b200 = _restate(expressions, kwargs)
            op._b200_why = None
        except (_Unconvertible, ValueError, TypeError, KeyError, AttributeError) as e:
            op._b200, op._b200_why = None, f"{type(e).__name__}: {e}"
        if op._b200 is None:
            # not one of the second-order propagators: a first-order system on a staggered grid?
            try:
                op._b200_sys = _restate_system(expressions, kwargs)
            except (_Unconvertible, ValueError, TypeError, KeyError, AttributeError, NotImplementedError) as e:
                op._b200_why = f"{op._b200_why}; as a linear system: {type(e).__name__}: {e}"
        return op

    @property
    def backend(self):
        if getattr(self, '_b200', None) is not None or getattr(self, '_b200_sys', None) is not None:
            return 'cuda-sm90a'
        return 'reference-cpu'

    @staticmethod
    def _system_coefs(plan, keys, values):
        """The coefficient arrays of a system, device-resident and cached across applies: they depend on dt, the
        spacings and the material parameters only, so they are re-tabulated (NumPy, `_eval_coef`) only when a
        fingerprint of those changes (sum and strided-sample sum of every parameter array involved)."""
        params = {}
        for k in keys:
            for n in sympy.preorder_traversal(plan.coef_exprs[k]):
                if isinstance(n, AbstractFunction):
                    params[n.function.name] = n.function
        fp = [tuple(sorted(values.items()))]
        for name in sorted(params):
            d = params[name].data_with_halo.view(np.ndarray)
            flat = d.reshape(-1)
            fp.append((name, d.shape, float(flat.sum(dtype=np.float64)), float(flat[::max(1, flat.size // 65536)].sum(dtype=np.float64))))
        fp = tuple(fp)
        cache = getattr(plan, '_coef_cache', None)
        if cache is not None and cache['fp'] == fp:
            return cache['objs']
        objs = [_coef_resident(_eval_coef(plan.coef_exprs[k], plan.grid, values)) for k in keys]
        plan._coef_cache = {'fp': fp, 'objs': objs}
        return objs

    def _apply_system(self, plan, **kwargs):
        """Run a staggered-grid system through `b2_system_forward` with the reference's own arrays."""
        from devito_b200.system import LinearSystem, Stage, Tap
        from devito_b200.operator import PerformanceSummary, PerfEntry
        kwargs.pop('autotune', None)
        with self._profiler.timer_on('arguments-preprocess'):
            args = self.arguments(**kwargs)
        grid, nd = plan.grid, plan.grid.dim
        values = dict(getattr(plan, 'values', {}))
        for sp in grid.spacing_symbols:
            if sp.name in args:
                values.setdefault(sp.name, float(args[sp.name]))
        values[grid.stepping_dim.spacing.name] = float(args['dt'])
        hold = []

        def dataobj(name):
            fo = L_.ForeignDataobj(_addr(args[name]), keep=args[name])
            hold.append(fo)
            return fo

        fields = [dataobj(f.name) for f in plan.fields]
        alloc = tuple(int(s) + 2 * plan.so for s in grid.shape)
        for sid, name in plan.scratch:
            arr = np.zeros((1,) + alloc, dtype=np.float32)
            hold.append(arr)
            fields.append(L_.make_dataobj(host=arr))
        keys = list(plan.coef_exprs)
        coefs = self._system_coefs(plan, keys, values)
        kid = {k: i for i, k in enumerate(keys)}
        def scalar(ex):
            ex = sympy.sympify(ex)
            return float(ex.xreplace({q: values[q.name] for q in ex.free_symbols if q.name in values}))
        stages = [Stage(out, ts, [Tap(f, t, o, scalar(c), kid[key] if key is not None else -1) for f, t, o, c, key in taps],
                        ext) for out, ts, taps, ext in plan.stages]

        def sparse(sf):
            ws = [dataobj(f"{sf.name}_w{'xyz'[i]}" if f"{sf.name}_w{'xyz'[i]}" in args else f"wsincrp_{sf.name}{'xyz'[i]}")
                  for i in range(nd)]
            return L_.ForeignSparse(sf.name, dataobj(sf.name), dataobj(f"{sf.name}_gp"), ws,
                                    p_m=int(args[f'p_{sf.name}_m']), p_M=int(args[f'p_{sf.name}_M']), r=int(sf.r))
        inj = []
        for sf, ids, ts, scale, pkind, pfn in plan.injections:
            inj.append((sparse(sf), ids, ts, scalar(scale), pkind, dataobj(pfn.name) if pfn is not None else None))
        itp = [(sparse(sf), fidx, ts) for sf, fidx, ts in plan.interpolations]
        system = LinearSystem(nd, plan.so, len(fields), stages, inj, itp)
        lo = [int(args[d.min_name]) for d in grid.dimensions]
        hi = [int(args[d.max_name]) for d in grid.dimensions]
        dev = dv.configuration['deviceid']
        timers, wall = system.apply(fields, coefs, lo, hi, int(args['time_m']), int(args['time_M']),
                                    deviceid=0 if dev is None or dev < 0 else dev)
        nsteps = int(args['time_M']) - int(args['time_m']) + 1
        pts = float(np.prod([h - l + 1 for l, h in zip(lo, hi)])) * nsteps
        summary = PerformanceSummary()
        for nm in ('section0', 'section1', 'section2'):
            t = getattr(timers, nm)
            summary[nm] = PerfEntry(t, gpointss=(pts / t / 1e9 if t > 0 and nm == 'section0' else None))
        summary.globals['fdlike'] = PerfEntry(wall, gpointss=pts / wall / 1e9 if wall > 0 else None)
        self._b200_last = {'wall': wall, 'stages': len(stages), 'coefficient_arrays': len(coefs),
                           'taps': sum(len(s.taps) for s in stages)}
        return summary

    def arguments(self, **kwargs):
        # thread-count defaults ask `configuration['platform']` — the GPU here — for its "cores"
        # (devito/types/parallel.py:66-70): give the host's instead
        names = {p.name for p in self.parameters}
        host = get_platform()
        for n in ('nthreads', 'nthreads_nonaffine'):
            if n in names:
                kwargs.setdefault(n, int(os.environ.get('OMP_NUM_THREADS', host.cores_physical)))
        return super().arguments(**kwargs)

    def apply(self, **kwargs):
        if _force_cpu[0]:
            return super().apply(**kwargs)
        shadow = getattr(self, '_b200', None)
        if shadow is None and getattr(self, '_b200_sys', None) is not None:
            return self._apply_system(self._b200_sys, **kwargs)
        if shadow is None:
            return super().apply(**kwargs)
        kwargs.pop('autotune', None)
        # the reference's own argument processing: defaults, overrides, checks, struct dataobj
        with self._profiler.timer_on('arguments-preprocess'):
            args = self.arguments(**kwargs)
        p = shadow._plan
        ov = {'resident': False, 'dt': float(args['dt']), 'time_m': int(args['time_m']), 'time_M': int(args['time_M'])}
        for d in p['grid'].dimensions:
            ov[d.min_name], ov[d.max_name] = int(args[d.min_name]), int(args[d.max_name])
        hold = []

        def dataobj(name):
            fo = L_.ForeignDataobj(_addr(args[name]), keep=args[name])
            hold.append(fo)
            return fo

        fields = [p['u']] + ([p['v']] if p['kind'] == 'tti' else [])
        for f in fields + [p.get(k) for k in ('damp', 'usave', 'grad', 'born_U', 'born_dm', 'snap')]:
            if f is not None:
                ov[f.name] = dataobj(f.name)
        if p['kind'] == 'iso':
            kind, obj = p['m_role']
            if obj is not None:
                ov[obj.name] = dataobj(obj.name) if kind.endswith('_f') else float(args[obj.name])
        else:
            for n, c in p['consts'].items():
                ov[n] = dataobj(n) if hasattr(c, 'space_order') else float(args[n])
        for key in ('src', 'rec'):
            sf = p.get(key)
            if sf is None:
                continue
            nd = p['grid'].dim
            # weight tables: `<name>_wx..` (linear, interpolators.py:674-718), `wsincrp_<name>x..` (sinc, :721-789)
            ws = [dataobj(f"{sf.name}_w{'xyz'[i]}" if f"{sf.name}_w{'xyz'[i]}" in args else f"wsincrp_{sf.name}{'xyz'[i]}")
                  for i in range(nd)]
            ov[sf.name] = L_.ForeignSparse(sf.name, dataobj(sf.name), dataobj(f"{sf.name}_gp"), ws,
                                           p_m=int(args[f'p_{sf.name}_m']), p_M=int(args[f'p_{sf.name}_M']), r=sf.r)
        t0 = _time.perf_counter()
        summary = shadow.apply(**ov)
        self._b200_last = {'wall': _time.perf_counter() - t0, 'arguments': sorted(ov)}
        return summary


def register():
    """`operator_registry.add(...)` exactly like devito/core/__init__.py:37-83 does for the stock backends."""
    operator_registry.add(B200CudaOperator, Hopper, 'advanced', 'cuda')
    operator_registry.add(B200CudaOperator, Hopper, 'noop', 'cuda')
    operator_registry.add(B200CudaOperator, Hopper, 'advanced-fsg', 'cuda')


def activate():
    """What `DEVITO_PLATFORM=hopper DEVITO_LANGUAGE=cuda` does."""
    register()
    configuration['platform'] = 'hopper'
    configuration['language'] = 'cuda'


register()
