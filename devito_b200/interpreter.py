"""NumPy interpreter for operators that are NOT the wave-propagation hot path.

The reference JIT-compiles every Operator, including tiny set-up ones (`initdamp`,
`initialize_function`, `norm`, the 2-D diffusion tutorial). Those are not performance
relevant; here they are evaluated with NumPy slicing over shifted views — the same idea as the
reference's own NumPy twin in examples/cfd/example_diffusion.py:61-83. The recognised
acoustic/TTI propagators never come here (operator.py dispatches them to the CUDA library
and fails loudly when it is unavailable).
"""
import numpy as np

from .symbolics import Number, Add, Mul, Pow, Call, _np_funcs
from .exceptions import InvalidArgument

__all__ = ['Interpreter']


class _Env:
    """Evaluation context for one equation at one time step."""

    def __init__(self, ranges, axes, time, scalars, shape):
        self.ranges = ranges      # {root_dim_name or subdim name: (lo, hi)} per iteration dim
        self.axes = axes          # {dim name: axis position in the broadcast shape}
        self.time = time
        self.scalars = scalars    # {symbol name: value}
        self.shape = shape


def _subsampled(f):
    """The factor of a function saved on a time ConditionalDimension (snapshots), else None."""
    td = getattr(f, 'time_dim', None)
    if getattr(f, 'is_buffered', True) or not getattr(td, 'is_Conditional', False) or not td.factor:
        return None
    return int(td.factor)


def _time_index(f, idx, time):
    if idx.absolute is not None:
        return idx.absolute
    fac = _subsampled(f)
    if fac is not None:
        # usave[t_sub + shift] with t_sub = time / factor
        return time // fac + int(idx.shift)
    t = time + int(idx.shift)
    if getattr(f, 'is_buffered', False):
        return t % f.time_size
    return t


def _slice_access(acc, env, for_write=False):
    """View of the function's allocated array for this access over the iteration ranges,
    reshaped to broadcast against the iteration shape."""
    f = acc.function
    arr = f.storage.host if for_write else f.storage.host_ro
    sl = []
    out_axes = []
    for axis, (idx, d) in enumerate(zip(acc.index_objs, f.dimensions)):
        hl = f.halo[axis][0]
        if d.is_Time:
            sl.append(_time_index(f, idx, env.time))
            continue
        if idx.absolute is not None:
            sl.append(idx.absolute + hl)
            continue
        name = idx.base.name
        if name not in env.ranges:
            raise InvalidArgument(f"dimension {name} of {f.name} is not iterated")
        if idx.shift.denominator != 1:
            raise InvalidArgument(f"non-integer index shift {idx.shift} on {f.name}")
        lo, hi = env.ranges[name]
        s = int(idx.shift)
        if lo + hl + s < 0 or hi + 1 + hl + s > arr.shape[axis]:
            raise InvalidArgument(f"OOB detected due to {f.name}[{name}{s:+d}] over [{lo},{hi}]")
        sl.append(slice(lo + hl + s, hi + 1 + hl + s))
        out_axes.append(env.axes[name])
    view = arr[tuple(sl)]
    # place the view's axes into the broadcast shape
    nd = len(env.shape)
    if view.ndim == 0:
        return view
    order = np.argsort(out_axes)
    view = np.transpose(view, order) if list(order) != list(range(view.ndim)) else view
    shape = [1] * nd
    for ax, n in zip(sorted(out_axes), view.shape):
        shape[ax] = n
    return view.reshape(shape)


def evaluate(expr, env):
    if isinstance(expr, Number):
        v = expr.value
        return float(v) if not isinstance(v, int) else v
    if expr.is_Access:
        return _slice_access(expr, env)
    if expr.is_Dimension:
        name = expr.name
        if name in env.ranges:
            lo, hi = env.ranges[name]
            shape = [1] * len(env.shape)
            shape[env.axes[name]] = hi - lo + 1
            return np.arange(lo, hi + 1, dtype=np.float64).reshape(shape)
        if expr.is_Time:
            return env.time
        raise InvalidArgument(f"dimension {name} not iterated")
    if expr.is_Constant:
        return expr.data if expr.name not in env.scalars else env.scalars[expr.name]
    if expr.is_Symbol:
        if expr.name in env.scalars:
            return env.scalars[expr.name]
        raise InvalidArgument(f"no value for symbol {expr.name}")
    if isinstance(expr, Add):
        out = evaluate(expr.args[0], env)
        for a in expr.args[1:]:
            out = out + evaluate(a, env)
        return out
    if isinstance(expr, Mul):
        out = evaluate(expr.args[0], env)
        for a in expr.args[1:]:
            out = out * evaluate(a, env)
        return out
    if isinstance(expr, Pow):
        b = evaluate(expr.base, env)
        e = evaluate(expr.exponent, env)
        if isinstance(e, int) and e == -1:
            return 1.0 / b
        return b ** e
    if isinstance(expr, Call):
        return _np_funcs[expr.name](evaluate(expr.arg, env))
    if expr.is_Derivative:
        return evaluate(expr.evaluate, env)
    raise TypeError(f"cannot evaluate {type(expr).__name__}")


class Interpreter:
    def __init__(self, eqs, sparse_ops, subs, name='Kernel'):
        from .equation import Eq
        self.name = name
        self.subs = dict(subs or {})
        self.items = []      # ordered list of ('eq', Eq) / ('inject', op) / ('interp', op)
        for kind, obj in eqs:
            if kind == 'eq':
                lhs = obj.lhs
                rhs = obj.rhs.evaluate
                if self.subs:
                    rhs = rhs.subs(self.subs)
                self.items.append(("eq", None, obj, lhs, rhs))
            else:
                self.items.append((kind, None, obj, None, None))
        self.functions = self._collect()

    def _collect(self):
        fs = {}
        for kind, _, obj, lhs, rhs in self.items:
            if kind == 'eq':
                for e in (lhs, rhs):
                    for n in e.preorder():
                        if n.is_Access:
                            fs[n.function.name] = n.function
            elif kind == 'inject':
                fs[obj.sfunction.name] = obj.sfunction
                for fld, ex in zip(obj.fields, obj.exprs):
                    fs[fld.function.name] = fld.function
                    for n in ex.preorder():
                        if n.is_Access:
                            fs[n.function.name] = n.function
            else:
                fs[obj.sfunction.name] = obj.sfunction
                for n in obj.expr.preorder():
                    if n.is_Access:
                        fs[n.function.name] = n.function
        return fs

    @property
    def has_time(self):
        return any(getattr(f, 'is_TimeFunction', False) or getattr(f, 'is_SparseTimeFunction', False)
                   for f in self.functions.values())

    def time_shifts(self):
        lo, hi = 0, 0
        for kind, _, obj, lhs, rhs in self.items:
            if kind != 'eq':
                continue
            for e in (lhs, rhs):
                for n in e.preorder():
                    if n.is_Access and getattr(n.function, 'is_TimeFunction', False):
                        idx = n.index_objs[0]
                        if idx.absolute is None:
                            lo = min(lo, int(idx.shift))
                            hi = max(hi, int(idx.shift))
        return lo, hi

    def direction(self):
        """+1 / -1: the reference iterates time backward when the updates write an earlier level than they
        read (`f.backward = ...`, devito/ir/support/space.py Backward); a mix is refused."""
        shifts = set()
        for kind, _, obj, lhs, rhs in self.items:
            if kind == 'eq' and lhs.is_Access and getattr(lhs.function, 'is_TimeFunction', False):
                idx = lhs.index_objs[0]
                if idx.absolute is None:
                    shifts.add(int(idx.shift))
        if any(s < 0 for s in shifts):
            if any(s > 0 for s in shifts):
                raise InvalidArgument("forward and backward time updates in one operator")
            return -1
        return 1

    # -- iteration space of one equation ---------------------------------------------------------
    def _ranges(self, eq, lhs, bounds):
        f = lhs.function
        ranges, axes = {}, {}
        sdmap = eq.subdomain.dimension_map if eq.subdomain is not None else {}
        ax = 0
        for idx, d in zip(lhs.index_objs, f.dimensions):
            if d.is_Time or idx.absolute is not None:
                continue
            base = idx.base
            root = base.root
            n = f.shape[f.dimensions.index(d)]
            pmin, pmax = bounds.get(root.name, (0, n - 1))
            if base.is_Sub:
                lo, hi = base.bounds(pmin, pmax)
            elif root in sdmap and sdmap[root].is_Sub:
                lo, hi = sdmap[root].bounds(pmin, pmax)
            else:
                lo, hi = pmin, pmax
            ranges[base.name] = (lo, hi)
            ranges.setdefault(root.name, (lo, hi))
            axes[base.name] = ax
            axes.setdefault(root.name, ax)
            ax += 1
        shape = [0] * ax
        for nme, a in axes.items():
            lo, hi = ranges[nme]
            shape[a] = hi - lo + 1
        return ranges, axes, tuple(shape)

    def _run_eq(self, eq, lhs, rhs, time, scalars, bounds):
        ranges, axes, shape = self._ranges(eq, lhs, bounds)
        if any(s <= 0 for s in shape):
            return
        env = _Env(ranges, axes, time, scalars, shape)
        val = evaluate(rhs, env)
        dst = _slice_access(lhs, env, for_write=True)
        f = lhs.function
        val = np.asarray(val, dtype=np.float64) if np.ndim(val) else val
        if eq.is_Increment:
            dst += np.asarray(val).astype(f.dtype, copy=False) if np.ndim(val) else f.dtype(val)
        else:
            dst[...] = np.asarray(val).astype(f.dtype, copy=False) if np.ndim(val) else f.dtype(val)

    # -- sparse ops --------------------------------------------------------------------------------
    def _cells(self, sf, field_fn, bounds):
        """Index arrays (per dim) of the support cells, validity mask and weights."""
        gp, ws = sf.tabulate()
        r = sf.r
        nd = gp.shape[1]
        n = 2 * r
        w = np.ones((sf.npoint,) + (n,) * nd)
        idxs = []
        valid = np.ones((sf.npoint,) + (n,) * nd, dtype=bool)
        space_dims = [d for d in field_fn.dimensions if d.is_Space]
        for j in range(nd):
            sh = (sf.npoint,) + tuple(n if i == j else 1 for i in range(nd))
            k = np.arange(n).reshape((1,) + sh[1:])
            cell = gp[:, j].reshape((-1,) + (1,) * nd) + k - r + 1
            d = space_dims[j]
            size = field_fn.shape[field_fn.dimensions.index(d)]
            lo, hi = bounds.get(d.name, (0, size - 1))
            valid = valid & (cell >= lo - r) & (cell <= hi + r)
            hl = field_fn.halo[field_fn.dimensions.index(d)][0]
            valid = valid & (cell + hl >= 0) & (cell + hl < size + 2 * hl)
            idxs.append(np.broadcast_to(cell, valid.shape))
            w = w * ws[j].astype(np.float64).reshape(sh)
        return idxs, valid, w

    def _eval_at_cells(self, expr, sf, idxs, time, scalars):
        """Evaluate expr where grid functions are gathered at cells and sparse functions at p."""
        def rec(e):
            if isinstance(e, Number):
                return float(e.value)
            if e.is_Access:
                f = e.function
                if getattr(f, 'is_SparseFunction', False):
                    data = f.storage.host_ro
                    if getattr(f, 'is_SparseTimeFunction', False):
                        row = data[time + int(e.index_objs[0].shift)]
                    else:
                        row = data
                    return row.reshape((-1,) + (1,) * len(idxs)).astype(np.float64)
                arr = f.storage.host_ro
                ind = []
                j = 0
                for axis, (idx, d) in enumerate(zip(e.index_objs, f.dimensions)):
                    if d.is_Time:
                        ind.append(_time_index(f, idx, time))
                    else:
                        hl = f.halo[axis][0]
                        ind.append(np.clip(idxs[j] + hl + int(idx.shift), 0, arr.shape[axis] - 1))
                        j += 1
                return arr[tuple(ind)].astype(np.float64)
            if e.is_Constant:
                return float(scalars.get(e.name, e.data))
            if e.is_Symbol:
                return float(scalars[e.name])
            if isinstance(e, Add):
                return sum(rec(a) for a in e.args)
            if isinstance(e, Mul):
                out = 1.0
                for a in e.args:
                    out = out * rec(a)
                return out
            if isinstance(e, Pow):
                return rec(e.base) ** rec(e.exponent)
            if isinstance(e, Call):
                return _np_funcs[e.name](rec(e.arg))
            raise TypeError(type(e).__name__)
        return rec(expr.evaluate.subs(self.subs) if self.subs else expr.evaluate)

    def _run_inject(self, op, time, scalars, bounds):
        sf = op.sfunction
        for fld, ex in zip(op.fields, op.exprs):
            f = fld.function
            idxs, valid, w = self._cells(sf, f, bounds)
            val = self._eval_at_cells(ex, sf, idxs, time, scalars) * w
            arr = f.storage.host
            ind = []
            j = 0
            for axis, (idx, d) in enumerate(zip(fld.index_objs, f.dimensions)):
                if d.is_Time:
                    ind.append(np.full(valid.shape, _time_index(f, idx, time)))
                else:
                    hl = f.halo[axis][0]
                    ind.append(np.clip(idxs[j] + hl, 0, arr.shape[axis] - 1) + np.zeros(valid.shape, dtype=np.int64))
                    j += 1
            val = np.broadcast_to(val, valid.shape)
            np.add.at(arr, tuple(i[valid] for i in ind), val[valid].astype(f.dtype))

    def _run_interp(self, op, time, scalars, bounds):
        sf = op.sfunction
        fields = [n.function for n in op.expr.preorder()
                  if n.is_Access and not getattr(n.function, 'is_SparseFunction', False)]
        if not fields:
            raise InvalidArgument("interpolate: expression has no grid function")
        idxs, valid, w = self._cells(sf, fields[0], bounds)
        val = self._eval_at_cells(op.expr, sf, idxs, time, scalars)
        val = np.where(valid, np.broadcast_to(val, valid.shape) * w, 0.0)
        res = val.reshape(sf.npoint, -1).sum(axis=1)
        data = sf.storage.host
        if getattr(sf, 'is_SparseTimeFunction', False):
            if op.increment:
                data[time] += res.astype(sf.dtype)
            else:
                data[time] = res.astype(sf.dtype)
        else:
            data[:] = res.astype(sf.dtype) if not op.increment else data + res.astype(sf.dtype)

    # -- driver ------------------------------------------------------------------------------------
    def run(self, time_m, time_M, scalars, bounds):
        steps = range(time_m, time_M + 1) if self.has_time else [0]
        if self.has_time and self.direction() < 0:
            steps = reversed(steps)
        for time in steps:
            for kind, _, obj, lhs, rhs in self.items:
                if kind == 'eq':
                    fac = _subsampled(lhs.function) if lhs.is_Access else None
                    if fac is not None and time % fac:
                        continue            # a snapshot is written where time % factor == 0 only
                    self._run_eq(obj, lhs, rhs, time, scalars, bounds)
                elif kind == 'inject':
                    self._run_inject(obj, time, scalars, bounds)
                else:
                    self._run_interp(obj, time, scalars, bounds)
