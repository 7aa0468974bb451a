"""Operators the seismic solvers and users build, and mutations of them, for the recogniser soundness tests.

`build(case, mutation, dtype)` returns a `Built`: the Operator, every dense and sparse function it reads or
writes (by name), and the keyword arguments of a K-step apply. Everything is seeded by name, so the float32
build and its float64 twin (`dtype=np.float64`) start from the same values: white noise in every slot and halo
cell of the wavefields, parameters drawn in physical ranges, sources and receivers at off-grid positions.

A mutation changes the equations by a small amount: a tap scaled by 1 + 1e-3, a parameter raised to a power
or read off-centre, the damping sign, an injection or interpolation expression, the dtype of one array. What
the recogniser accepts must be what the kernel computes: `test_recogniser_soundness.py` records which (case,
mutation) pairs are accepted, and `test_recogniser_soundness_matrix.py` runs every accepted pair on the GPU
against its float64 twin on the interpreter.
"""
import zlib
from functools import lru_cache
from typing import NamedTuple

import numpy as np

from devito_b200 import (ConditionalDimension, Constant, Eq, Function, Grid, Inc, Operator, SparseTimeFunction,
                         TimeFunction, solve)
from devito_b200.equation import FreeSurface
from devito_b200.operator import _space_offsets
from devito_b200.seismic import demo_model, setup_geometry
from devito_b200.seismic import acoustic as A
from devito_b200.seismic import self_adjoint as S
from devito_b200.seismic import tti as T
from devito_b200.sparse import Injection, Interpolation
from devito_b200.symbolics import Access, linear_terms

K = 4                               # time steps of every apply: time_m = 1 .. time_M = K
NT = K + 4                          # samples of every sparse function and saved field
SHAPE3, NBL3 = (15, 12, 20), 3      # -> a (21, 18, 26) grid
SHAPE2, NBL2 = (24, 35), 3          # -> a (30, 41) grid
SPACING3 = (10.0, 12.5, 8.0)
SPACING2 = (10.0, 7.5)
VPMAX = 2.5


# -- seeded values ---------------------------------------------------------------------------------------------
def _rng(name, salt=''):
    return np.random.default_rng(zlib.crc32(f'{name}:{salt}'.encode()))


# every parameter is drawn in a physical range; the float32 draw is the value of both twins
_RANGES = {'vp': (1.5, VPMAX), 'm': (1 / VPMAX ** 2, 1 / 1.5 ** 2), 'damp': (0.0, 0.03), 'epsilon': (0.0, 0.2),
           'delta': (0.0, 0.1), 'theta': (0.0, 0.6), 'phi': (0.0, 0.6), 'b': (0.5, 1.0), 'dm': (-0.1, 0.1)}


def seed(f):
    """White noise over the allocated array of `f` (every slot, halo included), in `_RANGES[name]` for a
    parameter and in [-1, 1] otherwise; for a sparse function also off-grid coordinates inside the domain."""
    lo, hi = _RANGES.get(f.name, (-1.0, 1.0))
    if getattr(f, 'is_SparseFunction', False):
        g = f.grid
        ext = np.array([(n - 1) * float(h) for n, h in zip(g.shape, g.spacing)])
        org = np.array([float(o) for o in g.origin])
        r = f.r
        pos = _rng(f.name, 'coords').uniform(0, 1, size=f.coordinates_data.shape)
        # keep every support cell (r on each side) inside the domain
        cell = pos * (np.array(g.shape) - 1 - 2 * r) + r
        f.coordinates_data[:] = (org + cell / (np.array(g.shape) - 1) * ext).astype(np.float32)
        f.data[:] = _rng(f.name).uniform(lo, hi, size=f.data.shape).astype(np.float32)
        return
    arr = f.data_with_halo
    arr[:] = _rng(f.name).uniform(lo, hi, size=arr.shape).astype(np.float32)


# -- models ------------------------------------------------------------------------------------------------------
def _model(preset, nd, so, dtype):
    shape, nbl, spacing = (SHAPE3, NBL3, SPACING3) if nd == 3 else (SHAPE2, NBL2, SPACING2)
    return demo_model(preset, shape=shape, nbl=nbl, spacing=spacing, space_order=so, dtype=dtype, nlayers=3)


def _geometry(model):
    # NT samples: the time axis 0 .. NT - 1 at step 1 (the apply passes its own dt)
    return setup_geometry(model, float(NT - 1)).resample(1.0)


def _sa_model(nd, so, dtype):
    shape, nbl, spacing = (SHAPE3, NBL3, SPACING3) if nd == 3 else (SHAPE2, NBL2, SPACING2)
    from devito_b200.seismic.model import Model
    return Model(origin=(0.0,) * nd, shape=shape, vp=1.5 * np.ones(shape), b=np.ones(shape), spacing=spacing,
                 nbl=nbl, space_order=so, bcs='damp', dtype=dtype)


def _dt(nd, so, h):
    """A stable float32-exact time step for vp <= VPMAX and epsilon <= 0.2."""
    from fractions import Fraction
    from devito_b200.symbolics import fd_weights
    w = fd_weights(2, list(range(-so, so + 1)), Fraction(0))
    cfl = np.sqrt(4.0 / (nd * sum(abs(float(c)) for c in w)))
    return float(np.float32(0.5 * cfl * min(h) / (VPMAX * np.sqrt(1.4))))


class Base(NamedTuple):
    items: list         # expression objects, in order
    subs: dict
    family: str         # 'iso', 'tti' or 'sa'
    nd: int
    so: int
    param: object       # the parameter the power / off-centre / m64 mutations change (vp, m or b)
    mexpr: object       # m (squared slowness) as an expression, for the injection mutations
    dt: float
    adjoint: bool


def _solver_items(op):
    return [o for _, o in op._items]


def _iso_solver(kind, nd=3, so=8, dtype=np.float32, kernel='OT2'):
    model = _model('layers-isotropic', nd, so, dtype)
    geom = _geometry(model)
    if kind == 'fwd':
        op = A.ForwardOperator(model, geom, space_order=so, kernel=kernel)
    elif kind == 'adj':
        op = A.AdjointOperator(model, geom, space_order=so, kernel=kernel)
    elif kind == 'born':
        op = A.BornOperator(model, geom, space_order=so)
    elif kind == 'grad':
        op = A.GradientOperator(model, geom, space_order=so)
    else:
        op = A.ForwardOperator(model, geom, space_order=so)
    items = _solver_items(op)
    if kind == 'snap':
        u = items[0].lhs.function
        t_sub = ConditionalDimension('t_sub', parent=model.grid.time_dim, factor=2)
        usave = TimeFunction(name='usave', grid=model.grid, time_order=2, space_order=so, save=NT // 2,
                             time_dim=t_sub)
        items.append(Eq(usave, u))
    return Base(items, dict(model.spacing_map), 'iso', nd, so, model.vp, model.m,
                _dt(nd, so, model.spacing), kind in ('adj', 'grad'))


def _tti_solver(kind, nd, so=8, dtype=np.float32):
    model = _model('layers-tti', nd, so, dtype)
    model._initialize_bcs(bcs='damp')
    geom = _geometry(model)
    op = (T.ForwardOperator if kind == 'fwd' else T.AdjointOperator)(model, geom, space_order=so)
    return Base(_solver_items(op), dict(model.spacing_map), 'tti', nd, so, model.vp, model.m,
                _dt(nd, so, model.spacing), kind == 'adj')


def _sa_solver(kind, nd, so=8, dtype=np.float32):
    model = _sa_model(nd, so, dtype)
    geom = _geometry(model)
    op = (S.IsoFwdOperator if kind == 'fwd' else S.IsoAdjOperator)(model, geom, space_order=so)
    return Base(_solver_items(op), dict(model.spacing_map), 'sa', nd, so, model.b, model.b / model.vp ** 2,
                _dt(nd, so, model.spacing), kind == 'adj')


def _hand(spelling, nd=3, so=8, dtype=np.float32):
    """The isotropic update written by hand: `solve(...)`, explicit, with m or vp, Function or Constant."""
    shape = tuple(n + 2 * nbl for n, nbl in zip(*((SHAPE3, (NBL3,) * 3) if nd == 3 else (SHAPE2, (NBL2,) * 2))))
    spacing = SPACING3 if nd == 3 else SPACING2
    grid = Grid(shape=shape, extent=tuple((n - 1) * h for n, h in zip(shape, spacing)), dtype=dtype)
    u = TimeFunction(name='u', grid=grid, time_order=2, space_order=so)
    damp = Function(name='damp', grid=grid, space_order=so)
    dt = grid.stepping_dim.spacing
    if spelling == 'vp_const':
        vp = param = Constant(name='vp', value=2.0, dtype=dtype)
        m = 1 / vp ** 2
    elif spelling == 'vp_func':
        vp = param = Function(name='vp', grid=grid, space_order=so)
        m = 1 / vp ** 2
    else:
        m = param = Function(name='m', grid=grid, space_order=4 if spelling == 'param_so4' else so)
    if spelling == 'explicit':
        eq = Eq(u.forward, 2 * u - u.backward + dt ** 2 / m * u.laplace)
    elif spelling == 'nodamp':
        eq = Eq(u.forward, solve(m * u.dt2 - u.laplace, u.forward))
    else:
        eq = Eq(u.forward, solve(m * u.dt2 - u.laplace + damp * u.dt, u.forward))
    src = SparseTimeFunction(name='src', grid=grid, npoint=3, nt=NT)
    rec = SparseTimeFunction(name='rec', grid=grid, npoint=7, nt=NT)
    hs = [float(h) for h in grid.spacing]
    step = _dt(nd, so, hs)
    inj = src * (float(np.float32(step)) ** 2 if spelling == 'lit_dt' else dt ** 2) / m
    items = [eq] + src.inject(field=u.forward, expr=inj) + \
        rec.interpolate(expr=u.forward if spelling == 'rec_forward' else u)
    subs = {}
    if spelling == 'subs':
        # spacings overridden with other values than the grid's: the weights follow `subs`
        subs = {d.spacing: h * 1.25 for d, h in zip(grid.dimensions, hs)}
        step = _dt(nd, so, [h * 1.25 for h in hs])
    return Base(items, subs, 'iso', nd, so, param, m, step, False)


# name -> builder(dtype). Solver operators first, then the hand spellings that must stay on the fast path.
BASES = {
    'iso_fwd': lambda dt: _iso_solver('fwd', dtype=dt),
    'iso_fwd_so4_2d': lambda dt: _iso_solver('fwd', nd=2, so=4, dtype=dt),
    'iso_adj': lambda dt: _iso_solver('adj', dtype=dt),
    'iso_born': lambda dt: _iso_solver('born', so=4, dtype=dt),
    'iso_grad': lambda dt: _iso_solver('grad', so=4, dtype=dt),
    'iso_ot4': lambda dt: _iso_solver('fwd', so=4, dtype=dt, kernel='OT4'),
    'iso_snap': lambda dt: _iso_solver('snap', so=4, dtype=dt),
    'tti_fwd': lambda dt: _tti_solver('fwd', 3, dtype=dt),
    'tti_adj': lambda dt: _tti_solver('adj', 3, so=4, dtype=dt),
    'tti_fwd_2d': lambda dt: _tti_solver('fwd', 2, dtype=dt),
    'tti_adj_2d': lambda dt: _tti_solver('adj', 2, so=4, dtype=dt),
    'sa_fwd': lambda dt: _sa_solver('fwd', 3, dtype=dt),
    'sa_adj': lambda dt: _sa_solver('adj', 2, dtype=dt),
    'hand_solve': lambda dt: _hand('solve', dtype=dt),
    'hand_solve_2d': lambda dt: _hand('solve', nd=2, so=4, dtype=dt),
    'hand_explicit': lambda dt: _hand('explicit', dtype=dt),
    'hand_vp_func': lambda dt: _hand('vp_func', dtype=dt),
    'hand_vp_const': lambda dt: _hand('vp_const', so=4, dtype=dt),
    'hand_nodamp': lambda dt: _hand('nodamp', so=4, dtype=dt),
    'hand_param_so4': lambda dt: _hand('param_so4', dtype=dt),
    'hand_subs': lambda dt: _hand('subs', so=4, dtype=dt),
    'hand_rec_forward': lambda dt: _hand('rec_forward', so=4, dtype=dt),
    'hand_lit_dt': lambda dt: _hand('lit_dt', so=4, dtype=dt),
}


# -- mutations ---------------------------------------------------------------------------------------------------
def _updates(items):
    """Indices of the plain time updates (not increments, not snapshot copies)."""
    out = []
    for i, o in enumerate(items):
        if isinstance(o, Eq) and not isinstance(o, Inc) and not isinstance(o, FreeSurface):
            f = o.lhs.function
            if getattr(f, 'is_TimeFunction', False) and f.is_buffered:
                out.append(i)
    return out


def _map_updates(items, fn, first_only=False):
    """`fn(rhs, eq)` applied to the evaluated right-hand side of the time updates."""
    out = list(items)
    for i in _updates(items)[:1] if first_only else _updates(items):
        e = items[i]
        out[i] = Eq(e.lhs, fn(e.rhs.evaluate, e), subdomain=e.subdomain)
    return out


def _scale_tap(items, pick, by=1e-3):
    """Scale one wavefield tap of the first update by 1 + `by`: `pick(time_shift, offsets, dirn)`."""
    def fn(rhs, e):
        u = e.lhs.function
        dirn = _space_offsets(e.lhs, None)[0]
        terms, _ = linear_terms(rhs, lambda a: a.function is u)
        for acc, coef in terms.items():
            t, o = _space_offsets(acc, None)
            if pick(t, o, dirn):
                return rhs + by * coef * acc
        raise AssertionError("no such tap")
    return _map_updates(items, fn, first_only=True)


def _subs_param(items, f, fn, centre_only=False):
    """Replace the accesses of `f` in the time updates by `fn(access)`."""
    def go(rhs, e):
        accs = [n for n in rhs.preorder() if (n.is_Access and n.function is f) or n is f]
        if centre_only:
            accs = [a for a in accs if not a.is_Access or not any(_space_offsets(a, None)[1])]
        return rhs.subs({a: fn(a) for a in accs})
    return _map_updates(items, go)


def _retype(items, old, new):
    """Every access of `old` (updates, injections, interpolations) read from `new` instead."""
    def sub(ex):
        accs = {n for n in ex.preorder() if n.is_Access and n.function is old}
        return ex.subs({a: Access(new, a.index_objs) for a in accs}) if accs else ex
    out = []
    for o in items:
        if isinstance(o, Inc):
            out.append(Inc(sub(o.lhs), sub(o.rhs.evaluate)))
        elif isinstance(o, Eq):
            out.append(Eq(sub(o.lhs), sub(o.rhs.evaluate), subdomain=o.subdomain))
        elif isinstance(o, Injection):
            sf = new if o.sfunction is old else o.sfunction
            out.extend(sf.inject(field=tuple(sub(a) for a in o.fields), expr=tuple(sub(x) for x in o.exprs)))
        elif isinstance(o, Interpolation):
            sf = new if o.sfunction is old else o.sfunction
            out.extend(sf.interpolate(expr=sub(o.expr)))
        else:
            out.append(o)
    return out


def _inject(items, make):
    """Replace the injection by `make(sf, access, dtsym, expr) -> (field access, expr)` per target."""
    out = []
    for o in items:
        if isinstance(o, Injection):
            sf = o.sfunction
            dts = sf.grid.stepping_dim.spacing
            pairs = [make(sf, a, dts, x) for a, x in zip(o.fields, o.exprs)]
            out.extend(sf.inject(field=tuple(p[0] for p in pairs), expr=tuple(p[1] for p in pairs)))
        else:
            out.append(o)
    return out


def _interpolate(items, make):
    out = []
    for o in items:
        out.extend(o.sfunction.interpolate(expr=make(o.expr)) if isinstance(o, Interpolation) else [o])
    return out


def _named(items, name):
    for o in items:
        exprs = [o.lhs, o.rhs.evaluate] if isinstance(o, Eq) else []
        for ex in exprs:
            for n in ex.preorder():
                if n.is_Access and n.function.name == name:
                    return n.function
    return None


def _eps_scaled(a):
    # (1 + 2 eps) -> (1 + 2 eps) (1 + 1e-3)
    return ((1 + 2 * a) * 1.001 - 1) / 2


def _delta_scaled(a):
    # sqrt(1 + 2 delta) -> sqrt(1 + 2 delta) (1 + 1e-3)
    return ((1 + 2 * a) * 1.001 ** 2 - 1) / 2


def _copy64(f):
    if getattr(f, 'is_SparseFunction', False):
        return SparseTimeFunction(name=f.name, grid=f.grid, npoint=f.npoint, nt=f.nt, dtype=np.float64,
                                  interpolation=f.interpolation, r=f.r)
    return Function(name=f.name, grid=f.grid, space_order=f.space_order, dtype=np.float64)


def _rebuilt(b):
    """The operator passed through every rebuild helper above with a change of zero: it must stay accepted, so that
    the refusals of the real mutations are due to the mutation and not to the rebuilding."""
    items = _scale_tap(b.items, lambda t, o, dirn: t == 0 and o[-1] == 1 and not any(o[:-1]), by=0.0)
    items = _subs_param(items, b.param, lambda a: a)
    items = _inject(items, lambda sf, a, dts, ex: (a, ex))
    items = _interpolate(items, lambda e: e)
    return _retype(items, b.param, b.param)


def _lit(b):
    return float(np.float32(b.dt)) ** 2


MUTATIONS = {
    'none': lambda b: b.items,
    'rebuilt': _rebuilt,
    # the stencil
    'tap': lambda b: _scale_tap(b.items, lambda t, o, dirn: t == 0 and o[-1] == 1 and not any(o[:-1])),
    'tm1': lambda b: _scale_tap(b.items, lambda t, o, dirn: t == -dirn and not any(o)),
    'pow2': lambda b: _subs_param(b.items, b.param, lambda a: a ** 2),
    'powm1': lambda b: _subs_param(b.items, b.param, lambda a: 1 / a),
    'offc': lambda b: _subs_param(b.items, b.param, lambda a: a._shift(b.param.grid.dimensions[0], 1)),
    'damp_sign': lambda b: _subs_param(b.items, _named(b.items, 'damp'), lambda a: -a),
    'eps': lambda b: _subs_param(b.items, _named(b.items, 'epsilon'), _eps_scaled),
    'delta': lambda b: _subs_param(b.items, _named(b.items, 'delta'), _delta_scaled),
    'b': lambda b: _subs_param(b.items, _named(b.items, 'b'), lambda a: a * 1.001, centre_only=True),
    # the injection
    'inj_lit_m2': lambda b: _inject(b.items, lambda sf, a, dts, ex: (a, sf * _lit(b) / b.mexpr ** 2)),
    'inj_lit_m': lambda b: _inject(b.items, lambda sf, a, dts, ex: (a, sf * _lit(b) * b.mexpr)),
    'inj_dt2_no_m': lambda b: _inject(b.items, lambda sf, a, dts, ex: (a, sf * dts ** 2)),
    'inj_lit_no_m': lambda b: _inject(b.items, lambda sf, a, dts, ex: (a, sf * 0.01)),
    'inj_twice': lambda b: _inject(b.items, lambda sf, a, dts, ex: (a, 2 * sf * dts ** 2 / b.mexpr)),
    'inj_level': lambda b: _inject(b.items, lambda sf, a, dts, ex: (a.function, sf * dts ** 2 / b.mexpr)),
    # the interpolation
    'itp_twice': lambda b: _interpolate(b.items, lambda e: 2 * e),
    'itp_plus_param': lambda b: _interpolate(b.items, lambda e: e + _named(b.items, 'damp')),
    'itp_dt': lambda b: _interpolate(b.items, lambda e: e.dt),
    # dtypes (the float64 grid is the builder's dtype argument)
    'grid64': None,
    'param64': lambda b: _retype(b.items, b.param, _copy64(b.param)),
    'sparse64': lambda b: _retype(b.items, _sparse(b.items)[0], _copy64(_sparse(b.items)[0])),
}


def _sparse(items):
    out = []
    for o in items:
        if isinstance(o, (Injection, Interpolation)) and o.sfunction not in out:
            out.append(o.sfunction)
    return out


def applies(case, mutation):
    """Whether `mutation` makes sense for `case`."""
    fam = case.split('_')[0]
    if mutation in ('eps', 'delta'):
        return fam == 'tti'
    if mutation == 'b':
        return fam == 'sa'
    if mutation in ('offc', 'param64'):
        # a parameter Function (not a Constant)
        return case != 'hand_vp_const'
    if mutation.startswith('inj_'):
        # the literal-dt spelling is the one injection that has no dt symbol to mutate
        return case != 'hand_lit_dt'
    if mutation.startswith('itp_') and case == 'iso_grad':
        # the gradient operator samples no receivers
        return False
    if mutation in ('damp_sign', 'itp_plus_param'):
        return case not in ('hand_explicit', 'hand_nodamp')
    return True


CASES = [(c, m) for c in BASES for m in MUTATIONS if applies(c, m)]


# -- the built operator --------------------------------------------------------------------------------------------
class Built(NamedTuple):
    op: Operator
    functions: dict     # name -> dense or sparse function read or written
    kwargs: dict        # apply arguments: dt, time_m, time_M
    family: str


def _functions(items):
    fs = {}
    for o in items:
        exprs = []
        if isinstance(o, Eq):
            exprs = [o.lhs, o.rhs.evaluate]
        elif isinstance(o, Injection):
            fs[o.sfunction.name] = o.sfunction
            exprs = list(o.fields) + list(o.exprs)
        elif isinstance(o, Interpolation):
            fs[o.sfunction.name] = o.sfunction
            exprs = [o.expr.evaluate]
        for ex in exprs:
            for n in ex.preorder():
                if n.is_Access:
                    fs[n.function.name] = n.function
    return fs


@lru_cache(maxsize=None)
def _base(case, dtype):
    return BASES[case](dtype)


def build(case, mutation='none', dtype=np.float32):
    """The Operator of `case` under `mutation`, its functions seeded, and its apply arguments."""
    b = _base(case, np.float64 if mutation == 'grid64' else dtype)
    items = b.items if mutation == 'grid64' else MUTATIONS[mutation](b)
    op = Operator(items, subs=b.subs, name=f'{case}-{mutation}')
    fns = _functions(items)
    for f in fns.values():
        seed(f)
    return Built(op, fns, {'dt': b.dt, 'time_m': 1, 'time_M': K}, b.family)
