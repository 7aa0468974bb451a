"""Centred-TTI adjoint and gradient against the float64 restatement (tests/tti_adjoint_ref.py) on the anisotropic,
non-cubic grid of tests/kernel_cases.py, for the adjoint variant of every TTI sweep the forward selects.

The operators are built with the DSL in the formulation of devito_b200/seismic/tti.py (`AdjointOperator`: the pair
(p, r) solved for .backward, the receivers injected into both at the level written, srca sampling p + r;
`JacobianAdjOperator`: the same pair plus Inc(grad, -(usave * p.dt2 + vsave * r.dt2))). Every time slot starts as
white noise, halo included; usave, vsave and grad (halo KC.GRAD_HALO) are white noise too. The update box is the
whole grid, an interior box, or one whose z extent ends in a partial float4 group (kernel_cases.ZTAIL tail1 / tail3:
the adjoint sweeps' partial loads of p and r). Each case asserts from `b2_last_sweep_kernel` which sweep variant ran:
the scalar so=8 sweep k_tti_ws has no adjoint variant (it would spill registers), so its adjoint runs
k_tti_fused<4>. Tolerance: rel L-inf 1e-4 for p, r, the traces and grad.
"""
import functools
from types import SimpleNamespace

import numpy as np
import pytest

from helpers import rel_linf
import kernel_cases as KC
import tti_adjoint_ref as TA

pytestmark = pytest.mark.gpu

TOL = 1e-4


def _last_kernel():
    from devito_b200 import _lib
    return _lib.lib().b2_last_sweep_kernel().decode()


def adj_case(so, arrays, box=None, seed=0, shape=KC.SHAPE):
    c = KC.tti_case(so, arrays, shape=shape, box=box, seed=seed)
    rng = np.random.default_rng(seed + 100 * so + 71)
    c['usave'] = rng.standard_normal((KC.K + 2,) + c['u'].shape[1:]).astype(np.float32)
    c['vsave'] = rng.standard_normal((KC.K + 2,) + c['u'].shape[1:]).astype(np.float32)
    c['grad'] = rng.standard_normal(tuple(n + 2 * KC.GRAD_HALO for n in shape)).astype(np.float32)
    return c


@functools.lru_cache(maxsize=None)
def _setup(so, arrays, gradient, box=None, shape=KC.SHAPE, seams=None):
    """(operator, functions, case, receiver tables) on `shape`; `seams`: KC.sparse_coordinates' points beside the
    tile and x-chunk seams, added to its usual points"""
    from devito_b200 import (Constant, Eq, Function, Grid, Inc, Operator, SparseTimeFunction, TimeFunction, solve,
                             sqrt)
    from devito_b200.seismic.tti import Gzz_centered
    c = adj_case(so, arrays, box, shape=shape)
    grid = Grid(shape=shape, extent=tuple((n - 1) * h for n, h in zip(shape, KC.SPACING)))

    def fn(name, values, space_order=so):
        f = Function(name=name, grid=grid, space_order=space_order)
        f.data_with_halo[:] = values
        return f
    p = TimeFunction(name='p', grid=grid, time_order=2, space_order=so)
    r = TimeFunction(name='r', grid=grid, time_order=2, space_order=so)
    damp = fn('damp', c['damp'])
    P = {n: (fn(n, x) if arrays else Constant(name=n, value=float(x))) for n, x in c['params'].items()}
    model = SimpleNamespace(theta=P['theta'], phi=P['phi'], grid=grid)
    m = 1 / (P['vp'] * P['vp'])
    sd, e2 = sqrt(1 + 2 * P['delta']), 1 + 2 * P['epsilon']
    a, b = e2 * p + sd * r, sd * p + r
    H0, Hz = a.laplace - Gzz_centered(model, a), Gzz_centered(model, b)
    eqs = [Eq(p.backward, solve(m * p.dt2 - H0 + damp * p.dt.T, p.backward)),
           Eq(r.backward, solve(m * r.dt2 - Hz + damp * r.dt.T, r.backward))]
    interpolation = 'sinc' if so >= 8 else 'linear'
    coords = KC.sparse_coordinates(shape, seams=seams)
    tables = KC.sparse_tables(coords, interpolation, KC.K + 2)
    sp = lambda n: SparseTimeFunction(name=n, grid=grid, npoint=len(coords), nt=KC.K + 2, interpolation=interpolation,
                                      r=tables['r'], coordinates=coords)
    rec, srca = sp('rec'), sp('srca')
    rec.data[:] = tables['data']
    dt = grid.stepping_dim.spacing
    eqs += rec.inject(field=(p.backward, r.backward), expr=rec * dt ** 2 / m)
    f = dict(p=p, r=r, srca=srca)
    if gradient:
        mk = lambda n: TimeFunction(name=n, grid=grid, time_order=2, space_order=so, save=KC.K + 2)
        f['u0'], f['v0'] = mk('u0'), mk('v0')
        f['u0'].data_with_halo[:] = c['usave']
        f['v0'].data_with_halo[:] = c['vsave']
        f['grad'] = Function(name='grad', grid=grid, space_order=KC.GRAD_HALO)
        eqs.append(Inc(f['grad'], -(f['u0'] * p.dt2 + f['v0'] * r.dt2)))
    else:
        eqs += srca.interpolate(expr=p + r)
    op = Operator(eqs)
    assert op.backend == 'cuda-sm90a', op._why_not
    return op, f, c, tables


@functools.lru_cache(maxsize=None)
def _reference(key):
    _, _, c, tables = _setup(*key)
    (w2, w1), _ = KC.weights('tti', c['so'])
    grad = c['grad'].astype(np.float64)
    gradient = key[2]
    p, r, tr = TA.tti_adjoint(c['u'], c['v'], c['so'], w2, w1, c['dt'], 1, KC.K, c['damp'], c['params'], lo=c['lo'],
                              hi=c['hi'], src=tables,
                              rec=None if gradient else dict(tables, data=np.zeros_like(tables['data'])),
                              grad=grad if gradient else None, gh=KC.GRAD_HALO, usave=c['usave'], vsave=c['vsave'])
    return dict(p=p, r=r, srca=tr, grad=grad)


def _check(key, sweep, **kw):
    op, f, c, _ = _setup(*key)
    f['p'].data_with_halo[:] = c['u']
    f['r'].data_with_halo[:] = c['v']
    names = ['p', 'r']
    if key[2]:
        f['grad'].data_with_halo[:] = c['grad']
        names.append('grad')
    else:
        f['srca'].data[:] = 0.0
    lo, hi = c['lo'], c['hi']
    op.apply(time_m=1, time_M=KC.K, dt=c['dt'], x_m=lo[0], x_M=hi[0], y_m=lo[1], y_M=hi[1], z_m=lo[2], z_M=hi[2],
             **kw)
    assert _last_kernel() == sweep
    want = _reference(key)
    got = {n: np.array(f[n].data_ro_with_halo) for n in names}
    if not key[2]:
        got['srca'] = np.array(f['srca'].data)
        names.append('srca')
    for n in names:
        err = rel_linf(got[n], want[n])
        assert err < TOL, f"{n}: {err:.2e}"


# variables the library does not read: set to what once selected other array-parameter sweeps, they change nothing
STALE_ARR_ENV = {'B2_TTI_ARR_CT': '0', 'B2_TTI_ARR_PREFETCH': '0', 'B2_TTI_ARR_FUSED': '0'}

VARIANTS = [
    # (so, arrays, environment, apply kernel=, sweep variant)
    (4, False, {}, 1, 'tti_two_pass+adj'),
    (4, False, {}, 0, 'tti_fused<2>+adj'),
    (8, False, {}, 1, 'tti_two_pass+adj'),
    (8, False, {'B2_TTI_KERNEL': '2'}, 0, 'tti_fused<4>+adj'),
    (8, False, {}, 0, 'tti_fused<4>+adj'),          # the forward runs k_tti_ws here
    (12, False, {}, 0, 'tti_two_pass+adj'),
    (4, True, {}, 0, 'tti_arr_ct2<2>+adj'),
    (8, True, {}, 0, 'tti_arr_ct2<4>+adj'),
    (4, True, {'B2_TTI_ARR_HINT': '0'}, 0, 'tti_arr_ct2<2>+adj'),
    (8, True, {'B2_TTI_ARR_HINT': '0'}, 0, 'tti_arr_ct2<4>+adj'),
    (4, True, STALE_ARR_ENV, 0, 'tti_arr_ct2<2>+adj'),
    (8, True, STALE_ARR_ENV, 0, 'tti_arr_ct2<4>+adj'),
    (8, True, {}, 1, 'tti_two_pass+adj'),
    (12, True, {}, 0, 'tti_two_pass+adj'),
]


BOXES = dict(full=None, sub=KC.SUBBOX, tail1=KC.ZTAIL['tail1'], tail3=KC.ZTAIL['tail3'])


@pytest.mark.parametrize('box', list(BOXES))
@pytest.mark.parametrize('gradient', [False, True], ids=['adjoint', 'gradient'])
@pytest.mark.parametrize('so,arrays,env,kernel,sweep', VARIANTS,
                         ids=[f"so{v[0]}-{'arr' if v[1] else 'scalar'}-{v[4]}-{'-'.join(v[2].values()) or 'default'}"
                              f"-k{v[3]}" for v in VARIANTS])
def test_tti_adjoint(so, arrays, env, kernel, sweep, gradient, box, monkeypatch):
    monkeypatch.setenv('B2_TTI_LX', '12')
    for k, val in env.items():
        monkeypatch.setenv(k, val)
    _check((so, arrays, gradient, BOXES[box]), sweep, kernel=kernel)
