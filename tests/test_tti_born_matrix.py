"""Centred-TTI Born (linearised) modelling against the float64 reference (tests/tti_born_ref.py::tti_born_forward)
on the anisotropic, non-cubic grid of tests/kernel_cases.py, for every TTI sweep variant.

The operator is built with the DSL in the formulation of devito_b200/seismic/tti.py::JacobianOperator (the
background pair (u0, v0) driven by the sources, the linearised pair (du, dv) by -dm * u0.dt2 / -dm * v0.dt2, the
receivers sampling du + dv). Every time slot of the four wavefields starts as white noise, halo included; dm is
white noise with halo 0 or 3. The update box is the whole grid, an interior box, or one whose z extent ends in a
partial float4 group (kernel_cases.ZTAIL tail1 / tail3). Each case asserts from `b2_last_sweep_kernel` which sweep
variant ran for both pairs and which path of the Born source term ran ("+born_v4": float4 along z, taken when dm's
halo keeps the z rows 16-byte aligned and the z extent is a multiple of 4; "+born_s" otherwise). Tolerance: rel L-inf
1e-4 for u0, v0, du, dv and the traces.
"""
import functools
from types import SimpleNamespace

import numpy as np
import pytest

from helpers import rel_linf
import kernel_cases as KC
import tti_born_ref as TB

pytestmark = pytest.mark.gpu

TOL = 1e-4


def _last_kernel():
    from devito_b200 import _lib
    return _lib.lib().b2_last_sweep_kernel().decode()


def born_case(so, arrays, box=None, dmh=0, seed=0, shape=KC.SHAPE):
    """A KC TTI case plus the linearised pair (white noise in every slot) and dm with halo `dmh`."""
    c = KC.tti_case(so, arrays, shape=shape, box=box, seed=seed)
    rng = np.random.default_rng(seed + 100 * so + 53)
    c['du'] = rng.standard_normal(c['u'].shape).astype(np.float32)
    c['dv'] = rng.standard_normal(c['u'].shape).astype(np.float32)
    c['dm'] = (0.05 * rng.standard_normal(tuple(n + 2 * dmh for n in shape))).astype(np.float32)
    c['dmh'] = dmh
    return c


@functools.lru_cache(maxsize=None)
def _setup(so, arrays, box=None, dmh=0, shape=KC.SHAPE, seams=None):
    """(operator, functions, case, source tables) on `shape`; `seams`: KC.sparse_coordinates' points beside the
    tile and x-chunk seams, added to its usual points"""
    from devito_b200 import (Constant, Eq, Function, Grid, Operator, SparseTimeFunction, TimeFunction, solve,
                             sqrt)
    from devito_b200.seismic.tti import Gzz_centered
    c = born_case(so, arrays, box, dmh, shape=shape)
    grid = Grid(shape=shape, extent=tuple((n - 1) * h for n, h in zip(shape, KC.SPACING)))

    def fn(name, values, space_order=so):
        f = Function(name=name, grid=grid, space_order=space_order)
        f.data_with_halo[:] = values
        return f
    mk = lambda n: TimeFunction(name=n, grid=grid, time_order=2, space_order=so)
    u0, v0, du, dv = mk('u0'), mk('v0'), mk('du'), mk('dv')
    damp = fn('damp', c['damp'])
    dm = fn('dm', c['dm'], dmh)
    P = {n: (fn(n, x) if arrays else Constant(name=n, value=float(x))) for n, x in c['params'].items()}
    model = SimpleNamespace(theta=P['theta'], phi=P['phi'])
    m = 1 / (P['vp'] * P['vp'])
    sd, e2 = sqrt(1 + 2 * P['delta']), 1 + 2 * P['epsilon']

    def pair(u, v, qu=0, qv=0):
        gxx = u.laplace - Gzz_centered(model, u)
        gzz = Gzz_centered(model, v)
        return [Eq(u.forward, solve(m * u.dt2 - (e2 * gxx + sd * gzz) - qu + damp * u.dt, u.forward)),
                Eq(v.forward, solve(m * v.dt2 - (sd * gxx + gzz) - qv + damp * v.dt, v.forward))]
    interpolation = 'sinc' if so >= 8 else 'linear'
    coords = KC.sparse_coordinates(shape, seams=seams)
    tables = KC.sparse_tables(coords, interpolation, KC.K + 2)
    sp = lambda n: SparseTimeFunction(name=n, grid=grid, npoint=len(coords), nt=KC.K + 2, interpolation=interpolation,
                                      r=tables['r'], coordinates=coords)
    src, rec = sp('src'), sp('rec')
    src.data[:] = tables['data']
    dt = grid.stepping_dim.spacing
    eqs = pair(u0, v0) + src.inject(field=(u0.forward, v0.forward), expr=src * dt ** 2 / m) + \
        pair(du, dv, qu=-dm * u0.dt2, qv=-dm * v0.dt2) + rec.interpolate(expr=du + dv)
    op = Operator(eqs)
    assert op.backend == 'cuda-sm90a', op._why_not
    return op, dict(u0=u0, v0=v0, du=du, dv=dv, rec=rec), c, tables


@functools.lru_cache(maxsize=None)
def _reference(key):
    _, _, c, tables = _setup(*key)
    so = c['so']
    (w2, w1), _ = KC.weights('tti', so)
    rec = dict(tables, data=np.zeros_like(tables['data']))
    u, v, du, dv, tr = TB.tti_born_forward(c['u'], c['v'], c['du'], c['dv'], c['dm'], c['dmh'], so, w2, w1,
                                           c['dt'], 1, KC.K, c['damp'], c['params'], lo=c['lo'], hi=c['hi'],
                                           src=tables, rec=rec)
    return dict(u0=u, v0=v, du=du, dv=dv, rec=tr)


def _apply(key, **kw):
    op, f, c, _ = _setup(*key)
    for n, k in (('u0', 'u'), ('v0', 'v'), ('du', 'du'), ('dv', 'dv')):
        f[n].data_with_halo[:] = c[k]
    f['rec'].data[:] = 0.0
    lo, hi = c['lo'], c['hi']
    op.apply(time_m=1, time_M=KC.K, dt=c['dt'], x_m=lo[0], x_M=hi[0], y_m=lo[1], y_M=hi[1], z_m=lo[2], z_M=hi[2],
             **kw)
    out = {n: np.array(f[n].data_ro_with_halo) for n in ('u0', 'v0', 'du', 'dv')}
    out['rec'] = np.array(f['rec'].data)
    return out


def _check(key, sweep, **kw):
    got = _apply(key, **kw)
    _, _, c, _ = _setup(*key)
    # float4 along z needs dm's z rows 16-byte aligned (halo 0) and a z extent of whole float4 groups
    born = 'v4' if key[3] == 0 and (c['hi'][2] - c['lo'][2] + 1) % 4 == 0 else 's'
    assert _last_kernel() == f'{sweep}+born_{born}'
    want = _reference(key)
    assert np.abs(got['du']).max() > 0.1
    for n in ('u0', 'v0', 'du', 'dv', 'rec'):
        err = rel_linf(got[n], want[n])
        assert err < TOL, f"{n}: {err:.2e}"


# variables the library does not read: set to what once selected other array-parameter sweeps, they change nothing
STALE_ARR_ENV = {'B2_TTI_ARR_CT': '0', 'B2_TTI_ARR_PREFETCH': '0', 'B2_TTI_ARR_FUSED': '0'}

VARIANTS = [
    # (so, arrays, environment, apply kernel=, sweep variant)
    (4, False, {}, 1, 'tti_two_pass'),
    (4, False, {}, 0, 'tti_fused<2>'),
    (8, False, {}, 1, 'tti_two_pass'),
    (8, False, {'B2_TTI_KERNEL': '2'}, 0, 'tti_fused<4>'),
    (8, False, {}, 0, 'tti_ws<pf1>'),
    (12, False, {}, 0, 'tti_two_pass'),
    (4, True, {}, 0, 'tti_arr_ct2<2>'),
    (8, True, {}, 0, 'tti_arr_ct2<4>'),
    (4, True, {'B2_TTI_ARR_HINT': '0'}, 0, 'tti_arr_ct2<2>'),
    (8, True, {'B2_TTI_ARR_HINT': '0'}, 0, 'tti_arr_ct2<4>'),
    (4, True, STALE_ARR_ENV, 0, 'tti_arr_ct2<2>'),
    (8, True, STALE_ARR_ENV, 0, 'tti_arr_ct2<4>'),
    (8, True, {}, 1, 'tti_two_pass'),
    (12, True, {}, 0, 'tti_two_pass'),
]


BOXES = dict(full=None, sub=KC.SUBBOX, tail1=KC.ZTAIL['tail1'], tail3=KC.ZTAIL['tail3'])


@pytest.mark.parametrize('box', list(BOXES))
@pytest.mark.parametrize('dmh', [0, 3])
@pytest.mark.parametrize('so,arrays,env,kernel,sweep', VARIANTS,
                         ids=[f"so{v[0]}-{'arr' if v[1] else 'scalar'}-{v[4]}-{'-'.join(v[2].values()) or 'default'}"
                              f"-k{v[3]}" for v in VARIANTS])
def test_tti_born(so, arrays, env, kernel, sweep, dmh, box, monkeypatch):
    monkeypatch.setenv('B2_TTI_LX', '12')
    for k, val in env.items():
        monkeypatch.setenv(k, val)
    _check((so, arrays, BOXES[box], dmh), sweep, kernel=kernel)
