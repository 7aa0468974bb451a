"""Every sweep-kernel variant against the float64 reference (tests/ref64.py) on an anisotropic, non-cubic grid.

Operators are built with the DSL (`Grid(shape, extent)` with spacing (10, 12.5, 8); the iso update
`solve(m*u.dt2 - u.laplace + damp*u.dt, u.forward)`, the TTI update built like devito_b200/seismic/tti.py), the
white-noise levels and halo of tests/kernel_cases.py are written into `data_with_halo`, the operator is applied for
time 1..K, and every time slot, halo included, is compared with float64. Each case names the kernel variant it is
meant to exercise and asserts it through `b2_last_sweep_kernel`: a layout that silently falls back to another
kernel fails instead of passing vacuously. Tolerances: rel L-inf 1e-5 (iso), 1e-4 (TTI), receiver traces included.

Switches are set with monkeypatch; the library reads them per call.
"""
import functools
from types import SimpleNamespace

import numpy as np
import pytest

from helpers import rel_linf
import kernel_cases as KC

pytestmark = pytest.mark.gpu

PK = {'scalar': 'scalar', 'vp': 'vp', 'm': 'm'}


def _last_kernel():
    from devito_b200 import _lib
    return _lib.lib().b2_last_sweep_kernel().decode()


def _grid(shape):
    from devito_b200 import Grid
    return Grid(shape=shape, extent=tuple((n - 1) * h for n, h in zip(shape, KC.SPACING)))


def _function(name, grid, so, values):
    from devito_b200 import Function
    f = Function(name=name, grid=grid, space_order=so)
    f.data_with_halo[:] = values
    return f


@functools.lru_cache(maxsize=None)
def _iso_setup(so, param, shape=KC.SHAPE, box=None, interpolation=None):
    """(operator, u, rec, case, source tables); one operator per configuration, re-run for every variant."""
    from devito_b200 import Constant, Eq, Operator, SparseTimeFunction, TimeFunction, solve
    c = KC.iso_case(so, param, shape=shape, box=box)
    grid = _grid(shape)
    u = TimeFunction(name='u', grid=grid, time_order=2, space_order=so)
    damp = _function('damp', grid, so, c['damp'])
    kind, pv = c['param']
    if param == 'scalar':
        vp = Constant(name='vp', value=float(pv))
        m = 1 / vp ** 2
    elif kind == 'vp':
        vp = _function('vp', grid, so, pv)
        m = 1 / vp ** 2
    else:
        m = _function('m', grid, so, pv)
    eqs = [Eq(u.forward, solve(m * u.dt2 - u.laplace + damp * u.dt, u.forward))]
    rec, tables = None, None
    if interpolation is not None:
        coords = KC.sparse_coordinates(shape)
        tables = KC.sparse_tables(coords, interpolation, KC.K + 2)
        r = tables['r']
        src = SparseTimeFunction(name='src', grid=grid, npoint=len(coords), nt=KC.K + 2,
                                 interpolation=interpolation, r=r, coordinates=coords)
        src.data[:] = tables['data']
        rec = SparseTimeFunction(name='rec', grid=grid, npoint=len(coords), nt=KC.K + 2,
                                 interpolation=interpolation, r=r, coordinates=coords)
        dt = grid.stepping_dim.spacing
        eqs += src.inject(field=u.forward, expr=src * dt ** 2 / m) + rec.interpolate(expr=u)
    op = Operator(eqs)
    assert op.backend == 'cuda-sm90a'
    return op, u, rec, c, tables


@functools.lru_cache(maxsize=None)
def _tti_setup(so, arrays, box=None, shape=KC.SHAPE, seams=None):
    """(operator, (u, v), rec, case, source tables). With `seams` (see KC.sparse_coordinates) the sources are injected
    into u and v and the receivers sample u + v, as in devito_b200/seismic/tti.py (sinc from so = 8 on, else linear);
    without, the operator has no sparse terms and rec and the tables are None."""
    from devito_b200 import Constant, Eq, Operator, SparseTimeFunction, TimeFunction, solve, sqrt
    from devito_b200.seismic.tti import Gzz_centered
    c = KC.tti_case(so, arrays, shape=shape, box=box)
    grid = _grid(shape)
    u = TimeFunction(name='u', grid=grid, time_order=2, space_order=so)
    v = TimeFunction(name='v', grid=grid, time_order=2, space_order=so)
    damp = _function('damp', grid, so, c['damp'])
    P = {n: (_function(n, grid, so, x) if arrays else Constant(name=n, value=float(x)))
         for n, x in c['params'].items()}
    model = SimpleNamespace(theta=P['theta'], phi=P['phi'])
    m = 1 / (P['vp'] * P['vp'])
    gxx = u.laplace - Gzz_centered(model, u)
    gzz = Gzz_centered(model, v)
    sd, e2 = sqrt(1 + 2 * P['delta']), 1 + 2 * P['epsilon']
    eqs = [Eq(u.forward, solve(m * u.dt2 - (e2 * gxx + sd * gzz) + damp * u.dt, u.forward)),
           Eq(v.forward, solve(m * v.dt2 - (sd * gxx + gzz) + damp * v.dt, v.forward))]
    rec, tables = None, None
    if seams is not None:
        interpolation = 'sinc' if so >= 8 else 'linear'
        coords = KC.sparse_coordinates(shape, seams=seams)
        tables = KC.sparse_tables(coords, interpolation, KC.K + 2)
        sp = lambda n: SparseTimeFunction(name=n, grid=grid, npoint=len(coords), nt=KC.K + 2,
                                          interpolation=interpolation, r=tables['r'], coordinates=coords)
        src, rec = sp('src'), sp('rec')
        src.data[:] = tables['data']
        dt = grid.stepping_dim.spacing
        eqs += src.inject(field=(u.forward, v.forward), expr=src * dt ** 2 / m) + rec.interpolate(expr=u + v)
    op = Operator(eqs)
    assert op.backend == 'cuda-sm90a'
    return op, (u, v), rec, c, tables


@functools.lru_cache(maxsize=None)
def _reference(key):
    """float64 result of a configuration (shared by all its kernel variants)."""
    *_, c, tables = (_iso_setup if key[0] == 'iso' else _tti_setup)(*key[1:])
    rec = dict(tables, data=np.zeros_like(tables['data'])) if tables is not None else None
    return KC.reference(c, src=tables, rec=rec)


def _run(fields, c, op, expect, rec=None, **kw):
    for f, name in zip(fields, ('u', 'v')):
        f.data_with_halo[:] = c[name]
    if rec is not None:
        rec.data[:] = 0.0
    lo, hi = c['lo'], c['hi']
    bounds = dict(x_m=lo[0], x_M=hi[0], y_m=lo[1], y_M=hi[1], z_m=lo[2], z_M=hi[2])
    op.apply(time_m=1, time_M=KC.K, dt=c['dt'], **bounds, **kw)
    assert _last_kernel() == expect
    return [np.array(f.data_ro_with_halo) for f in fields]


def _check_iso(key, expect, **kw):
    op, u, rec, c, _ = _iso_setup(*key[1:])
    (got,) = _run([u], c, op, expect, rec=rec, **kw)
    (want,), traces = _reference(key)
    assert np.abs(got).max() > 0.5
    assert rel_linf(got, want) < KC.TOL['iso']
    if rec is not None:
        assert rel_linf(np.array(rec.data), traces) < KC.TOL['iso']        # atomics order: same bound


def _check_tti(key, expect, **kw):
    op, (u, v), rec, c, _ = _tti_setup(*key[1:])
    got = _run([u, v], c, op, expect, rec=rec, **kw)
    want, traces = _reference(key)
    for g, w in zip(got, want):
        assert rel_linf(g, w) < KC.TOL['tti']
    if rec is not None:
        assert np.abs(traces).max() > 0
        assert rel_linf(np.array(rec.data), traces) < KC.TOL['tti']


PARAMS = ['scalar', 'vp', 'm']


@pytest.mark.parametrize('param', PARAMS)
@pytest.mark.parametrize('so', [4, 8, 12, 16])
def test_iso_generic(so, param):
    _check_iso(('iso', so, param), 'iso_generic', kernel=1)


ISO_TMA = [pytest.param(so, param, lx, None, id=f'{so}-{param}-{lx}')
           for so in (4, 8, 12, 16) for param in PARAMS for lx in (None, '12')] + \
          [pytest.param(so, param, None, box, id=f'{so}-{param}-{box}')
           for so in (4, 8, 12, 16) for param in PARAMS for box in KC.ZTAIL]


@pytest.mark.parametrize('so,param,lx,box', ISO_TMA)
def test_iso_tma(so, param, lx, box, monkeypatch):
    """Default selection; B2_ISO_LX=12 cuts the 37 x-planes into four chunks, the last of one plane. The z-tail boxes
    (kernel_cases.ZTAIL) end every row in a partial float4 group, which the sweep stores point by point."""
    if lx:
        monkeypatch.setenv('B2_ISO_LX', lx)
    key = ('iso', so, param) if box is None else ('iso', so, param, KC.SHAPE, KC.ZTAIL[box])
    _check_iso(key, f'iso_tma<{so // 2},{PK[param]}>')


MULTI_TILE = [(8, 'scalar'), (8, 'vp'), (8, 'm'), (4, 'scalar'), (12, 'scalar'), (16, 'scalar')]
MULTI_GRIDS = {'multi': (KC.MULTI, None), 'multi_tail': (KC.MULTI, KC.MULTI_TAIL), 'exact': (KC.EXACT, None)}


@pytest.mark.parametrize('grid', list(MULTI_GRIDS))
@pytest.mark.parametrize('so,param', MULTI_TILE)
def test_iso_tma_several_tiles(so, param, grid, monkeypatch):
    """Grids that every tile configuration cuts into several yz-tiles (kernel_cases.MULTI: >= 2 in y and >= 3 in z,
    the last of each partial; with a z extent of 298 as well) or into full tiles only (EXACT), with B2_ISO_LX=5
    (x-chunks of five planes, the last partial on MULTI)."""
    monkeypatch.setenv('B2_ISO_LX', '5')
    shape, box = MULTI_GRIDS[grid]
    _check_iso(('iso', so, param, shape, box), f'iso_tma<{so // 2},{PK[param]}>')


@pytest.mark.parametrize('shape,box', [((37, 45, 67), None), (KC.SHAPE, ((0, 0, 3), (36, 44, 67)))],
                         ids=['nz67', 'zm3'])
def test_iso_fallback_to_generic(shape, box):
    """Layouts the TMA kernel does not take (nz % 4 != 0; z_m = 3) run the generic kernel, correctly."""
    _check_iso(('iso', 8, 'vp', shape, box), 'iso_generic')


def test_iso_sub_box():
    """An interior update box (x_m = 1, y_m = 2, z_m = 4, upper ends inside too): cells outside it keep their
    white noise, and the stencil still reads the halo in x and y."""
    _check_iso(('iso', 8, 'vp', KC.SHAPE, KC.SUBBOX), 'iso_tma<4,vp>')


@pytest.mark.parametrize('gate', list(KC.GATE))
@pytest.mark.parametrize('param', ['scalar', 'vp'])
@pytest.mark.parametrize('so', [4, 8])
def test_iso_size_gate(so, param, gate):
    """Boxes on either side of iso_plan_init's size gate (n[1] >= 8 and n[2] >= 16): n = (8, 8, 16) runs the TMA
    sweep, (8, 7, 16) and (8, 8, 12) the generic kernel."""
    expect = f'iso_tma<{so // 2},{PK[param]}>' if gate == 'gate_in' else 'iso_generic'
    _check_iso(('iso', so, param, KC.SHAPE, KC.GATE[gate]), expect)


@pytest.mark.parametrize('param', ['scalar', 'vp'])
@pytest.mark.parametrize('so', [4, 8, 12, 16])
def test_iso_one_x_plane(so, param):
    """x_m == x_M: the march primes 2R planes for a single output plane (z extent 59, a tail of 3)."""
    _check_iso(('iso', so, param, KC.SHAPE, KC.XPLANE), f'iso_tma<{so // 2},{PK[param]}>')


def _tti_fused_name(so, arrays):
    """the sweep the default selection runs on a layout the fused kernels take"""
    if arrays:
        return f'tti_arr_ct2<{so // 2}>'
    return 'tti_fused<2>' if so == 4 else 'tti_ws<pf1>'


@pytest.mark.parametrize('gate', list(KC.GATE))
@pytest.mark.parametrize('arrays', [False, True], ids=['scalar', 'arrays'])
@pytest.mark.parametrize('so', [4, 8])
def test_tti_size_gate(so, arrays, gate):
    """tti_plan_init's size gate: n = (8, 8, 16) runs the fused sweep, (8, 7, 16) and (8, 8, 12) the two-pass one."""
    expect = _tti_fused_name(so, arrays) if gate == 'gate_in' else 'tti_two_pass'
    _check_tti(('tti', so, arrays, KC.GATE[gate]), expect)


@pytest.mark.parametrize('arrays', [False, True], ids=['scalar', 'arrays'])
@pytest.mark.parametrize('so', [4, 8])
def test_tti_one_x_plane(so, arrays):
    _check_tti(('tti', so, arrays, KC.XPLANE), _tti_fused_name(so, arrays))


@pytest.mark.parametrize('arrays', [False, True], ids=['scalar', 'arrays'])
@pytest.mark.parametrize('so', [4, 8, 12, 16])
def test_tti_two_pass(so, arrays):
    _check_tti(('tti', so, arrays), 'tti_two_pass', kernel=1)


@pytest.mark.parametrize('so,switch,expect', [
    (4, None, 'tti_fused<2>'),
    (8, '2', 'tti_fused<4>'),
    (8, '3', 'tti_ws<pf1>'),
])
def test_tti_fused_scalar(so, switch, expect, monkeypatch):
    monkeypatch.setenv('B2_TTI_LX', '12')
    if switch is not None:
        monkeypatch.setenv('B2_TTI_KERNEL', switch)
    _check_tti(('tti', so, False), expect)


@pytest.mark.parametrize('name,env', [
    ('ct2', {}),
    ('hint0', {'B2_TTI_ARR_HINT': '0'}),
    # the library does not read these variables: each environment that once selected another array-parameter sweep,
    # alone or all together, still runs the default kernel
    ('stale_ct0', {'B2_TTI_ARR_CT': '0'}),
    ('stale_ct1', {'B2_TTI_ARR_CT': '1'}),
    ('stale_fused0', {'B2_TTI_ARR_FUSED': '0'}),
    ('stale', {'B2_TTI_ARR_CT': '0', 'B2_TTI_ARR_PREFETCH': '0', 'B2_TTI_ARR_FUSED': '0'}),
])
@pytest.mark.parametrize('so', [4, 8])
def test_tti_fused_arrays(so, name, env, monkeypatch):
    monkeypatch.setenv('B2_TTI_LX', '12')
    for k, val in env.items():
        monkeypatch.setenv(k, val)
    _check_tti(('tti', so, True), f'tti_arr_ct2<{so // 2}>')


@pytest.mark.parametrize('interpolation', ['linear', 'sinc'])
@pytest.mark.parametrize('param', ['vp', 'm'])
def test_sparse_faces_outside_and_shared_cells(param, interpolation):
    """Sources and receivers within one cell of every face, outside the domain (supports in the halo, or nowhere)
    and two in one cell (atomic deposits into the same cells)."""
    _check_iso(('iso', 8, param, KC.SHAPE, None, interpolation), f'iso_tma<4,{param}>')
