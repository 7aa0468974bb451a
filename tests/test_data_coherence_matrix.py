"""Sequences of applies with views of the data kept by the caller, against float64 runs of what the caller intended.

Dense arrays stay on the device between applies; a view the caller took before the first apply and keeps to the end
must see what every apply wrote, and every write through it must reach the next apply (tests/test_data_coherence.py
checks the storage protocol on the CPU). Sequences:
  - shot loop: three shots, each resetting the wavefields through a kept `data_with_halo` view (zeros or new noise),
    moving the sources, writing their traces through a kept `src.data` view; the kept wavefield and `rec.data` views
    against float64 after every shot;
  - model update: parameters and damping written through kept views between applies, with `dt` passed explicitly
    (against float64) and with the solvers' default `dt` (which must be the recomputed `critical_dt`);
  - read back: kept views of every array an apply writes (u, v, a saved wavefield, grad, snapshots, Born U, the SA
    wavefield, the generic update's field) equal a fresh accessor bit for bit after the apply, and float64;
  - alternation: resident, host-staged (`resident=False`) and NumPy-interpreter applies on the same fields, written
    through kept views between them;
  - no view held: two resident applies make no host <-> device copy of any dense array.
Inputs are the white-noise cases of tests/kernel_cases.py (anisotropic spacing, non-cubic grid), references
tests/ref64.py, tests/sa_ref.py and tests/linear_cases.py. Tolerances: rel L-inf 1e-5 (iso, SA), 1e-4 (TTI; Born U,
its traces and grad as in tests/test_scheme_matrix.py). Each row asserts the sweep kernel that ran.
"""
import numpy as np
import pytest
from types import SimpleNamespace

from helpers import rel_linf
import kernel_cases as KC
import linear_cases as LC
import ref64
import sa_ref as SA
import test_iso_two_level_matrix as TIL
import test_sa_matrix as TSA
import test_scheme_matrix as TSM
from test_ref64 import OUT_TOL

pytestmark = pytest.mark.gpu

SO = 8


def _kernel():
    from devito_b200 import _lib
    return _lib.lib().b2_last_sweep_kernel().decode()


def _grid(shape=KC.SHAPE):
    from devito_b200 import Grid
    return Grid(shape=shape, extent=tuple((n - 1) * h for n, h in zip(shape, KC.SPACING)))


def _function(name, grid, values):
    from devito_b200 import Function
    f = Function(name=name, grid=grid, space_order=SO)
    f.data_with_halo[:] = values
    return f


def _sparse(grid, name, coords, interpolation, r):
    from devito_b200 import SparseTimeFunction
    return SparseTimeFunction(name=name, grid=grid, npoint=len(coords), nt=KC.K + 2, interpolation=interpolation,
                              r=r, coordinates=coords)


def _tables(kind, coords, data):
    if kind == 'sa':
        t = TSA.sparse_tables(coords, 'sinc', KC.K + 2, KC.SPACING)
    else:
        t = KC.sparse_tables(coords, 'sinc', KC.K + 2)
    return dict(t, data=np.asarray(data, dtype=np.float32))


def _build(kind):
    """A fresh operator, its fields and array parameters, sources (sinc, so = 8) injected and receivers sampled on the
    KC points; `ref(u0s, params, src traces, src coordinates)` runs the same K steps in float64."""
    from devito_b200 import Constant, Eq, Operator, TimeFunction, solve, sqrt
    grid = _grid()
    coords = KC.sparse_coordinates()
    src, rec = _sparse(grid, 'src', coords, 'sinc', 4), _sparse(grid, 'rec', coords, 'sinc', 4)
    dt = grid.stepping_dim.spacing
    u = TimeFunction(name='u', grid=grid, time_order=2, space_order=SO)
    if kind.startswith('iso'):
        param = kind.split('-')[1]
        c = KC.iso_case(SO, param)
        damp = _function('damp', grid, c['damp'])
        pname, pv = c['param']
        P = {} if param == 'scalar' else {pname: _function(pname, grid, pv)}
        m = 1 / Constant(name='vp', value=float(pv)) ** 2 if param == 'scalar' else \
            (1 / P['vp'] ** 2 if param == 'vp' else P['m'])
        eqs = [Eq(u.forward, solve(m * u.dt2 - u.laplace + damp * u.dt, u.forward))]
        eqs += src.inject(field=u.forward, expr=src * dt ** 2 / m) + rec.interpolate(expr=u)
        fields, tol, expect, dtv = [u], KC.TOL['iso'], f'iso_tma<{SO // 2},{param}>', c['dt']
        w64, _ = KC.weights('iso', SO)

        def ref(u0s, p, traces, xy, d):
            pp = ('vp', np.float32(pv)) if param == 'scalar' else (pname, p[pname])
            rec_t = _tables(kind, coords, np.zeros_like(traces))
            uu, tr = ref64.iso_forward(u0s[0], SO, w64, dtv, 1, KC.K, damp=d, param=pp,
                                       src=_tables(kind, xy, traces), rec=rec_t)
            return [uu], tr
    elif kind == 'tti':
        from devito_b200.seismic.tti import Gzz_centered
        c = KC.tti_case(SO, True)
        v = TimeFunction(name='v', grid=grid, time_order=2, space_order=SO)
        damp = _function('damp', grid, c['damp'])
        P = {n: _function(n, grid, x) for n, x in c['params'].items()}
        m = 1 / (P['vp'] * P['vp'])
        gxx = u.laplace - Gzz_centered(SimpleNamespace(theta=P['theta'], phi=P['phi']), u)
        gzz = Gzz_centered(SimpleNamespace(theta=P['theta'], phi=P['phi']), v)
        sd, e2 = sqrt(1 + 2 * P['delta']), 1 + 2 * P['epsilon']
        eqs = [Eq(u.forward, solve(m * u.dt2 - (e2 * gxx + sd * gzz) + damp * u.dt, u.forward)),
               Eq(v.forward, solve(m * v.dt2 - (sd * gxx + gzz) + damp * v.dt, v.forward))]
        eqs += src.inject(field=(u.forward, v.forward), expr=src * dt ** 2 / m) + rec.interpolate(expr=u + v)
        fields, tol, expect, dtv = [u, v], KC.TOL['tti'], f'tti_arr_ct2<{SO // 2}>', c['dt']
        (w2, w1), _ = KC.weights('tti', SO)

        def ref(u0s, p, traces, xy, d):
            rec_t = _tables(kind, coords, np.zeros_like(traces))
            uu, vv, tr = ref64.tti_forward(u0s[0], u0s[1], SO, w2, w1, dtv, 1, KC.K, d, p,
                                           src=_tables(kind, xy, traces), rec=rec_t)
            return [uu, vv], tr
    else:
        from devito_b200.seismic.self_adjoint import iso_stencil
        c = TSA.sa_case(SO, True)
        P = {'vp': _function('vp', grid, c['vp']), 'b': _function('b', grid, c['b'])}
        damp = _function('damp', grid, c['w'])
        model = SimpleNamespace(vp=P['vp'], b=P['b'], damp=damp, grid=grid)
        eqs = iso_stencil(u, model, forward=True)
        eqs += src.inject(field=u.forward, expr=src * dt ** 2 * model.vp ** 2 / model.b) + rec.interpolate(expr=u)
        fields, tol, expect, dtv = [u], TSA.TOL, f'sa_tma<{SO // 2}>', TSA.DT
        weights = [SA.sa_weights(SO // 2, h) for h in KC.SPACING]

        def ref(u0s, p, traces, xy, d):
            rec_t = _tables(kind, coords, np.zeros_like(traces))
            uu, tr = SA.sa_forward(u0s[0], SO, weights, dtv, 1, KC.K, p['b'], p['vp'], d,
                                   src=_tables(kind, xy, traces), rec=rec_t)
            return [uu], tr
    op = Operator(eqs)
    assert op.backend == 'cuda-sm90a', getattr(op, '_why_not', None)
    src.data[:] = KC.sparse_tables(coords, 'sinc', KC.K + 2)['data']
    u0s = [c['u']] + ([c['v']] if kind == 'tti' else [])
    return SimpleNamespace(op=op, fields=fields, params=P, damp=damp, src=src, rec=rec, coords=coords, ref=ref,
                           tol=tol, expect=expect, dt=dtv, u0s=u0s)


# the sweep each kind runs: iso_tma<R, parameter>, the array-parameter TTI sweep, the self-adjoint TMA sweep
KINDS = ['iso-scalar', 'iso-vp', 'iso-m', 'tti', 'sa']


def _apply(k, **kw):
    k.op.apply(time_m=1, time_M=KC.K, dt=k.dt, **kw)
    assert _kernel() == k.expect


def _check(k, kept, kept_rec, want, want_tr):
    for view, f, w in zip(kept, k.fields, want):
        assert np.abs(view).max() > 0.1
        assert rel_linf(view, w) < k.tol
        assert np.array_equal(view, f.data_ro_with_halo)         # a kept view is a fresh accessor, bit for bit
    assert np.abs(want_tr).max() > 0
    assert rel_linf(kept_rec, want_tr) < k.tol
    assert np.array_equal(kept_rec, k.rec.data)


def _noise(shape, seed):
    return np.random.default_rng(seed).standard_normal(shape).astype(np.float32)


@pytest.mark.parametrize('kind', KINDS)
def test_shot_loop(kind):
    """Three shots: the wavefields reset through kept views (noise, zeros, noise), the sources moved and their traces
    written through a kept view, the kept wavefield and receiver views checked after each shot."""
    k = _build(kind)
    kept = [f.data_with_halo for f in k.fields]
    kept_src, kept_rec, xy = k.src.data, k.rec.data, k.src.coordinates.data
    params = {n: np.array(f.data_ro_with_halo) for n, f in k.params.items()}
    damp = np.array(k.damp.data_ro_with_halo)
    for shot in range(3):
        u0s = [np.zeros_like(u0) if shot == 1 else _noise(u0.shape, 40 + 2 * shot + i) for i, u0 in enumerate(k.u0s)]
        for view, u0 in zip(kept, u0s):
            view[...] = u0
        xy[...] = k.coords + np.float32(0.37 * shot) * np.asarray(KC.SPACING, dtype=np.float32)
        traces = _noise(kept_src.shape, 60 + shot)
        kept_src[...] = traces
        kept_rec[...] = 0.0
        _apply(k)
        want, want_tr = k.ref(u0s, params, traces, np.array(xy), damp)
        _check(k, kept, kept_rec, want, want_tr)


# parameters written through kept views between applies: new white noise within each parameter's range
UPDATES = {
    'iso-vp': {'vp': (1.6, 2.4)}, 'iso-m': {'m': (1 / 2.4 ** 2, 1 / 1.6 ** 2)},
    'tti': {'epsilon': (0.05, 0.3), 'theta': (0.1, 1.4)},
    'sa': {'b': (0.5, 1.1), 'vp': (1.6, 2.9)},
}


@pytest.mark.parametrize('kind', list(UPDATES))
def test_model_update_between_applies(kind):
    """Parameters and damping written through views kept from before the first apply; two applies, each against a
    float64 run with the values the caller wrote."""
    k = _build(kind)
    kept = [f.data_with_halo for f in k.fields]
    kept_p = {n: f.data_with_halo for n, f in k.params.items()}
    kept_damp, kept_rec = k.damp.data_with_halo, k.rec.data
    traces = np.array(k.src.data)
    for step in range(2):
        if step:
            rng = np.random.default_rng(70)
            for n, (lo, hi) in UPDATES[kind].items():
                kept_p[n][...] = rng.uniform(lo, hi, kept_p[n].shape).astype(np.float32)
            kept_damp[...] *= np.float32(0.5)
        for view, u0 in zip(kept, k.u0s):
            view[...] = u0
        kept_rec[...] = 0.0
        _apply(k)
        want, want_tr = k.ref(k.u0s, {n: np.array(v) for n, v in kept_p.items()}, traces, k.coords,
                              np.array(kept_damp))
        _check(k, kept, kept_rec, want, want_tr)


def _model(kind):
    from devito_b200.seismic import SeismicModel, AcquisitionGeometry
    from devito_b200.seismic import AcousticWaveSolver, AnisotropicWaveSolver, SaIsoAcousticWaveSolver
    shape = (29, 37, 44)
    rng = np.random.default_rng(80)
    vp = rng.uniform(1.5, 2.5, shape).astype(np.float32)
    extra = dict(epsilon=rng.uniform(0.05, 0.3, shape).astype(np.float32),
                 delta=rng.uniform(0.02, 0.15, shape).astype(np.float32),
                 theta=rng.uniform(0.2, 1.2, shape).astype(np.float32),
                 phi=rng.uniform(-0.6, 0.9, shape).astype(np.float32)) if kind == 'tti' else {}
    bcs = 'damp'
    if kind == 'sa':
        from devito_b200.seismic import setup_w_over_q
        extra = dict(b=rng.uniform(0.5, 1.1, shape).astype(np.float32))
        bcs = lambda f, nbl: setup_w_over_q(f, 2.0 * np.pi * 0.025, 0.1, 1000.0, nbl)
    model = SeismicModel(origin=(0., 0., 0.), spacing=KC.SPACING, shape=shape, space_order=SO, vp=vp, nbl=6,
                         bcs=bcs, **extra)
    dom = model.domain_size
    geometry = AcquisitionGeometry(model, np.array([[dom[0] * .4, y, dom[2] * .3] for y in np.linspace(0, dom[1], 7)]),
                                   np.array([[dom[0] * .5, dom[1] * .45, dom[2] * .5]]), t0=0.0, tn=60.0,
                                   src_type='Ricker', f0=0.025)
    solver = {'iso': AcousticWaveSolver, 'tti': AnisotropicWaveSolver,
              'sa': SaIsoAcousticWaveSolver}[kind](model, geometry, space_order=SO)
    return model, geometry, solver


def _fresh_cfl(model, vp, eps=None):
    """The CFL step of examples/seismic/model.py:353-382 from the values the caller holds (the self-adjoint solver
    scales it by its `dt_scale` of 0.5)"""
    from oracle import oracle as O
    return O.critical_dt(SO, 3, float(min(model.spacing)) * float(model.dt_scale),
                         float(np.max(np.asarray(vp, dtype=np.float64))),
                         eps_max=None if eps is None else float(np.max(np.asarray(eps, dtype=np.float64))))


@pytest.mark.parametrize('kind', ['iso', 'tti', 'sa'])
def test_default_dt_after_a_model_update(kind):
    """vp (and epsilon) written through kept views: the solver's default dt is the CFL step of the new values, and a
    forward at that default equals, bit for bit, one given that step explicitly (a stale step or stale parameters on
    the device would differ)."""
    from devito_b200 import TimeFunction
    model, geometry, solver = _model(kind)
    u = TimeFunction(name='u', grid=model.grid, time_order=2, space_order=SO)
    v = TimeFunction(name='v', grid=model.grid, time_order=2, space_order=SO) if kind == 'tti' else None
    fkw = dict(v=v) if kind == 'tti' else {}
    kept_u = [f.data_with_halo for f in (u, v) if f is not None]
    kept_vp = model.vp.data
    kept_eps = model.epsilon.data if kind == 'tti' else None
    kept_rec = geometry.rec.data
    solver.forward(u=u, **fkw)
    kept_vp[...] *= np.float32(1.25)
    if kept_eps is not None:
        kept_eps[...] += np.float32(0.1)
    want_dt = _fresh_cfl(model, kept_vp, kept_eps)
    assert solver.dt == want_dt
    outs = []
    for dt in (None, want_dt):
        for view in kept_u:
            view[...] = 0.0
        kw = dict(fkw) if dt is None else dict(fkw, dt=dt)
        solver.forward(u=u, **kw)
        assert _kernel() == {'iso': 'iso_tma<4,vp>', 'tti': 'tti_arr_ct2<4>', 'sa': 'sa_tma<4>'}[kind]
        assert np.abs(kept_u[0]).max() > 0
        outs.append([np.array(x) for x in kept_u] + [np.array(kept_rec)])
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


def _scheme(scheme, box=None):
    """A fresh operator of tests/test_scheme_matrix.py (never shared with that file's cached ones)."""
    return TSM._setup.__wrapped__(scheme, SO, 'vp', box, 0, 'sinc')


@pytest.mark.parametrize('scheme,expect', [('adjoint', 'iso_tma<4,vp>'), ('grad', 'iso_tma<4,vp>'),
                                           ('born', 'iso_tma<4,vp>'), ('snap', 'iso_tma<4,vp>')])
def test_read_back_of_every_written_array(scheme, expect):
    """Kept views of everything the apply writes (the wavefield, grad, Born U, the snapshots, the traces), taken and
    written before the first apply, over two applies."""
    op, roles, c, tables = _scheme(scheme, KC.SUBBOX if scheme == 'snap' else None)
    kept = {r: (f.data if r in ('rec', 'src') else f.data_with_halo) for r, f in roles.items()}
    bounds = {f'{a}_m': lo for a, lo in zip('xyz', c['lo'])}
    bounds.update({f'{a}_M': hi for a, hi in zip('xyz', c['hi'])})
    want = None
    for step in range(2):
        kept['u'][...] = c['u']
        kept['src'][...] = tables['data']
        for r in ('U', 'grad', 'snap'):
            if r in kept:
                kept[r][...] = c[r]
        if 'rec' in kept:
            kept['rec'][...] = 0.0
        op.apply(time_m=1, time_M=KC.K, dt=c['dt'], **bounds)
        assert _kernel() == expect
        if want is None:
            rec = dict(tables, data=np.zeros_like(tables['data'])) if 'rec' in roles else None
            want = KC.scheme_reference(c, src=tables, rec=rec)
        for r, w in want.items():
            if w is None:
                continue
            view = kept['rec' if r == 'traces' else r]
            tol = 1e-4 if scheme == 'born' and r == 'traces' else OUT_TOL[r]
            assert rel_linf(view, w) < tol, r
            f = roles['rec' if r == 'traces' else r]
            assert np.array_equal(view, f.data if r == 'traces' else f.data_ro_with_halo), r


def test_read_back_of_a_saved_wavefield():
    """`u` with save = K + 2 (what forward(save=True) allocates): a kept view of every time level against float64."""
    from devito_b200 import Eq, Operator, TimeFunction, solve
    c = KC.iso_case(SO, 'vp')
    grid = _grid()
    u = TimeFunction(name='u', grid=grid, time_order=2, space_order=SO, save=KC.K + 2)
    damp = _function('damp', grid, c['damp'])
    vp = _function('vp', grid, c['param'][1])
    op = Operator([Eq(u.forward, solve(u.dt2 / vp ** 2 - u.laplace + damp * u.dt, u.forward))])
    kept = u.data_with_halo
    w64, _ = KC.weights('iso', SO)
    for seed in (1, 2):
        u0 = np.zeros(kept.shape, dtype=np.float32)             # levels 0 and 1 given, the others zero (halo too)
        u0[:2] = _noise(c['u'][:2].shape, seed)
        kept[...] = u0
        op.apply(time_m=1, time_M=KC.K, dt=c['dt'])
        assert _kernel() == 'iso_tma<4,vp>'
        # the float64 run on K + 2 slots: level t in slot t, as in the saved array
        ref, _ = ref64.iso_forward(u0, SO, w64, c['dt'], 1, KC.K, damp=c['damp'], param=c['param'])
        for t in range(2, KC.K + 2):
            assert rel_linf(kept[t], ref[t]) < KC.TOL['iso'], t
        assert np.array_equal(kept[:2], u0[:2])
        assert np.array_equal(kept, u.data_ro_with_halo)


def test_read_back_of_the_generic_update():
    """`b2_linear_forward` (it reports no sweep kernel: its plan kind is asserted) with a kept view of its field,
    rewritten through that view before the second apply."""
    import test_linear_matrix as TLM
    m = next(x for x in LC.MATRIX if x[0] == 3 and x[3] == 'whole')
    c0 = LC.case(*m)
    op, f, _, _ = LC.build(c0)
    assert op._plan['kind'] == 'linear'
    kept = f.data_with_halo
    for seed in (0, 9):
        c = dict(c0, f=LC.case(*m, seed=seed)['f'])            # the operator's taps, new initial data
        kept[...] = c['f']
        TLM._apply(c, op)
        LC.check(c, np.array(kept), LC.reference(c))
        assert np.array_equal(kept, f.data_with_halo)


def test_two_level_pass_with_kept_views(monkeypatch):
    """The so = 8 two-level pass (forced with B2_ISO2=2, as tests/test_iso_two_level_matrix.py does) over two applies
    with u and damp written through views kept from before the first."""
    c = TIL._setup.__wrapped__()
    box = ((0, 0, 0), tuple(n - 1 for n in c.shape))
    kept_u, kept_d, kept_rec = c.u.data_with_halo, c.damp.data_with_halo, c.rec.data
    monkeypatch.setenv('B2_ISO2', '2')
    monkeypatch.setenv('B2_ISO_LX', str(TIL.LX))
    for seed in (1, 2):
        u0, d = TIL._noise_u(c.shape, box, seed), TIL._white_damp(c.shape, seed)
        kept_u[...] = u0
        kept_d[...] = d
        kept_rec[...] = 0.0
        c.op.apply(time_m=1, time_M=KC.K, dt=TIL.DT)
        assert _kernel() == TIL.TWO
        rec = dict(c.rtab, data=np.zeros_like(c.rtab['data']))
        want, traces = ref64.iso_forward(u0, TIL.SO, TIL.W64, TIL.DT, 1, KC.K, damp=d, param=('vp', 2.0),
                                         src=c.stab, rec=rec)
        assert rel_linf(kept_u, want) < KC.TOL['iso']
        assert rel_linf(kept_rec, traces) < KC.TOL['iso']
        assert np.array_equal(kept_u, c.u.data_ro_with_halo)


def test_alternating_resident_host_staged_and_interpreted_applies():
    """On the same fields with views kept throughout: a resident apply, a host-staged one, an operator the recogniser
    refuses (a nonlinear update, run by the NumPy interpreter) and a resident one again, each written through the
    kept views before it runs; the float64 state carried from call to call."""
    from devito_b200 import Eq, Operator
    k = _build('iso-vp')
    (u,) = k.fields
    kept_u, kept_vp, kept_rec = u.data_with_halo, k.params['vp'].data_with_halo, k.rec.data
    damp = np.array(k.damp.data_ro_with_halo)
    traces = np.array(k.src.data)
    square = Operator([Eq(u.forward, u * u)])
    assert square.backend == 'numpy-interpreter'
    kept_u[...] = k.u0s[0]
    state = k.u0s[0].astype(np.float64)
    dom = u._domain_slices()[1:]
    rng = np.random.default_rng(90)

    def iso(**kw):
        nonlocal state
        kept_rec[...] = 0.0
        _apply(k, **kw)
        want, want_tr = k.ref([state], {'vp': np.array(kept_vp)}, traces, k.coords, damp)
        _check(k, [kept_u], kept_rec, want, want_tr)
        state = want[0]

    iso()
    kept_u[0] *= np.float32(0.5)
    state[0] = kept_u[0].astype(np.float64)
    kept_vp[...] = rng.uniform(1.6, 2.4, kept_vp.shape).astype(np.float32)
    iso(resident=False)
    kept_u[1] = -kept_u[1]
    state[1] = -state[1]
    square.apply(time_m=1, time_M=1)
    want = state.copy()
    want[2][dom] = state[1][dom] ** 2
    assert rel_linf(kept_u, want) < KC.TOL['iso']
    assert np.array_equal(kept_u, u.data_ro_with_halo)
    state = np.array(kept_u, dtype=np.float64)
    kept_vp[...] = rng.uniform(1.6, 2.4, kept_vp.shape).astype(np.float32)
    kept_u[2] = 0.0
    state[2] = 0.0
    iso()


def _count_copies(monkeypatch):
    from devito_b200.types import FieldStorage
    counts = {'up': 0, 'down': 0}
    up, down = FieldStorage._upload, FieldStorage.sync_to_host

    def counted_up(self):
        counts['up'] += 1
        return up(self)

    def counted_down(self):
        counts['down'] += 1
        return down(self)
    monkeypatch.setattr(FieldStorage, '_upload', counted_up)
    monkeypatch.setattr(FieldStorage, 'sync_to_host', counted_down)
    return counts


@pytest.mark.parametrize('kind', KINDS + ['linear', 'solver-iso', 'solver-tti', 'solver-sa'])
def test_no_views_held_no_copies(kind, monkeypatch):
    """Two resident applies with no view kept copy nothing between host and device: u, damp and the parameters stay
    on the device (the resident path the benchmark times)."""
    if kind == 'linear':
        m = next(x for x in LC.MATRIX if x[0] == 3)
        c = LC.case(*m)
        op, f, _, _ = LC.build(c)
        import test_linear_matrix as TLM
        run = lambda: TLM._apply(c, op)
        arrays = [f]
    elif kind.startswith('solver'):
        from devito_b200 import TimeFunction
        model, _, solver = _model(kind.split('-')[1])
        u = TimeFunction(name='u', grid=model.grid, time_order=2, space_order=SO)
        fkw = dict(v=TimeFunction(name='v', grid=model.grid, time_order=2, space_order=SO)) if kind == 'solver-tti' \
            else {}

        def run():
            solver.forward(u=u, **fkw)
        arrays = [u] + list(fkw.values()) + [getattr(model, n) for n in ('vp', 'damp', 'epsilon', 'b')
                                             if hasattr(getattr(model, n, None), 'storage')]
    else:
        k = _build(kind)
        run = lambda: _apply(k)
        arrays = k.fields + [k.damp] + list(k.params.values())
    run()
    counts = _count_copies(monkeypatch)
    run()
    run()
    assert counts == {'up': 0, 'down': 0}
    for f in arrays:
        assert not f.storage.views_held()
