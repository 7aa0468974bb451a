"""Second-order SLS viscoacoustic modelling (`ViscoacousticWaveSolver`, `b2_visco_forward`).

CPU: the float64 restatement (tests/visco_ref.py) against the reference's goldens (oracle/make_golden_visco.py), its
mutations and its dot test; the tables, the adjoint's mix and the point body of k_visco_generic emulated on the CPU; recognition of the solver's operators and the look-alikes the recogniser refuses; the
kernels and orders that are not on this path.
GPU: both goldens through `forward` / `adjoint` with both sweeps, a kernel matrix against float64, the reference's
test_adjoint_F in float32, split time ranges, the NaN check and the staging left behind.
"""
import ctypes
import functools
import os
import shutil
import subprocess

import numpy as np
import pytest

from helpers import load_golden, rel_linf
import visco_ref as VR
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDENS = ['visco3d_so8', 'visco2d_so8']
TOL = 1e-5
# the memory variable r is small next to p: the float64 restatement misses the reference's float32 last levels of r by
# up to 1.1e-5 (2-D, 222 steps), so the reference's own float32 rounding is of that size; r is held to 2e-5
TOL_R = 2e-5


def _model(shape, so, nbl, arrays=True, spacing=10.):
    from devito_b200.seismic import Model
    vp, b, qp = VR.smooth_vp_b_qp(shape)
    if not arrays:
        vp, b, qp = 1.8, 0.7, 40.0
    return Model(origin=(0.,) * len(shape), shape=shape, vp=vp, b=b, qp=qp, spacing=(spacing,) * len(shape),
                 nbl=nbl, space_order=so, bcs="mask", dtype=np.float32)


def _golden_solver(name):
    from devito_b200.seismic import ViscoacousticWaveSolver, setup_geometry
    g = load_golden(name)
    shape = tuple(int(x) for x in g['shape'])
    so = int(g['so'])
    model = _model(shape, so, int(g['nbl']))
    geometry = setup_geometry(model, float(g['tn']))
    solver = ViscoacousticWaveSolver(model, geometry, space_order=so)
    assert geometry.nt == int(g['nt']) and np.float32(solver.dt) == g['dt']
    return g, model, geometry, solver


def _sub(g, a):
    return np.asarray(a)[(slice(None, None, int(g['step'])),) * (a.ndim)]


def _reference64(model, geometry, dt, nt, src_data, rec_data, adjoint, so, lo=None, hi=None):
    """The float64 restatement of one forward (or adjoint) run of the solver's problem."""
    c = [VR.sa_weights(so // 2, h) for h in model.spacing]
    arr = lambda f: np.array(f.data_with_halo) if hasattr(f, 'data_with_halo') else float(f.data)
    B, V, Q, D = arr(model.b), arr(model.vp), arr(model.qp), np.array(model.damp.data_with_halo)
    gp, ws = geometry.src.tabulate()
    src = dict(gp=gp, w=ws, r=geometry.src.r, data=src_data)
    gp, ws = geometry.rec.tabulate()
    rec = dict(gp=gp, w=ws, r=geometry.rec.r, data=rec_data)
    z = np.zeros((3,) + D.shape)
    if adjoint:
        src, rec = dict(rec, data=rec_data), dict(src, data=np.zeros_like(src_data))
    else:
        rec = dict(rec, data=np.zeros_like(rec_data))
    return VR.visco_forward(z, z, so, c, dt, float(np.float32(geometry._f0)), 1, nt - 2, B, V, Q, D, lo=lo, hi=hi,
                            src=src, rec=rec, adjoint=adjoint)


@functools.lru_cache(maxsize=None)
def _golden_reference(name):
    g, model, geometry, solver = _golden_solver(name)
    so, nt, dt = int(g['so']), int(g['nt']), float(g['dt'])
    dom = lambda a: a[(slice(so, -so),) * (a.ndim)]
    p, r, tr = _reference64(model, geometry, dt, nt, g['src'], np.zeros_like(g['rec']), False, so)
    pa, ra, tra = _reference64(model, geometry, dt, nt, np.zeros_like(g['srca']), g['rec'], True, so)
    last = (nt - 1) % 3
    return g, dict(rec=tr, srca=tra, p=_sub(g, dom(p[last])), r=_sub(g, dom(r[last])), pa=_sub(g, dom(pa[0])),
                   ra=_sub(g, dom(ra[0])), damp=_sub(g, np.asarray(model.damp.data)))


# ---------------------------------------------------------------------------------------------------------------
# the float64 restatement
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', GOLDENS)
def test_float64_vs_reference_golden(name):
    g, got = _golden_reference(name)
    assert rel_linf(got['damp'], g['damp']) < 1e-6
    for k in ('rec', 'srca', 'p', 'pa'):
        assert rel_linf(got[k], g[k]) < TOL, k
    for k in ('r', 'ra'):
        assert rel_linf(got[k], g[k]) < TOL_R, k


def _noise_case(so, nd=3, seed=7):
    shape = (14, 15, 17)[:nd] if nd == 3 else (19, 23)
    alloc = tuple(n + 2 * so for n in shape)
    rng = np.random.default_rng(seed)
    c = dict(so=so, shape=shape, spacing=(10.0, 12.5, 8.0)[:nd])
    c['p'] = rng.standard_normal((3,) + alloc)
    c['r'] = 0.1 * rng.standard_normal((3,) + alloc)
    c['b'] = rng.uniform(0.4, 1.2, alloc)
    c['vp'] = rng.uniform(1.5, 3.0, alloc)
    c['qp'] = rng.uniform(5.0, 60.0, alloc)
    c['damp'] = rng.uniform(0.7, 1.0, alloc)
    c['c'] = [VR.sa_weights(so // 2, h) for h in c['spacing']]
    return c


@pytest.mark.parametrize('adjoint', [False, True], ids=['fwd', 'adj'])
@pytest.mark.parametrize('mut', sorted(VR.MUTATIONS))
def test_mutations_move_the_result(mut, adjoint):
    """Every mutation moves p by more than 100x the GPU tolerance on the white-noise case."""
    if adjoint and mut in ('tt_ts_swap',):
        pytest.skip("the adjoint's memory variable does not carry the swapped factor into p in three steps")
    c = _noise_case(8)
    args = (c['p'], c['r'], 8, c['c'], 0.9, 0.01, 1, 3, c['b'], c['vp'], c['qp'], c['damp'])
    ref, _, _ = VR.visco_forward(*args, adjoint=adjoint)
    bad, _, _ = VR.visco_forward(*args, adjoint=adjoint, mut=mut)
    assert rel_linf(bad, ref) > 100 * TOL, mut


def _interior_sparse(shape, spacing, nt, npoint, seed):
    rng = np.random.default_rng(seed)
    coords = rng.uniform(3, np.array(shape) - 4, size=(npoint, len(shape))) * np.array(spacing)
    gp, ws = O.tabulate(coords, (0.0,) * len(shape), spacing, 1, 'linear', dtype=np.float64)
    return dict(data=rng.standard_normal((nt, npoint)), gp=gp, w=ws, r=1)


@pytest.mark.parametrize('nd', [2, 3])
@pytest.mark.parametrize('so', [4, 8])
def test_float64_dot_test(so, nd):
    """<F s, d> = <s, F^T d>: the forward run from zero fields with source traces s, sampled by the receivers, and
    the adjoint run with receiver traces d, sampled at the sources, with variable b, vp and qp and no absorbing
    layer (damp = 1): the reference's mask multiplies the solved updates, which the transpose does not reproduce
    term by term."""
    c = _noise_case(so, nd)
    c['damp'] = np.ones_like(c['damp'])
    nt = 30
    s = _interior_sparse(c['shape'], c['spacing'], nt, 3, 1)
    d = _interior_sparse(c['shape'], c['spacing'], nt, 4, 2)
    z = np.zeros_like(c['p'])
    args = (so, c['c'], 0.5, 0.01, 1, nt - 2, c['b'], c['vp'], c['qp'], c['damp'])
    _, _, Fs = VR.visco_forward(z, z, *args, src=s, rec=dict(d, data=np.zeros_like(d['data'])))
    _, _, Ftd = VR.visco_forward(z, z, *args, src=d, rec=dict(s, data=np.zeros_like(s['data'])), adjoint=True)
    lhs = float(np.sum(Fs * d['data']))
    rhs = float(np.sum(s['data'] * Ftd))
    assert abs(lhs - rhs) / abs(lhs) < 1e-11


@pytest.fixture(scope='module')
def emu(tmp_path_factory):
    if shutil.which('nvcc') is None:
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp('emu') / 'libemu_visco.so'
    cmd = ['nvcc', '-O1', '-shared', '-Xcompiler', '-fPIC', '-I', os.path.join(ROOT, 'include'),
           '-I', os.path.join(ROOT, 'devito_b200', 'csrc'), os.path.join(ROOT, 'tests', 'support', 'emu_visco.cu'),
           '-o', str(out)]
    subprocess.run(cmd, check=True, capture_output=True)
    lib = ctypes.CDLL(str(out))
    lib.emu_visco_step.restype = ctypes.c_int
    return lib


@pytest.mark.parametrize('interior', [False, True], ids=['whole', 'interior'])
@pytest.mark.parametrize('adjoint', [False, True], ids=['fwd', 'adj'])
@pytest.mark.parametrize('nd', [2, 3])
@pytest.mark.parametrize('so', [4, 8])
def test_emulated_point_body(emu, so, nd, adjoint, interior):
    """The tables of k_visco_coef, the adjoint's mix and k_visco_generic's point body run on the CPU for one step
    against float64: p and r in the whole slot (outside the box they must stay as they were)."""
    c = _noise_case(so, nd)
    f32 = lambda x: np.ascontiguousarray(x, dtype=np.float32)
    p, r = f32(c['p']), f32(c['r'])
    b, vp, qp, damp = f32(c['b']), f32(c['vp']), f32(c['qp']), f32(c['damp'])
    dt, f0 = 0.9, 0.01
    if interior:
        lo = [1, 2, 4][:nd] if nd == 3 else [1, 4]
        hi = [n - 2 for n in c['shape']]
    else:
        lo, hi = [0] * nd, [n - 1 for n in c['shape']]
    t0, t1, t2 = (1, 0, 2) if adjoint else (1, 2, 0)
    p1, r1 = p[t1].copy(), r[t1].copy()
    a3 = (1,) * (3 - nd) + p.shape[1:]
    lo3 = [0] * (3 - nd) + lo
    n3 = [1] * (3 - nd) + [h - l + 1 for l, h in zip(lo, hi)]
    r3 = [0] * (3 - nd) + [so // 2] * nd
    cw = np.zeros((3, 8), dtype=np.float32)
    for d in range(nd):
        cw[3 - nd + d, :so // 2] = c['c'][d]
    ip = lambda x: (ctypes.c_int * 3)(*x)
    fp = lambda x: x.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    rc = emu.emu_visco_step(fp(p[t0]), fp(p[t2]), fp(p1), fp(r[t0]), fp(r1), fp(b), fp(vp), fp(qp), fp(damp),
                            ip(a3), ip(lo3), ip(n3), ip(r3), fp(cw), ctypes.c_int(so), ctypes.c_float(dt),
                            ctypes.c_float(f0), ctypes.c_int(int(adjoint)))
    assert rc == 0
    wp, wr, _ = VR.visco_forward(p, r, so, c['c'], dt, float(np.float32(f0)), 1, 1, b, vp, qp, damp, lo=lo, hi=hi,
                                 adjoint=adjoint)
    assert rel_linf(p1, wp[t1]) < 1e-5
    assert rel_linf(r1, wr[t1]) < 1e-5


# ---------------------------------------------------------------------------------------------------------------
# recognition
# ---------------------------------------------------------------------------------------------------------------
def _solver(shape=(21, 22, 24), so=8, arrays=True, nbl=6, tn=30.0):
    from devito_b200.seismic import ViscoacousticWaveSolver, setup_geometry
    model = _model(shape, so, nbl, arrays)
    return ViscoacousticWaveSolver(model, setup_geometry(model, tn), space_order=so)


@pytest.mark.parametrize('arrays', [True, False], ids=['arrays', 'scalars'])
@pytest.mark.parametrize('nd', [2, 3])
@pytest.mark.parametrize('so', [4, 8])
def test_solver_operators_are_recognised(so, nd, arrays):
    solver = _solver((21, 22, 24)[:nd], so, arrays)
    fwd, adj = solver.op_fwd(), solver.op_adj()
    for op in (fwd, adj):
        assert op.backend == 'cuda-sm90a', op._why_not
        p = op._plan
        assert p['kind'] == 'visco' and p['R'] == so // 2 and p['damp'].name == 'damp'
        assert (p['b_role'][1].name, p['vp_role'][1].name, p['qp_role'][1].name) == ('b', 'vp', 'qp')
        assert abs(p['f0'] - 0.010) < 1e-8
        assert 'b2_visco_forward' in str(op)
    assert not fwd._plan['adjoint'] and adj._plan['adjoint']
    assert (fwd._plan['src'].name, fwd._plan['rec'].name) == ('src', 'rec')
    assert (adj._plan['src'].name, adj._plan['rec'].name) == ('rec', 'src')


def _lookalike(kind):
    """The solver's forward (or adjoint) pair with one mistake."""
    from devito_b200 import Eq, Operator, TimeFunction, solve, sqrt
    from devito_b200.seismic.viscoacoustic import _nested, _src_rec
    solver = _solver((13, 14, 16), 8, True, nbl=4, tn=20.0)
    model, geometry = solver.model, solver.geometry
    b, m, damp, qp = model.b, model.m, model.damp, model.qp
    f0 = geometry._f0
    t_s = (sqrt(1. + 1. / qp ** 2) - 1. / qp) / f0
    tt = 1. / (f0 ** 2 * t_s) / t_s - 1.
    rho = 1. / b
    p = TimeFunction(name='p', grid=model.grid, time_order=2, space_order=8)
    r = TimeFunction(name='r', grid=model.grid, time_order=2, space_order=8)
    dims = p.dimensions[1:]
    L = _nested(p, b, dims)
    if kind == 'b_at_output':
        L = 0
        for d, dn in zip(dims, ('dx', 'dy', 'dz')):
            L = L + b * getattr(getattr(p, dn)(x0=d + d.spacing / 2), dn)(x0=d - d.spacing / 2)
    if kind == 'b_half_node':
        L = 0
        for d, dn in zip(dims, ('dx', 'dy', 'dz')):
            bh = (b + b.subs({d: d + d.spacing})) / 2
            L = L + getattr(bh * getattr(p, dn)(x0=d + d.spacing / 2), dn)(x0=d - d.spacing / 2)
    rho_ = 1 if kind == 'no_rho' else rho
    a_, g_ = (1. / t_s, tt) if kind == 'tt_ts_swap' else (tt, 1. / t_s)
    pde_r = r.dt - a_ * g_ * rho_ * L + g_ * r
    rr = r if kind == 'r_at_t' else r.forward
    pde_p = m * p.dt2 - rho_ * (1. + tt) * L + rr + (1 - damp) * p.dt
    mask = (lambda x: x + damp - 1) if kind == 'damp_added' else (lambda x: damp * x)
    eqs = [Eq(r.forward, mask(solve(pde_r, r.forward))), Eq(p.forward, mask(solve(pde_p, p.forward)))]
    if kind == 'fwd_run_backward':
        # the forward combination assigned to the levels behind and run backward
        eqs = [Eq(r.backward, e.rhs) for e in eqs[:1]] + [Eq(p.backward, eqs[1].rhs)]
    return Operator(eqs + _src_rec(p, model, geometry, forward=kind != 'fwd_run_backward'))


LOOKALIKES = ['b_at_output', 'b_half_node', 'no_rho', 'tt_ts_swap', 'r_at_t', 'fwd_run_backward', 'damp_added']


def test_lookalike_builder_builds_the_scheme():
    assert _lookalike('ref').backend == 'cuda-sm90a'


@pytest.mark.parametrize('kind', LOOKALIKES)
def test_lookalikes_are_refused(kind):
    op = _lookalike(kind)
    assert op.backend == 'numpy-interpreter', kind


@pytest.mark.parametrize('kw', [dict(kernel='kv'), dict(kernel='maxwell'), dict(time_order=1)])
def test_other_kernels_raise(kw):
    from devito_b200.seismic import ViscoacousticWaveSolver, setup_geometry
    model = _model((11, 12), 4, 4)
    with pytest.raises(NotImplementedError, match="kernel='sls' with time_order=2"):
        ViscoacousticWaveSolver(model, setup_geometry(model, 10.), space_order=4, **kw)


def test_linearised_operators_raise():
    solver = _solver((11, 12), 4, nbl=4, tn=10.)
    for call in (lambda: solver.jacobian(None), lambda: solver.jacobian_adjoint(None, None)):
        with pytest.raises(NotImplementedError, match="kernel='sls' with time_order=2"):
            call()


def test_decomposed_grid_raises_invalid_argument():
    """The pair is recognised on a decomposed grid (only the grid's distributor says it is split), and preparing
    its arguments, the first thing an apply does after loading the library, raises InvalidArgument."""
    import types
    from devito_b200 import InvalidArgument
    solver = _solver((13, 14, 16), 8, True, nbl=4, tn=20.0)
    grid = solver.model.grid
    real = grid._distributor
    grid._distributor = types.SimpleNamespace(is_parallel=True)
    try:
        for op in (solver.op_fwd(), solver.op_adj()):
            assert op.backend == 'cuda-sm90a', op._why_not
            with pytest.raises(InvalidArgument, match='decomposed'):
                op.arguments(dt=solver.dt)
    finally:
        grid._distributor = real


def test_layers_viscoacoustic_preset():
    from devito_b200.seismic import demo_model
    m = demo_model('layers-viscoacoustic', shape=(30, 31), nbl=5, space_order=4)
    qp = np.asarray(m.qp.data)
    vp = np.asarray(m.vp.data)
    assert np.allclose(qp, 3.516 * (vp * 1000.) ** 2.2 * 1e-6, rtol=1e-5)
    assert np.allclose(np.asarray(m.b.data), 1 / (0.31 * (1e3 * vp) ** 0.25), rtol=1e-5)


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
def _last_kernel():
    from devito_b200 import _lib
    return _lib.lib().b2_last_sweep_kernel().decode()


@pytest.mark.gpu
@pytest.mark.parametrize('kernel', [1, 0], ids=['generic', 'auto'])
@pytest.mark.parametrize('name', GOLDENS)
def test_forward_and_adjoint_vs_reference_golden(name, kernel):
    g, model, geometry, solver = _golden_solver(name)
    nt = int(g['nt'])
    rec, p, _, _ = solver.forward(kernel=kernel)
    assert rel_linf(rec.data, g['rec']) < TOL
    assert rel_linf(_sub(g, np.asarray(p.data)[(nt - 1) % 3]), g['p']) < TOL
    rec.data[:] = g['rec']
    srca, pa, _, _ = solver.adjoint(rec, kernel=kernel)
    assert rel_linf(srca.data, g['srca']) < TOL
    assert rel_linf(_sub(g, np.asarray(pa.data)[0]), g['pa']) < TOL
    # the 3-D golden's layout takes the TMA sweep unless the generic kernel is asked for
    want = 'visco_tma<4>+adj' if name.startswith('visco3d') and kernel == 0 else 'visco_generic+adj'
    assert _last_kernel() == want


# (shape, so, arrays, kernel, variant): 3-D shapes whose allocated z extent is a multiple of 4 take the TMA sweep;
# with nbl=6 the (140, 38, 56) case is a 152 x 50 x 68 grid: three full and one partial 16-row y-tile, one full and
# one partial 64-column z-tile, and 152 x-planes make several x-chunks
MATRIX = [
    ((30, 20, 24), 8, True, 2, 'visco_tma<4>'),
    ((30, 20, 24), 8, False, 2, 'visco_tma<4>'),
    ((25, 21, 24), 4, True, 2, 'visco_tma<2>'),
    ((25, 21, 24), 4, False, 0, 'visco_tma<2>'),
    ((140, 38, 56), 8, True, 0, 'visco_tma<4>'),
    ((23, 19, 21), 8, True, 0, 'visco_generic'),
    ((20, 18, 22), 2, True, 0, 'visco_generic'),
    ((20, 18, 22), 16, False, 0, 'visco_generic'),
    ((41, 37), 8, True, 0, 'visco_generic'),
    ((41, 37), 2, False, 0, 'visco_generic'),
    ((41, 37), 16, True, 0, 'visco_generic'),
]


@pytest.mark.gpu
@pytest.mark.parametrize('interior', [False, True], ids=['whole', 'interior'])
@pytest.mark.parametrize('adjoint', [False, True], ids=['fwd', 'adj'])
@pytest.mark.parametrize('case', MATRIX, ids=lambda c: f"{'x'.join(map(str, c[0]))}-so{c[1]}-"
                         f"{'arr' if c[2] else 'scal'}-k{c[3]}")
def test_kernel_matrix_vs_float64(case, adjoint, interior):
    shape, so, arrays, kernel, variant = case
    if interior and shape == (140, 38, 56):
        pytest.skip("the large case runs on the whole box only")
    from devito_b200.seismic import ViscoacousticWaveSolver, setup_geometry
    nbl = 6
    model = _model(shape, so, nbl, arrays)
    geometry = setup_geometry(model, 24.0)
    solver = ViscoacousticWaveSolver(model, geometry, space_order=so)
    nt, dt = geometry.nt, float(np.float32(solver.dt))
    full = model.grid.shape
    kw, lo, hi = {}, None, None
    if interior:
        # a box that keeps the start of z 16-byte aligned (z_m a multiple of 4)
        lo = [3, 2, 4][:len(shape)] if len(shape) == 3 else [3, 4]
        hi = [n - 3 for n in full]
        for d, l_, h_ in zip(model.grid.dimensions, lo, hi):
            kw[d.min_name], kw[d.max_name] = l_, h_
    rng = np.random.default_rng(3)
    if not adjoint:
        src = geometry.src
        rec, p, _, _ = solver.forward(kernel=kernel, **kw)
        got_tr, got_p = np.asarray(rec.data), np.asarray(p.data_with_halo)[(nt - 1) % 3]
        want_p, _, want_tr = _reference64(model, geometry, dt, nt, np.asarray(src.data), np.zeros_like(rec.data),
                                          False, so, lo, hi)
        want_p = want_p[(nt - 1) % 3]
    else:
        rec = geometry.rec
        rec.data[:] = rng.standard_normal(rec.data.shape).astype(np.float32)
        srca, pa, _, _ = solver.adjoint(rec, kernel=kernel, **kw)
        got_tr, got_p = np.asarray(srca.data), np.asarray(pa.data_with_halo)[0]
        want_p, _, want_tr = _reference64(model, geometry, dt, nt, np.zeros_like(srca.data), np.asarray(rec.data),
                                          True, so, lo, hi)
        want_p = want_p[0]
    assert _last_kernel() == variant + ('+adj' if adjoint else '')
    assert rel_linf(got_tr, want_tr) < TOL
    assert rel_linf(got_p, want_p) < TOL


@pytest.mark.gpu
@pytest.mark.parametrize('shape,so,nlayers', [((20, 25), 4, 2), ((20, 25), 2, 2), ((20, 25, 20), 4, 2),
                                              ((20, 25, 20), 2, 2), ((71, 61), 8, 3), ((71, 61, 52), 8, 3)])
def test_adjoint_F_float32(shape, so, nlayers):
    """<r, F(s)> = <F^T(r), s> in float32 on the 'layers-viscoacoustic' preset (15 m spacing, 10 absorbing cells,
    tn = 500). The first four cases are those of the reference's test_adjoint_F for kernel='sls', time_order=2
    (tests/test_adjoint.py:57-65, there in float64 to 1e-11); the last two are larger grids at so=8, the order of the
    TMA sweep's golden."""
    from devito_b200.seismic import ViscoacousticWaveSolver, demo_model, setup_geometry
    model = demo_model('layers-viscoacoustic', shape=shape, spacing=(15.,) * len(shape), nbl=10, space_order=so,
                       nlayers=nlayers)
    geometry = setup_geometry(model, 500.)
    solver = ViscoacousticWaveSolver(model, geometry, space_order=so, kernel='sls', time_order=2)
    src1, rec1 = solver.geometry.src, solver.geometry.rec
    rec2, _, _, _ = solver.forward(src=src1)
    rec1.data[:] = rec2.data[:]
    src2, _, _, _ = solver.adjoint(rec=rec1)
    term1 = np.dot(src2.data.reshape(-1).astype(np.float64), src1.data.reshape(-1).astype(np.float64))
    term2 = np.dot(rec1.data.reshape(-1).astype(np.float64), rec2.data.reshape(-1).astype(np.float64))
    assert abs(term1 - term2) / abs(term1 + term2) < 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize('adjoint', [False, True], ids=['fwd', 'adj'])
def test_split_time_ranges_are_bitwise_one_call(adjoint):
    from devito_b200 import TimeFunction
    g, model, geometry, solver = _golden_solver('visco3d_so8')
    nt = geometry.nt
    mk = lambda n: TimeFunction(name=n, grid=model.grid, time_order=2, space_order=8)
    ranges = ((1, 30), (31, 31), (32, nt - 2))
    if not adjoint:
        rec_a, p_a, _, _ = solver.forward(p=mk('p'), r=mk('r'))
        rec_a, p_a = np.array(rec_a.data), np.array(p_a.data_with_halo)
        p, r, rec = mk('p'), mk('r'), geometry.rec
        for lo, hi in ranges:
            solver.forward(rec=rec, p=p, r=r, time_m=lo, time_M=hi)
        assert np.array_equal(np.array(rec.data), rec_a)
        assert np.array_equal(np.array(p.data_with_halo), p_a)
    else:
        rec = geometry.rec
        rec.data[:] = g['rec']
        s_a, pa_a, _, _ = solver.adjoint(rec, pa=mk('pa'), r=mk('r'))
        s_a, pa_a = np.array(s_a.data), np.array(pa_a.data_with_halo)
        pa, r, srca = mk('pa'), mk('r'), geometry.new_src(name='srca', src_type=None)
        for lo, hi in ranges[::-1]:
            solver.adjoint(rec, srca=srca, pa=pa, r=r, time_m=lo, time_M=hi)
        assert np.array_equal(np.array(srca.data), s_a)
        assert np.array_equal(np.array(pa.data_with_halo), pa_a)


@pytest.mark.gpu
def test_nan_is_caught_and_staging_released():
    """errctl finds a NaN written into p; a refused call (a forced TMA sweep on a 2-D grid) and the failed one leave
    no staging behind (host-staged arrays)."""
    from devito_b200 import ExecutionError, TimeFunction, _lib
    solver = _solver((20, 18, 24), 8, True, nbl=4, tn=30.0)
    model = solver.model
    L = _lib.lib()
    p = TimeFunction(name='p', grid=model.grid, time_order=2, space_order=8)
    p.data[1, 5, 5, 5] = np.nan
    with pytest.raises(ExecutionError, match='NaN'):
        solver.forward(p=p, errctl=1, resident=False)
    solver2 = _solver((31, 27), 8, True, nbl=4, tn=20.0)
    with pytest.raises(ExecutionError, match='210'):
        solver2.forward(kernel=2, resident=False)
    assert L.b2_staging_outstanding() == 0
    rec, p2, _, _ = solver.forward(resident=False)
    assert np.all(np.isfinite(np.asarray(p2.data)))
