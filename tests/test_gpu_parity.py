"""Parity of the CUDA path against the oracle and the reference's golden vectors.

All tests call through the public API (`Operator.apply`, which crosses the C ABI in
include/b200stencil.h exactly once per call). Tolerances: BASELINE.json north_star —
L-inf relative error < 1e-5 isotropic, < 1e-4 TTI."""
import numpy as np
import pytest

from oracle import oracle as O
from helpers import load_golden, rel_linf, iso_problem

pytestmark = pytest.mark.gpu


def _solver(kind, so, n, nbl, tn, interpolation='linear', **kw):
    from devito_b200.seismic import (demo_model, setup_geometry, AcousticWaveSolver,
                                     AnisotropicWaveSolver)
    preset = 'constant-isotropic' if kind == 'iso' else 'constant-tti'
    model = demo_model(preset, spacing=(10., 10., 10.), shape=(n, n, n), nbl=nbl, space_order=so, **kw)
    geometry = setup_geometry(model, tn, interpolation=interpolation)
    cls = AcousticWaveSolver if kind == 'iso' else AnisotropicWaveSolver
    return model, geometry, cls(model, geometry, space_order=so)


@pytest.mark.parametrize('name,so,interp', [('iso3d_so8', 8, 'linear'), ('iso3d_so12', 12, 'linear'),
                                            ('iso3d_so8_sinc', 8, 'sinc')])
@pytest.mark.parametrize('kernel', [1, 0])
def test_iso_vs_reference_golden(name, so, interp, kernel):
    g = load_golden(name)
    model, geometry, solver = _solver('iso', so, int(g['n']), int(g['nbl']), float(g['tn']), interp)
    assert solver.op_fwd().backend == 'cuda-sm90a'
    rec, u, summary = solver.forward(kernel=kernel)
    assert rel_linf(u.data, g['u']) < 1e-5
    assert rel_linf(rec.data, g['rec']) < 1e-5
    from devito_b200 import norm
    assert abs(float(norm(rec)) - float(g['norm_rec'])) < 1e-4 * float(g['norm_rec'])


def test_iso_array_vp_vs_reference_golden():
    g = load_golden('iso3d_so4_layers')
    from devito_b200.seismic import demo_model, setup_geometry, AcousticWaveSolver
    model = demo_model('layers-isotropic', spacing=(10., 10., 10.), shape=(20, 20, 20), nbl=8,
                       space_order=4, nlayers=3)
    assert rel_linf(model.vp.data, g['vp']) < 1e-6
    geometry = setup_geometry(model, float(g['tn']))
    solver = AcousticWaveSolver(model, geometry, space_order=4)
    rec, u, _ = solver.forward()
    assert rel_linf(u.data, g['u']) < 1e-5
    assert rel_linf(rec.data, g['rec']) < 1e-5


@pytest.mark.parametrize('name,so', [('tti3d_so8', 8), ('tti3d_so4', 4)])
@pytest.mark.parametrize('kernel', [1, 2])
def test_tti_vs_reference_golden(name, so, kernel):
    g = load_golden(name)
    model, geometry, solver = _solver('tti', so, int(g['n']), int(g['nbl']), float(g['tn']))
    assert solver.op_fwd().backend == 'cuda-sm90a'
    rec, u, v, _ = solver.forward(kernel=kernel)
    assert rel_linf(u.data, g['u']) < 1e-4
    assert rel_linf(v.data, g['v']) < 1e-4
    assert rel_linf(rec.data, g['rec']) < 1e-4


def test_kat2d_reference_known_answer():
    """tests/test_gpu_openacc.py:205-251 of the reference: norm(rec) = 490.56 +- 1e-2."""
    from devito_b200 import Grid, TimeFunction, Function, Eq, Operator, solve, norm
    from devito_b200.seismic import TimeAxis, RickerSource, Receiver
    shape, extent = (101, 101), (1000, 1000)
    v = np.empty(shape, dtype=np.float32)
    v[:, :51] = 1.5
    v[:, 51:] = 2.5
    grid = Grid(shape=shape, extent=extent, origin=(0., 0.))
    dt = 1.6
    time_range = TimeAxis(start=0., stop=1000., step=dt)
    src = RickerSource(name='src', grid=grid, f0=0.010, npoint=1, time_range=time_range)
    src.coordinates.data[0, :] = np.array(extent) * .5
    src.coordinates.data[0, -1] = 20.
    rec = Receiver(name='rec', grid=grid, npoint=101, time_range=time_range)
    rec.coordinates.data[:, 0] = np.linspace(0, extent[0], num=101)
    rec.coordinates.data[:, 1] = 20.
    u = TimeFunction(name="u", grid=grid, time_order=2, space_order=2)
    m = Function(name='m', grid=grid)
    m.data[:] = 1. / (v * v)
    stencil = Eq(u.forward, solve(m * u.dt2 - u.laplace, u.forward))
    src_term = src.inject(field=u.forward, expr=src * dt ** 2 / m)
    rec_term = rec.interpolate(expr=u.forward)
    op = Operator([stencil] + src_term + rec_term)
    assert op.backend == 'cuda-sm90a'
    op(time=time_range.num - 1, dt=dt)
    assert np.isclose(norm(rec), 490.56, atol=1e-2, rtol=0)
    g = load_golden('kat2d_so2')
    assert rel_linf(rec.data[::5, ::4], g['rec']) < 1e-4


@pytest.mark.parametrize('so,n,nbl', [(8, 56, 12), (12, 40, 10), (4, 32, 8), (16, 40, 8)])
def test_iso_tma_vs_oracle_larger(so, n, nbl):
    """TMA kernel vs the oracle at sizes that exercise several tiles, partial tiles in y and z,
    and several x-chunks."""
    p = iso_problem(n, nbl, so, 120.0)
    O.iso_forward(p['u'], so, p['w'], p['dt'], 1, p['nt'] - 2, damp=p['damp'], vp=1.5,
                  src=p['src'], rec=p['rec'])
    model, geometry, solver = _solver('iso', so, n, nbl, 120.0)
    rec, u, _ = solver.forward(kernel=2)
    assert rel_linf(u.data_with_halo, p['u']) < 1e-5
    assert rel_linf(rec.data, p['rec']['data']) < 1e-5


@pytest.mark.parametrize('so,n,nbl', [(8, 72, 12), (4, 60, 10)])
def test_tti_fused_vs_oracle_larger(so, n, nbl):
    """Fused TTI kernel vs the oracle with several tiles / partial tiles / several x-chunks."""
    import os
    p = iso_problem(n, nbl, so, 100.0)
    eps, delta, theta, phi = 0.3, 0.2, 0.7, 0.35
    dt = float(O.critical_dt(so, 3, 10.0, 1.5, eps_max=eps))
    nt, tv = O.time_axis(0.0, 100.0, dt)
    src = dict(p['src'], data=O.ricker(0.010, tv).astype(np.float32).reshape(-1, 1))
    rec = dict(p['rec'], data=np.zeros((nt, n * n), dtype=np.float32))
    u = np.zeros_like(p['u'])
    v = np.zeros_like(p['u'])
    w1 = [O.fd1_half_weights(so, 10.0)] * 3
    O.tti_forward(u, v, so, p['w'], w1, dt, 1, nt - 2, p['damp'], 1.5, eps, delta, theta, phi, src=src, rec=rec)
    os.environ['B2_TTI_LX'] = '24'
    try:
        model, geometry, solver = _solver('tti', so, n, nbl, 100.0)
        r, uu, vv, _ = solver.forward(kernel=2)
    finally:
        del os.environ['B2_TTI_LX']
    assert rel_linf(uu.data_with_halo, u) < 1e-4
    assert rel_linf(vv.data_with_halo, v) < 1e-4
    assert rel_linf(r.data, rec['data']) < 1e-4


def test_host_staged_call_equals_resident_call():
    """The C-ABI call with host buffers (dmap == NULL: H2D/D2H inside the call, like the
    reference's per-apply copies) gives the same answer as the device-resident call."""
    model, geometry, solver = _solver('iso', 8, 32, 8, 100.0)
    rec1, u1, _ = solver.forward()
    rec2, u2, _ = solver.forward(resident=False)
    assert np.array_equal(np.asarray(u1.data), np.asarray(u2.data))
    assert np.array_equal(np.asarray(rec1.data), np.asarray(rec2.data))


def _last_call_streamed():
    import ctypes
    from devito_b200 import _lib
    prof = (ctypes.c_double * 5)()
    _lib.lib().b2_last_call_profile(prof)
    return prof[4] == 1.0


@pytest.mark.parametrize('dim', [0, 1])
@pytest.mark.parametrize('interp,so,W', [('linear', 8, 16), ('sinc', 8, 24), ('linear', 4, 16)])
def test_streamed_time_loop_equals_resident_call(interp, so, W, dim, monkeypatch):
    """Host-staged applies of large grids run the streamed time loop (uploads / downloads overlapped with a
    skewed sweep, b2_api_iso.cu::iso_forward_streamed). Forced here on a small grid with narrow chunks
    (several x-ranges cut through the source and receiver supports): the wavefield must be bit-identical to
    the resident call, the traces equal up to the summation order of the partial sums."""
    model, geometry, solver = _solver('iso', so, 40, 12, 130.0, interp)
    rec1, u1, _ = solver.forward()
    assert not _last_call_streamed()
    monkeypatch.setenv('B2_STREAM', '2')
    monkeypatch.setenv('B2_STREAM_W', str(W))
    monkeypatch.setenv('B2_STREAM_DIM', str(dim))          # 0: skewed along x (single device), 1: along y (decomposed runs)
    rec2, u2, _ = solver.forward(resident=False)
    assert _last_call_streamed()
    assert np.array_equal(np.asarray(u1.data_with_halo), np.asarray(u2.data_with_halo))
    assert rel_linf(rec2.data, rec1.data) < 1e-6
    # sub-ranges of the time axis (restart) and a trace that samples the updated level (rec_toff)
    from devito_b200 import TimeFunction
    u3 = TimeFunction(name='u', grid=model.grid, time_order=2, space_order=so)
    rec3 = geometry.rec
    mid = geometry.nt // 2
    solver.forward(u=u3, rec=rec3, time_m=1, time_M=mid, resident=False)
    assert _last_call_streamed()
    solver.forward(u=u3, rec=rec3, time_m=mid + 1, time_M=geometry.nt - 2, resident=False)
    assert np.array_equal(np.asarray(u1.data), np.asarray(u3.data))
    assert rel_linf(rec3.data, rec1.data) < 1e-6


def test_streamed_time_loop_array_velocity(monkeypatch):
    g = load_golden('iso3d_so4_layers')
    from devito_b200.seismic import demo_model, setup_geometry, AcousticWaveSolver
    model = demo_model('layers-isotropic', spacing=(10., 10., 10.), shape=(20, 20, 20), nbl=8,
                       space_order=4, nlayers=3)
    solver = AcousticWaveSolver(model, setup_geometry(model, float(g['tn'])), space_order=4)
    monkeypatch.setenv('B2_STREAM', '2')
    monkeypatch.setenv('B2_STREAM_W', '12')
    rec, u, _ = solver.forward(resident=False)
    assert _last_call_streamed()
    assert rel_linf(u.data, g['u']) < 1e-5
    assert rel_linf(rec.data, g['rec']) < 1e-5


def test_restart_on_time_subranges():
    """Second caller of the C ABI in the reference (checkpointing/checkpoint.py:30-46): the loop
    must be restartable on arbitrary [time_m, time_M] sub-ranges."""
    model, geometry, solver = _solver('iso', 8, 32, 8, 120.0)
    rec1, u1, _ = solver.forward()
    from devito_b200 import TimeFunction
    u2 = TimeFunction(name='u', grid=model.grid, time_order=2, space_order=8)
    rec2 = geometry.rec
    nt = geometry.nt
    mid = nt // 2
    solver.forward(u=u2, rec=rec2, time_m=1, time_M=mid)
    solver.forward(u=u2, rec=rec2, time_m=mid + 1, time_M=nt - 2)
    assert np.array_equal(np.asarray(u1.data), np.asarray(u2.data))
    assert np.array_equal(np.asarray(rec1.data), np.asarray(rec2.data))


def test_linearity_large():
    """Size-independent property at a larger grid: the propagator is linear in the source."""
    model, geometry, solver = _solver('iso', 8, 104, 12, 60.0)
    src = geometry.src
    rec1, u1, _ = solver.forward(src=src)
    src2 = geometry.src
    src2.data[:] = 2.5 * src.data
    rec2, u2, _ = solver.forward(src=src2)
    assert rel_linf(2.5 * np.asarray(u1.data), u2.data) < 1e-5
    assert np.all(np.isfinite(u2.data))


def test_error_code_on_nan():
    """Return code 100 -> ExecutionError (devito/passes/iet/errors.py:192-198; operator.py:734-772)."""
    from devito_b200 import ExecutionError
    model, geometry, solver = _solver('iso', 8, 24, 6, 50.0)
    src = geometry.src
    src.data[3, 0] = np.nan
    with pytest.raises(ExecutionError):
        solver.forward(src=src, errctl=1)


def test_adjoint_vs_reference_golden_and_dot_product():
    """Adjoint operator (SURVEY §8f rank 1; acoustic/operators.py:153-187) on the same kernels run
    backward in time; plus the reference's adjoint identity <A x, y> = <x, A^T y>
    (tests/test_adjoint.py:21-121, there in float64 with 1e-11; float32 here)."""
    from devito_b200 import norm, inner
    g = load_golden('adj3d_so8')
    model, geometry, solver = _solver('iso', 8, int(g['n']), int(g['nbl']), float(g['tn']))
    assert solver.op_adj().backend == 'cuda-sm90a'
    rec, u, _ = solver.forward()
    srca, v, _ = solver.adjoint(rec)
    assert rel_linf(v.data, g['v']) < 1e-4          # atomics order, see tests/test_oracle_golden.py
    assert rel_linf(srca.data, g['srca']) < 1e-4
    src = geometry.src
    term1 = float(np.sum(np.asarray(srca.data, dtype=np.float64) * np.asarray(src.data, dtype=np.float64)))
    term2 = float(np.sum(np.asarray(rec.data, dtype=np.float64) ** 2))
    assert abs(term1 - term2) / abs(term2) < 1e-4


def test_tti_array_parameters_vs_reference_golden():
    """Preset `layers-tti` (vp, epsilon, delta, theta, phi arrays; SURVEY §8a a2, 48 B/point variant)."""
    g = load_golden('tti3d_so4_layers')
    from devito_b200.seismic import demo_model, setup_geometry, AnisotropicWaveSolver
    model = demo_model('layers-tti', spacing=(10., 10., 10.), shape=(20, 20, 20), nbl=8, space_order=4,
                       nlayers=3)
    geometry = setup_geometry(model, float(g['tn']))
    solver = AnisotropicWaveSolver(model, geometry, space_order=4)
    assert solver.op_fwd().backend == 'cuda-sm90a'
    rec, u, v, _ = solver.forward()
    assert rel_linf(u.data, g['u']) < 1e-4
    assert rel_linf(v.data, g['v']) < 1e-4
    assert rel_linf(rec.data, g['rec']) < 1e-4


@pytest.mark.parametrize('kernel', [0, 1])
def test_tti_array_parameters_varying_along_every_axis_vs_reference_golden(kernel):
    """The reference's own run with vp / epsilon / delta / theta / phi varying along x, y and z (fixture
    `tti3d_so8_varying`, oracle/make_golden.py::tti_varying): single-pass kernel with the TMA-staged factor tiles
    (kernel=0, the default) and the two-pass generic kernels (kernel=1)."""
    from helpers import varying_tti_parameters
    from devito_b200.seismic import SeismicModel, setup_geometry, AnisotropicWaveSolver
    g = load_golden('tti3d_so8_varying')
    n, nbl = int(g['n']), int(g['nbl'])
    model = SeismicModel(space_order=8, origin=(0., 0., 0.), shape=(n, n, n), dtype=np.float32,
                         spacing=(10., 10., 10.), nbl=nbl, bcs="damp", **varying_tti_parameters(n))
    assert np.float32(model.critical_dt) == g['dt']
    geometry = setup_geometry(model, float(g['tn']))
    assert geometry.nt == int(g['nt'])
    solver = AnisotropicWaveSolver(model, geometry, space_order=8)
    assert solver.op_fwd().backend == 'cuda-sm90a'
    rec, u, v, _ = solver.forward(kernel=kernel)
    slot = int(g['slot'])
    assert rel_linf(u.data[slot], g['u_last']) < 1e-4
    assert rel_linf(v.data[slot], g['v_last']) < 1e-4
    assert rel_linf(rec.data, g['rec']) < 1e-4


@pytest.mark.parametrize('so,shape,nbl', [(8, (40, 52, 72), 10), (4, (44, 40, 60), 8)])
def test_tti_array_parameters_fused_vs_two_pass(so, shape, nbl):
    """`layers-tti` through the single-pass kernel (k_tti_fused<.., ARR>: per-point rotation factors read from the
    tables at the Gz point and at the shifted point) against the two-pass generic kernels, which the reference golden
    above pins: several tiles, partial tiles in y and z, several x-chunks."""
    import os
    from devito_b200.seismic import SeismicModel, setup_geometry, AnisotropicWaveSolver
    # parameters varying along every axis (the layered preset varies along z only and would not see a factor sampled
    # at the wrong x- or y-shifted point)
    gx, gy, gz = np.meshgrid(*[np.linspace(0., 1., n, dtype=np.float32) for n in shape], indexing='ij')
    v = (1.5 + 0.6 * gx + 0.5 * gy + 0.9 * gz).astype(np.float32)
    model = SeismicModel(space_order=so, vp=v, origin=(0., 0., 0.), shape=shape, dtype=np.float32,
                         spacing=(10., 10., 10.), nbl=nbl, epsilon=(0.25 * gx * gz + 0.05).astype(np.float32),
                         delta=(0.12 * gy + 0.02).astype(np.float32),
                         theta=(0.2 + 0.9 * gx * gy + 0.3 * gz).astype(np.float32),
                         phi=(0.1 + 0.8 * gy * gz - 0.4 * gx).astype(np.float32), bcs="damp")
    geometry = setup_geometry(model, 90.0)
    solver = AnisotropicWaveSolver(model, geometry, space_order=so)
    r1, u1, v1, _ = solver.forward(kernel=1)
    os.environ['B2_TTI_LX'] = '24'
    try:
        r2, u2, v2, _ = solver.forward(kernel=2)
    finally:
        del os.environ['B2_TTI_LX']
    assert float(np.max(np.abs(u1.data))) > 0
    assert rel_linf(u2.data_with_halo, u1.data_with_halo) < 1e-4
    assert rel_linf(v2.data_with_halo, v1.data_with_halo) < 1e-4
    assert rel_linf(r2.data, r1.data) < 1e-4


def test_saved_wavefield():
    """`save=nt` (time slot == time index, no modulo): the saved history ends with the same three
    time levels as the buffered run."""
    from devito_b200 import TimeFunction
    model, geometry, solver = _solver('iso', 8, 24, 8, 100.0)
    rec1, u1, _ = solver.forward()
    rec2, u2, _ = solver.forward(save=True)
    nt = geometry.nt
    assert u2.data.shape[0] == nt
    for t in range(nt - 3, nt):
        assert np.array_equal(np.asarray(u2.data[t]), np.asarray(u1.data[t % 3]))
    assert np.array_equal(np.asarray(rec1.data), np.asarray(rec2.data))


def test_gradient_vs_reference_golden():
    """Gradient operator (SURVEY §8f rank 1; acoustic/operators.py:190-232): saved forward wavefield,
    adjoint propagation of the data, imaging condition grad -= u * v.dt2."""
    from devito_b200 import norm
    g = load_golden('grad3d_so8')
    model, geometry, solver = _solver('iso', 8, int(g['n']), int(g['nbl']), float(g['tn']))
    assert solver.op_grad().backend == 'cuda-sm90a'
    rec, u, _ = solver.forward(save=True)
    assert rel_linf(u.data[geometry.nt - 1], g['u_last']) < 1e-5
    grad, _ = solver.jacobian_adjoint(rec, u)
    assert rel_linf(grad.data, g['grad']) < 1e-4
    assert abs(float(norm(grad)) - float(g['norm_grad'])) < 1e-4 * float(g['norm_grad'])
