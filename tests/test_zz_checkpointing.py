"""The acoustic gradient with binomial checkpointing (`AcousticWaveSolver.jacobian_adjoint(checkpointing=True)`,
one call of b2_iso_gradient_revolve) against the saved-wavefield gradient (`forward(save=True)` + `jacobian_adjoint`).

The recomputed forward levels go through the same sweeps, in the same order, as the saved run's (restarts on time
sub-ranges are bitwise, tests/test_gpu_parity.py::test_restart_on_time_subranges), and the adjoint steps and the
imaging condition are the saved gradient's: the two gradients must agree bit for bit, whatever the number of
checkpoints. B2_ISO2=2 lets the two-level forward pass (k_iso_tma2) run on these small grids."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# (preset, space order, shape, nbl, forward sweep expected, adjoint sweep expected)
CASES = {
    'so8_constant': ('constant-isotropic', 8, (32, 36, 32), 8, 'iso_tma2<4,scalar>', 'iso_tma<4,scalar>'),
    'so8_layers': ('layers-isotropic', 8, (32, 36, 32), 8, 'iso_tma<4,vp>', 'iso_tma<4,vp>'),
    # z extent 19 + 2 * 6 + 2 * 4 = 39: not a multiple of 4, the one-thread-per-point kernel
    'so4_constant_unaligned': ('constant-isotropic', 4, (23, 21, 19), 6, 'iso_generic', 'iso_generic'),
    'so4_layers_unaligned': ('layers-isotropic', 4, (23, 21, 19), 6, 'iso_generic', 'iso_generic'),
}


def _solver(preset, so, shape, nbl, tn=80.0):
    from devito_b200.seismic import demo_model, setup_geometry, AcousticWaveSolver
    kw = {'nlayers': 3} if preset.startswith('layers') else {}
    model = demo_model(preset, spacing=(10., 10., 10.), shape=shape, nbl=nbl, space_order=so, **kw)
    geometry = setup_geometry(model, tn)
    return geometry, AcousticWaveSolver(model, geometry, space_order=so)


def _last_kernel():
    from devito_b200 import _lib
    return _lib.lib().b2_last_sweep_kernel().decode()


@pytest.fixture(scope='module')
def saved_gradients():
    """Per case: the solver, the data and the saved-wavefield gradient."""
    out = {}

    def get(name):
        if name not in out:
            preset, so, shape, nbl = CASES[name][:4]
            geometry, solver = _solver(preset, so, shape, nbl)
            rec, u, _ = solver.forward(save=True)
            grad, _ = solver.jacobian_adjoint(rec, u)
            assert np.abs(np.asarray(grad.data)).max() > 0
            out[name] = (geometry, solver, rec, np.array(grad.data))
        return out[name]
    return get


@pytest.mark.parametrize('case', sorted(CASES))
@pytest.mark.parametrize('nck', [1, 2, 3, 7, 'l'])
def test_checkpointed_gradient_is_bitwise_the_saved_one(case, nck, saved_gradients, monkeypatch):
    from devito_b200 import _lib
    monkeypatch.setenv('B2_ISO2', '2')
    geometry, solver, rec, want = saved_gradients(case)
    nsteps = rec.data.shape[0] - 2
    s = nsteps if nck == 'l' else nck
    grad, summary = solver.jacobian_adjoint(rec, checkpointing=True, n_checkpoints=s)
    fwd_k, adj_k = _last_kernel().split(';')
    # with a checkpoint per step every advance is one step: the two-level pass needs two
    want_fwd = 'iso_tma<4,scalar>' if CASES[case][4] == 'iso_tma2<4,scalar>' and s == nsteps else CASES[case][4]
    assert want_fwd in fwd_k.split(' '), fwd_k
    assert adj_k == CASES[case][5]
    assert np.array_equal(np.asarray(grad.data), want)
    assert _lib.lib().b2_staging_outstanding() == 0
    assert summary['section0'].time > 0


def test_default_number_of_checkpoints(saved_gradients):
    geometry, solver, rec, want = saved_gradients('so8_constant')
    grad, _ = solver.jacobian_adjoint(rec, checkpointing=True)
    assert np.array_equal(np.asarray(grad.data), want)


def test_staging_released_after_refused_and_failed_calls():
    """A schedule the library refuses (a reverse step whose forward level is not live) returns 210 and holds nothing;
    a call that stops after staging everything (NaN in the data, caught by the adjoint's NaN check) releases it."""
    import ctypes
    from devito_b200 import _lib, ExecutionError
    geometry, solver = _solver('constant-isotropic', 8, (32, 36, 32), 8)
    rec, _, _ = solver.forward()
    L = _lib.lib()
    c = solver._revolve_setup(rec, n_checkpoints=2)
    c.fwd.deviceid = c.grad.deviceid = c.dev
    acts = (ctypes.c_int * 3)(_lib.REVOLVE_ACTIONS['reverse'], c.args['time_M'], 0)
    assert L.b2_iso_gradient_revolve(ctypes.byref(c.fwd), ctypes.byref(c.grad), acts, 1, 2) == 210
    assert b'forward state' in L.b2_last_error()
    assert L.b2_staging_outstanding() == 0
    bad = geometry.rec
    bad.data[:] = np.asarray(rec.data)
    bad.data[-3, 0] = np.nan
    with pytest.raises(ExecutionError):
        solver.jacobian_adjoint(bad, checkpointing=True, n_checkpoints=2, errctl=1)
    assert L.b2_staging_outstanding() == 0


def test_nan_check_on_the_forward_steps():
    """A NaN in the source reaches u on the first advance; with errctl the forward steps' check stops the call (100)
    before any adjoint step, and the staging is released."""
    from devito_b200 import _lib, ExecutionError
    geometry, solver = _solver('constant-isotropic', 8, (32, 36, 32), 8)
    src = geometry.src
    src.data[3, 0] = np.nan
    with pytest.raises(ExecutionError, match='NaN/Inf detected in u '):
        solver.jacobian_adjoint(geometry.rec, src=src, checkpointing=True, n_checkpoints=2, errctl=1)
    assert _lib.lib().b2_staging_outstanding() == 0


def test_dot_product_float32():
    """<J dm, d> = <dm, J^T d> with J the Born operator (`jacobian`) and J^T the checkpointed gradient, around a
    constant background; float32, so 1e-4 as in the TTI dot tests."""
    from devito_b200.seismic import demo_model, setup_geometry, AcousticWaveSolver
    shape, spacing, nbl, so = (30, 34, 40), (10., 10., 10.), 10, 8
    model = demo_model('layers-isotropic', nlayers=2, vp_bottom=2., shape=shape, spacing=spacing, nbl=nbl,
                       space_order=so)
    model0 = demo_model('layers-isotropic', nlayers=2, vp_top=1.5, vp_bottom=1.5, shape=shape, spacing=spacing,
                        nbl=nbl, space_order=so, grid=model.grid)
    geometry = setup_geometry(model, 300.)
    solver = AcousticWaveSolver(model, geometry, space_order=so)
    dm = (np.asarray(model.vp.data, np.float64) ** -2 - np.asarray(model0.vp.data, np.float64) ** -2).astype(np.float32)
    assert np.abs(dm).max() > 0
    d = solver.jacobian(dm, model=model0)[0]
    im, _ = solver.jacobian_adjoint(d, checkpointing=True, n_checkpoints=5, model=model0)
    term1 = np.dot(np.asarray(im.data, np.float64).reshape(-1), dm.astype(np.float64).reshape(-1))
    term2 = np.sum(np.asarray(d.data, np.float64) ** 2)
    assert term2 > 0
    assert abs(term1 - term2) < 1e-4 * abs(term1), (term1, term2)
