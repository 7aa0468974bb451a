"""Binomial checkpointing without a GPU: the schedules of devito_b200/revolve.py on a toy propagator, the default
number of checkpoints, the two argument blocks `AcousticWaveSolver.jacobian_adjoint(checkpointing=True)` builds, and
the refusals of the solver and of the library's host-side checks (b2_revolve_check, and b2_iso_gradient_revolve's
argument checks, which run before it touches a device)."""
import ctypes

import numpy as np
import pytest

from devito_b200.revolve import schedule, optimal_forward_steps, repetitions, beta, default_n_checkpoints


def _simulate(l, s):
    """Runs the actions on a toy propagator whose state t is the integer t: returns the forward steps, the states the
    reverse steps saw, the most checkpoints live at once."""
    state, shots, steps, seen, live = 0, {}, 0, [], 0
    for act in schedule(l, s):
        if act[0] == 'advance':
            assert act[1] == state and act[2] > act[1]
            for _ in range(act[1], act[2]):
                state += 1
                steps += 1
        elif act[0] == 'takeshot':
            assert 0 <= act[1] < s and act[2] == state
            shots[act[1]] = state
        elif act[0] == 'restore':
            state = shots[act[1]]
        else:
            seen.append((act[1], state))
        live = max(live, len(shots))
    return steps, seen, live


@pytest.mark.parametrize('s', range(1, 9))
def test_schedule_on_a_toy_propagator(s):
    for l in range(1, 61):
        steps, seen, live = _simulate(l, s)
        assert [t for t, _ in seen] == list(range(l - 1, -1, -1))
        assert all(t == state for t, state in seen)
        assert live <= s
        r = repetitions(l, s)
        assert steps == optimal_forward_steps(l, s) == (r * l - beta(s + 1, r - 1) if l > 1 else 0), (l, s)


def test_repetitions_and_degenerate_schedule():
    assert (repetitions(254, 3), repetitions(254, 10), repetitions(998, 50)) == (10, 3, 2)
    # as many checkpoints as steps: checkpoint every state, never recompute
    steps, _, _ = _simulate(40, 40)
    assert steps == 39
    assert not any(a[0] == 'advance' and a[2] - a[1] > 1 for a in schedule(40, 60))
    with pytest.raises(ValueError):
        schedule(10, 0)


def test_default_number_of_checkpoints():
    slot = 528 ** 3 * 4
    assert default_n_checkpoints(1000, 40 * 2 ** 30, slot) == int(0.9 * 40 * 2 ** 30 // (2 * slot))
    assert default_n_checkpoints(5, 40 * 2 ** 30, slot) == 5
    assert default_n_checkpoints(100, slot, slot) == 0


def _solver(kernel='OT2', so=8):
    from devito_b200.seismic import demo_model, setup_geometry, AcousticWaveSolver
    model = demo_model('constant-isotropic', spacing=(10., 10., 10.), shape=(24, 24, 24), nbl=6, space_order=so)
    geometry = setup_geometry(model, 60.0)
    return geometry, AcousticWaveSolver(model, geometry, space_order=so, kernel=kernel)


def test_solver_builds_the_two_blocks():
    geometry, solver = _solver()
    assert solver.op_fwd(save=False).backend == 'cuda-sm90a'
    assert solver.op_grad(save=True).backend == 'cuda-sm90a'
    # a buffered saved field in the imaging condition is refused for a plain apply
    assert solver.op_grad(save=False).backend == 'numpy-interpreter'
    rec = geometry.rec
    c = solver._revolve_setup(rec, n_checkpoints=3, resident=False)
    assert ctypes.addressof(c.grad.usave.contents) == ctypes.addressof(c.fwd.u.contents)
    assert c.fwd.u.contents.size[0] == 3
    assert not c.fwd.rec and c.fwd.src and c.grad.src and c.grad.grad and not c.fwd.adjoint and c.grad.adjoint
    assert ctypes.addressof(c.grad.damp.contents) == ctypes.addressof(c.fwd.damp.contents)
    assert c.nsteps == rec.data.shape[0] - 2 == c.args['time_M'] - c.args['time_m'] + 1
    assert c.n_checkpoints == 3 and c.nactions == len(c.schedule)
    from devito_b200 import _lib
    L = _lib.load_library()
    acts = c.actions
    assert L.b2_revolve_check(acts, c.nactions, 3, c.fwd.time_m, c.fwd.time_M, c.grad.time_m, c.grad.time_M) == 0


def _refused(c, changes=None):
    from devito_b200 import _lib
    L = _lib.load_library()
    for (blk, name), val in (changes or {}).items():
        setattr(getattr(c, blk), name, val)
    rc = L.b2_iso_gradient_revolve(ctypes.byref(c.fwd), ctypes.byref(c.grad), c.actions, c.nactions, c.n_checkpoints)
    return rc, L.b2_last_error().decode()


@pytest.mark.parametrize('change,words', [
    ({('grad', 'ot4'): 1}, 'OT4'),
    ({('fwd', 'free_surface'): 1}, 'free surface'),
    ({('fwd', 'host_io'): 1}, 'host_io'),
    ({('grad', 'halo'): 'set'}, 'halo'),
    ({('fwd', 'ndim'): 2}, '3-D'),
    ({('grad', 'usave'): None}, 'usave'),
    ({('fwd', 'dt'): 0.5}, 'dt'),
    ({('grad', 'x_M'): 10}, 'box'),
    ({('grad', 'adjoint'): 0}, 'Gradient'),
])
def test_entry_point_refusals(change, words):
    geometry, solver = _solver()
    c = solver._revolve_setup(geometry.rec, n_checkpoints=2, resident=False)
    if ('grad', 'halo') in change:
        change = {('grad', 'halo'): 1}           # any non-NULL context is refused before it is used
    rc, msg = _refused(c, change)
    assert rc == 210 and words in msg, msg


def test_entry_point_refuses_born_snapshots_and_a_foreign_usave():
    from devito_b200 import _lib
    geometry, solver = _solver()
    c = solver._revolve_setup(geometry.rec, n_checkpoints=2, resident=False)
    for blk, member in (('fwd', 'born_U'), ('grad', 'snap')):
        setattr(getattr(c, blk), member, c.fwd.u)
        assert _refused(c)[0] == 210
        setattr(getattr(c, blk), member, None)
    other = _lib.make_dataobj(host=np.zeros((3, 4, 4, 4), np.float32))
    c.grad.usave = other.ptr
    rc, msg = _refused(c)
    assert rc == 210 and 'usave' in msg


def _check(acts, nck=2, tf=(1, 10), tg=(1, 10)):
    from devito_b200 import _lib
    L = _lib.load_library()
    flat = [x for a in acts for x in a]
    arr = (ctypes.c_int * max(len(flat), 1))(*flat)
    rc = L.b2_revolve_check(arr, len(acts), nck, tf[0], tf[1], tg[0], tg[1])
    return rc, L.b2_last_error().decode()


def test_action_list_refusals():
    A, T, R, V = 0, 1, 2, 3
    ok = [(T, 0, 1), (A, 1, 3), (V, 3, 0), (R, 0, 0), (A, 1, 2), (V, 2, 0), (V, 1, 0)]
    assert _check(ok, tf=(1, 10), tg=(1, 3))[0] == 0
    bad = {
        'advance beyond time_M': [(A, 1, 12)],
        'advance not from the current state': [(A, 2, 4)],
        'checkpoint out of range': [(T, 2, 1)],
        'restore of an empty checkpoint': [(R, 1, 0)],
        'reverse out of order': [(A, 1, 3), (V, 2, 0)],
        'reverse without its level': [(V, 3, 0)],
        'steps left unreversed': [(A, 1, 3), (V, 3, 0)],
        'unknown kind': [(7, 0, 0)],
    }
    for why, acts in bad.items():
        rc, msg = _check(acts, tf=(1, 10), tg=(1, 3))
        assert rc == 210, (why, msg)
    assert _check(ok, nck=0, tf=(1, 10), tg=(1, 3))[0] == 210


def test_solver_refusals_before_device_work():
    from devito_b200 import InvalidArgument
    geometry, solver = _solver()
    with pytest.raises(ValueError):
        solver.jacobian_adjoint(geometry.rec, checkpointing=True, n_checkpoints=0)
    with pytest.raises(TypeError):
        solver.jacobian_adjoint(geometry.rec)
    g4, s4 = _solver(kernel='OT4')
    with pytest.raises(NotImplementedError):
        s4.jacobian_adjoint(g4.rec, checkpointing=True, n_checkpoints=2)
    # a decomposed grid (the operators exist already; only the grid's distributor says it is split)
    import types
    solver.op_grad(save=True), solver.op_fwd(save=False)
    grid = solver.model.grid
    real = grid._distributor
    grid._distributor = types.SimpleNamespace(is_parallel=True)
    try:
        with pytest.raises(InvalidArgument, match='decomposed'):
            solver.jacobian_adjoint(geometry.rec, checkpointing=True, n_checkpoints=2)
    finally:
        grid._distributor = real


def test_stubs_point_at_the_solver_method():
    from devito_b200 import CheckpointOperator, DevitoCheckpoint, Revolver
    for c in (CheckpointOperator, DevitoCheckpoint, Revolver):
        with pytest.raises(NotImplementedError, match='jacobian_adjoint'):
            c()


def test_empty_time_range_needs_no_checkpoint_count():
    """No step to reverse: the default count is not computed (it would need the device) and the schedule is empty,
    which the library accepts as a call with nothing to do."""
    from devito_b200 import _lib
    geometry, solver = _solver()
    c = solver._revolve_setup(geometry.rec, time_M=0, resident=False)
    assert c.nsteps == 0 and c.nactions == 0 and c.n_checkpoints == 1
    L = _lib.load_library()
    assert L.b2_revolve_check(c.actions, 0, 1, c.fwd.time_m, c.fwd.time_M, c.grad.time_m, c.grad.time_M) == 0
