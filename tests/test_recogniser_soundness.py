"""What the wave-equation recogniser accepts (CPU): every (case, mutation) of `recogniser_cases` against a
recorded outcome, the interpreter runs of every refused pair, and the float64 twins of the base cases against
the restatements of the schemes (`ref64`, `sa_ref`), which makes them a trusted reference for the GPU matrix
(`test_recogniser_soundness_matrix.py`). Before the fixes this file tests, float64 operators, injections with a
literal dt and a wrong power of m, and injections without m were accepted (or raised KeyError)."""
import numpy as np
import pytest

import recogniser_cases as RC
import ref64
import sa_ref
import tti2d_ref
import tti_adjoint_ref
from devito_b200 import InvalidOperator, Operator

# Accepted (case, mutation) pairs and the plan kind they run as: every base case as built and as passed through the
# mutation helpers with a change of zero ('rebuilt'). Every other pair of `RC.CASES` is refused: the
# mutations change what is computed (a tap, a parameter's power or sampling point, the damping sign, a TTI or SA
# factor, the injected or interpolated expression), or hand the float32 kernels a float64 array.
ACCEPTED = {(case, mutation): kind for mutation in ('none', 'rebuilt') for case, kind in [
    ('iso_fwd', 'iso'), ('iso_fwd_so4_2d', 'iso'), ('iso_adj', 'iso'), ('iso_born', 'iso'), ('iso_grad', 'iso'),
    ('iso_ot4', 'iso'), ('iso_snap', 'iso'), ('tti_fwd', 'tti'), ('tti_adj', 'tti'), ('tti_fwd_2d', 'tti'),
    ('tti_adj_2d', 'tti'), ('sa_fwd', 'sa'), ('sa_adj', 'sa'), ('hand_solve', 'iso'), ('hand_solve_2d', 'iso'),
    ('hand_explicit', 'iso'), ('hand_vp_func', 'iso'), ('hand_vp_const', 'iso'), ('hand_nodamp', 'iso'),
    ('hand_param_so4', 'iso'), ('hand_subs', 'iso'), ('hand_rec_forward', 'iso'), ('hand_lit_dt', 'iso')]}

# What the refusal of a mutation says (a fragment of `Operator._why_not`), where it is the same for every case
REASON = {'grid64': 'the grid is float64', 'param64': 'is float64; the kernels read float32 arrays',
          'sparse64': 'float64; the kernels read float32 sparse data', 'inj_lit_m2': 'injected expression',
          'inj_lit_m': 'injected expression', 'inj_lit_no_m': 'injected expression',
          'inj_dt2_no_m': 'injected expression', 'inj_twice': 'injected expression'}


def test_every_mutation_applies_somewhere():
    assert set(RC.MUTATIONS) == {m for _, m in RC.CASES}
    assert set(ACCEPTED) <= set(RC.CASES)
    assert {c for c, _ in ACCEPTED} == set(RC.BASES)


@pytest.mark.parametrize('case,mutation', RC.CASES, ids=[f'{c}-{m}' for c, m in RC.CASES])
def test_outcome(case, mutation):
    """Building raises nothing; the plan kind is the recorded one; a refused operator says why and runs two steps
    on the interpreter."""
    try:
        b = RC.build(case, mutation)
    except (InvalidOperator, ValueError) as e:           # the documented refusals of Operator()
        pytest.fail(f"{case}/{mutation} cannot be built: {e}")
    want = ACCEPTED.get((case, mutation), 'refused')
    got = b.op._plan['kind'] if b.op._plan is not None else 'refused'
    assert got == want, b.op._why_not
    if got == 'refused':
        assert b.op.backend == 'numpy-interpreter'
        assert b.op._why_not
        if mutation in REASON:
            assert REASON[mutation] in b.op._why_not
        kw = dict(b.kwargs, time_M=b.kwargs['time_m'] + 1)
        b.op.apply(**kw)
        for f in b.functions.values():
            data = f.data if getattr(f, 'is_SparseFunction', False) else f.data_with_halo
            assert np.all(np.isfinite(data)), f.name


def test_no_injected_m_is_refused_not_a_keyerror():
    """An injection without m: refused with a reason (it used to raise KeyError looking up m's probe value)."""
    for mutation in ('inj_dt2_no_m', 'inj_lit_no_m'):
        b = RC.build('hand_solve', mutation)
        assert b.op._plan is None and 'injected expression' in b.op._why_not


# -- the float64 twins against the restatements -------------------------------------------------------------------
def _sparse(f):
    gp, ws = f.tabulate()
    return {'gp': gp, 'w': ws, 'r': f.r, 'data': np.array(f.data, dtype=np.float64)}


def _twin(case):
    b = RC.build(case, 'none', np.float64)
    assert b.op.backend == 'numpy-interpreter'
    init = {n: np.array(f.data if getattr(f, 'is_SparseFunction', False) else f.data_with_halo)
            for n, f in b.functions.items()}
    b.op.apply(**b.kwargs)
    return b, init


# The equations carry finite-difference weights rounded to 9 significant digits, like the reference's
# (`symbolics.fd_weights`); the restatements use the exact ones. The twins agree with them to ~5e-11 after K steps,
# five orders of magnitude inside the float32 tolerances of the GPU matrix.
TWIN_TOL = 1e-10


def _rel(a, b):
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def _tables(base, init):
    """The restatements' (gp, w, r, data) tables of the injected and the interpolated sparse functions."""
    srcf = next(o.sfunction for o in base.items if isinstance(o, RC.Injection))
    recf = next((o.sfunction for o in base.items if isinstance(o, RC.Interpolation)), None)
    src = dict(_sparse(srcf), data=init[srcf.name])
    rec = dict(_sparse(recf), data=init[recf.name]) if recf is not None else None
    return srcf, src, recf, rec


def _iso_weights(base, u):
    hs = [float(base.subs[d.spacing]) if base.subs else float(h) for d, h in zip(u.grid.dimensions, u.grid.spacing)]
    return [ref64.fd2_weights(u.space_order, h) for h in hs]


def _iso_param(fn, init, base, so):
    if 'vp' in fn:
        return ('vp', init['vp'])
    if 'm' in fn:
        # a parameter of another space order, in the wavefield's layout (only its box is read)
        return ('m', Operator._as_layout(fn['m'], so))
    return ('vp', float(base.param.data))


@pytest.mark.parametrize('case', ['iso_fwd', 'iso_fwd_so4_2d', 'iso_adj', 'iso_ot4', 'iso_grad', 'iso_snap',
                                  'hand_solve', 'hand_solve_2d', 'hand_explicit', 'hand_vp_func', 'hand_vp_const',
                                  'hand_nodamp', 'hand_param_so4', 'hand_subs', 'hand_rec_forward', 'hand_lit_dt'])
def test_iso_twin_matches_ref64(case):
    b, init = _twin(case)
    fn = b.functions
    base = RC._base(case, np.float64)
    u = next(f for f in fn.values() if getattr(f, 'is_TimeFunction', False) and f.is_buffered)
    so = u.space_order
    srcf, src, recf, rec = _tables(base, init)
    kw = {}
    if 'grad' in fn:
        kw = dict(grad=np.array(init['grad']), gh=fn['grad'].space_order, usave=init['u'][:, ...])
    if 'usave' in fn:
        us = fn['usave']
        kw = dict(snap=np.array(init['usave']), snap_h=us.space_order, snap_factor=int(us.time_dim.factor),
                  snap_toff=0)
    got_u, traces = ref64.iso_forward(init[u.name], so, _iso_weights(base, u), b.kwargs['dt'], 1, RC.K,
                                      damp=init.get('damp'), param=_iso_param(fn, init, base, so), src=src, rec=rec,
                                      adjoint=base.adjoint, ot4=case == 'iso_ot4',
                                      rec_toff=int(case == 'hand_rec_forward'), **kw)
    assert _rel(u.data_with_halo, got_u) < TWIN_TOL
    if rec is not None:
        assert _rel(recf.data, traces) < TWIN_TOL
    if 'grad' in fn:
        assert _rel(fn['grad'].data_with_halo, kw['grad']) < TWIN_TOL
    if 'usave' in fn:
        assert not np.array_equal(fn['usave'].data_with_halo, init['usave'])
        assert _rel(fn['usave'].data_with_halo, kw['snap']) < TWIN_TOL


def test_born_twin_matches_ref64():
    b, init = _twin('iso_born')
    fn = b.functions
    base = RC._base('iso_born', np.float64)
    u, U = fn['u'], fn['U']
    srcf, src, recf, rec = _tables(base, init)
    got_u, got_U, traces = ref64.born_forward(init['u'], init['U'], init['dm'], fn['dm'].space_order, u.space_order,
                                              _iso_weights(base, u), b.kwargs['dt'], 1, RC.K, damp=init['damp'],
                                              param=('vp', init['vp']), src=src, rec=rec)
    assert _rel(u.data_with_halo, got_u) < TWIN_TOL
    assert _rel(U.data_with_halo, got_U) < TWIN_TOL
    assert _rel(recf.data, traces) < TWIN_TOL


@pytest.mark.parametrize('case', ['tti_fwd', 'tti_adj', 'tti_fwd_2d', 'tti_adj_2d'])
def test_tti_twin_matches_restatement(case):
    from devito_b200.operator import half_node_first_derivative_weights, second_derivative_weights
    b, init = _twin(case)
    fn = b.functions
    base = RC._base(case, np.float64)
    f0, f1 = [o.lhs.function for o in base.items if isinstance(o, RC.Eq)][:2]
    so = f0.space_order
    hs = [float(h) for h in f0.grid.spacing]
    w2 = [second_derivative_weights(so, h) for h in hs]
    w1 = [half_node_first_derivative_weights(so, h) for h in hs]
    params = {n: init[n] for n in ('vp', 'epsilon', 'delta', 'theta', 'phi') if n in init}
    srcf, src, recf, rec = _tables(base, init)
    args = (init[f0.name], init[f1.name], so, w2, w1, b.kwargs['dt'], 1, RC.K, init['damp'], params)
    if base.nd == 2:
        run = tti2d_ref.adjoint if base.adjoint else tti2d_ref.forward
        out = run(*args, src=src, rec=rec)
        got0, got1, traces = out[0], out[1], out[-1]
    else:
        run = tti_adjoint_ref.tti_adjoint if base.adjoint else ref64.tti_forward
        got0, got1, traces = run(*args, src=src, rec=rec)
    assert _rel(f0.data_with_halo, got0) < TWIN_TOL
    assert _rel(f1.data_with_halo, got1) < TWIN_TOL
    assert _rel(recf.data, traces) < TWIN_TOL


@pytest.mark.parametrize('case', ['sa_fwd', 'sa_adj'])
def test_sa_twin_matches_sa_ref(case):
    b, init = _twin(case)
    fn = b.functions
    base = RC._base(case, np.float64)
    u = next(f for f in fn.values() if getattr(f, 'is_TimeFunction', False))
    so, R = u.space_order, u.space_order // 2
    c = [sa_ref.sa_weights(R, float(h)) for h in u.grid.spacing]
    srcf = next(o.sfunction for o in base.items if isinstance(o, RC.Injection))
    recf = next(o.sfunction for o in base.items if isinstance(o, RC.Interpolation))
    got_u, traces = sa_ref.sa_forward(init[u.name], so, c, b.kwargs['dt'], 1, RC.K, init['b'], init['vp'],
                                      w=init['damp'], src=dict(_sparse(srcf), data=init[srcf.name]),
                                      rec=dict(_sparse(recf), data=init[recf.name]), adjoint=base.adjoint)
    assert _rel(u.data_with_halo, got_u) < TWIN_TOL
    assert _rel(recf.data, traces) < TWIN_TOL


def test_float64_overrides_are_refused_at_apply():
    """An Operator on the CUDA path takes float32 arrays only, at apply as when it is built: wavefields, parameters,
    the sparse functions (traces and coordinates) and the field of the generic constant-coefficient update."""
    from devito_b200 import Eq, Function, Grid, InvalidArgument, Operator, SparseTimeFunction, TimeFunction
    b = RC.build('hand_solve')
    fn = b.functions
    u, m, src, rec = fn['u'], fn['m'], fn['src'], fn['rec']
    u64 = TimeFunction(name='u', grid=u.grid, time_order=2, space_order=u.space_order, dtype=np.float64)
    m64 = Function(name='m', grid=m.grid, space_order=m.space_order, dtype=np.float64)

    def sparse64(sf):
        out = SparseTimeFunction(name=sf.name, grid=sf.grid, npoint=sf.npoint, nt=sf.nt, dtype=np.float64)
        out.coordinates_data[:] = sf.coordinates_data
        return out
    for kw in ({'u': u64}, {'m': m64}, {'m': np.zeros(m.data_with_halo.shape)}, {'src': sparse64(src)},
               {'rec': sparse64(rec)}, {'src': np.zeros(src.data.shape)}):
        with pytest.raises(InvalidArgument, match='float32'):
            b.op.arguments(**kw, **b.kwargs)
    b.op.arguments(u=TimeFunction(name='u', grid=u.grid, time_order=2, space_order=u.space_order), **b.kwargs)

    grid = Grid(shape=(12, 10, 14), extent=(11., 9., 13.))
    f = TimeFunction(name='f', grid=grid, space_order=2)
    op = Operator(Eq(f.forward, f + 0.1 * f.laplace))
    assert op._plan['kind'] == 'linear'
    f64 = TimeFunction(name='f', grid=grid, space_order=2, dtype=np.float64)
    with pytest.raises(InvalidArgument, match='float32'):
        op.arguments(f=f64, time_M=2, dt=0.1)
    op.arguments(f=TimeFunction(name='f', grid=grid, space_order=2), time_M=2, dt=0.1)
