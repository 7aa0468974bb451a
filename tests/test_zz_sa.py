"""Self-adjoint variable-density visco-acoustic modelling (`SaIsoAcousticWaveSolver`, `b2_sa_forward`).

CPU: recognition of the solver's operators and of hand-written updates (so 4 / 8, 2-D / 3-D, scalar and array vp and
b); the look-alikes the recogniser refuses; the C adapter through a recording stub; the float64 restatement
(tests/sa_ref.py) against the reference's goldens (oracle/make_golden_sa.py), its mutations and its dot test;
`setup_w_over_q` against the reference's w/Q; the point body of k_sa_generic emulated on the CPU.
GPU: both goldens through `forward` / `adjoint`, the reference's test_adjoint_F in float32, and bit-for-bit
equalities (split time ranges, host staging, save=True).
"""
import ctypes
import functools
import os
import shutil
import subprocess

import numpy as np
import pytest

from helpers import load_golden, rel_linf
import kernel_cases as KC
import sa_ref as SA
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDENS = ['sa3d_so8', 'sa2d_so8']
TOL = 1e-5
# The 2-D golden runs 222 steps: there the float64 restatement misses the reference's float32 last levels of u and v
# by 4.1e-5 and 2.9e-5 (its traces by 6.6e-6 and 8.1e-6), so the reference's own float32 rounding is of that size;
# the last levels of that golden are held to 5e-5. Everything else meets 1e-5.
TOL_LEVEL_2D = 5e-5


def _golden_solver(name):
    from devito_b200.seismic import Model, SaIsoAcousticWaveSolver, setup_geometry, setup_w_over_q
    g = load_golden(name)
    shape = tuple(int(x) for x in g['shape'])
    so = int(g['so'])
    vp, b = SA.smooth_vp_b(shape)
    omega = 2.0 * np.pi * 0.010
    model = Model(origin=(0.,) * len(shape), shape=shape, vp=vp, b=b, spacing=(10.,) * len(shape),
                  nbl=int(g['nbl']), space_order=so, dtype=np.float32,
                  bcs=lambda f, nbl: setup_w_over_q(f, omega, 0.1, 1000.0, nbl))
    geometry = setup_geometry(model, float(g['tn']))
    solver = SaIsoAcousticWaveSolver(model, geometry, space_order=so)
    assert geometry.nt == int(g['nt']) and np.float32(solver.dt) == g['dt']
    return g, model, geometry, solver


def _sub(g, a):
    return np.asarray(a)[(slice(None, None, int(g['step'])),) * (a.ndim)]


# ---------------------------------------------------------------------------------------------------------------
# recognition
# ---------------------------------------------------------------------------------------------------------------
def _hand_written(so, nd, b_arr, vp_arr, kind='ref', forward=True):
    """The reference's update written with the DSL, or one look-alike of it."""
    from devito_b200 import Constant, Eq, Function, Grid, Operator, SparseTimeFunction, TimeFunction
    shape = (12, 13, 14)[:nd]
    grid = Grid(shape=shape, extent=tuple(10.0 * (n - 1) for n in shape))
    mkf = lambda n, v: Function(name=n, grid=grid, space_order=so)
    b = mkf('b', 1) if b_arr else Constant(name='b', value=0.8)
    vp = mkf('vp', 1) if vp_arr else Constant(name='vp', value=1.5)
    w = mkf('damp', 1)
    u = TimeFunction(name='u', grid=grid, time_order=2, space_order=so)
    t = u.dimensions[0]
    s = t.spacing
    nxt, prv = (u.forward, u.backward) if forward else (u.backward, u.forward)
    div = 0
    for d, dn in zip(u.dimensions[1:], ('dx', 'dy', 'dz')):
        if kind == 'b_at_output':
            div = div + b * getattr(getattr(u, dn)(x0=d + d.spacing / 2), dn)(x0=d - d.spacing / 2)
        elif kind == 'b_half_node':
            bh = (b + b.subs({d: d + d.spacing})) / 2 if b_arr else b
            div = div + getattr(bh * getattr(u, dn)(x0=d + d.spacing / 2), dn)(x0=d - d.spacing / 2)
        elif kind == 'order_mismatch':
            div = div + getattr(b * getattr(u, dn)(x0=d + d.spacing / 2), dn)(x0=d - d.spacing / 2,
                                                                                fd_order=so - 2)
        else:
            div = div + getattr(b * getattr(u, dn)(x0=d + d.spacing / 2), dn)(x0=d - d.spacing / 2)
    C = s ** 2 * vp ** 2 if kind == 'no_inv_b' else s ** 2 * vp ** 2 / b
    if kind == 'foreign_symbol':
        # a runtime symbol other than dt and the spacings where one factor dt belongs
        from devito_b200.symbolics import Symbol
        C = s * Symbol('tau') * vp ** 2 / b
    k0, km = (2 - s * w, s * w - 1) if kind != 'w_swap' else (s * w - 1, 2 - s * w)
    eqs = [Eq(nxt, C * div + k0 * u + km * prv)]
    if kind == 'fwd_run_backward':
        # the forward combination, u[t+1] = f(u[t], u[t-1]), solved for u[t-1] and run backward
        eqs = [Eq(u.backward, (u.forward - C * div - k0 * u) / km)]
    src = SparseTimeFunction(name='src', grid=grid, npoint=1, nt=10, coordinates=np.full((1, nd), 40.0))
    rec = SparseTimeFunction(name='rec', grid=grid, npoint=2, nt=10, coordinates=np.full((2, nd), 50.0))
    eqs += src.inject(field=nxt, expr=src * s ** 2 * vp ** 2 / b)
    eqs += rec.interpolate(expr=u)
    return Operator(eqs)


@pytest.mark.parametrize('forward', [True, False], ids=['fwd', 'adj'])
@pytest.mark.parametrize('b_arr,vp_arr', [(True, True), (False, False), (True, False), (False, True)],
                         ids=['b_arr-vp_arr', 'b_scalar-vp_scalar', 'b_arr-vp_scalar', 'b_scalar-vp_arr'])
@pytest.mark.parametrize('nd', [2, 3])
@pytest.mark.parametrize('so', [4, 8])
def test_hand_written_update_is_recognised(so, nd, b_arr, vp_arr, forward):
    op = _hand_written(so, nd, b_arr, vp_arr, forward=forward)
    assert op.backend == 'cuda-sm90a', op._why_not
    p = op._plan
    assert p['kind'] == 'sa' and p['R'] == so // 2 and p['adjoint'] == (not forward)
    assert p['b_role'][1].name == 'b' and p['vp_role'][1].name == 'vp' and p['damp'].name == 'damp'
    assert p['src'].name == 'src' and p['rec'].name == 'rec' and p['rec_toff'] == 0
    assert np.allclose(p['c'][0], SA.sa_weights(so // 2, 10.0), rtol=1e-8)
    assert 'b2_sa_forward' in str(op)


LOOKALIKES = ['b_at_output', 'b_half_node', 'no_inv_b', 'w_swap', 'order_mismatch', 'fwd_run_backward',
              'foreign_symbol']


@pytest.mark.parametrize('kind', LOOKALIKES)
def test_lookalikes_are_refused(kind):
    op = _hand_written(8, 3, True, True, kind=kind, forward=kind != 'fwd_run_backward')
    assert op.backend == 'numpy-interpreter', kind


@pytest.mark.parametrize('nd', [2, 3])
def test_solver_operators_are_recognised(nd):
    from devito_b200.seismic import acoustic_sa_setup
    solver = acoustic_sa_setup(shape=(21, 22, 23)[:nd], nbl=6, tn=30.0)
    fwd, adj, sav = solver.op_fwd(), solver.op_adj(), solver.op_fwd(True)
    for op, name in ((fwd, 'IsoFwdOperator'), (adj, 'IsoAdjOperator'), (sav, 'IsoFwdOperator')):
        assert (op.name, op.backend) == (name, 'cuda-sm90a'), op._why_not
    assert not fwd._plan['adjoint'] and adj._plan['adjoint']
    assert (fwd._plan['src'].name, fwd._plan['rec'].name) == ('src', 'rec')
    assert (adj._plan['src'].name, adj._plan['rec'].name) == ('rec', 'src')
    assert solver.model.dt_scale == .5
    for call in (lambda: solver.jacobian(None), lambda: solver.jacobian_adjoint(None, None), solver.op_jac,
                 solver.op_jacadj):
        with pytest.raises(NotImplementedError, match='linearised'):
            call()


def test_cinterface_recording_stub_sees_the_sa_struct(tmp_path):
    """The generated adapter of IsoAdjOperator, compiled against a recording stub of b2_sa_forward, packs the
    weights, the arrays, the direction and the sparse tables into struct b2_sa_args."""
    if shutil.which('gcc') is None:
        pytest.skip("gcc not available")
    from devito_b200 import cinterface as ci
    from devito_b200.seismic import acoustic_sa_setup
    solver = acoustic_sa_setup(shape=(21, 22, 23), nbl=6, tn=30.0)
    op = solver.op_adj()
    ccode, hcode = ci.generate(op._plan, 'IsoAdjOperator')
    (tmp_path / 'IsoAdjOperator.c').write_text(ccode)
    (tmp_path / 'IsoAdjOperator.h').write_text(hcode)
    (tmp_path / 'stub.c').write_text('''#include "b200stencil.h"
static struct b2_sa_args g;
static float g_c[3][8];
int b2_sa_forward(const struct b2_sa_args *a) { g = *a; for (int d = 0; d < 3; ++d) for (int i = 0; i < a->radius; ++i)
  g_c[d][i] = a->c[d][i]; return 0; }
void *seen(int i) { void *p[6] = {g.u, g.b, g.vp, g.damp, g.src ? g.src->data : 0, g.rec ? g.rec->data : 0};
  return p[i]; }
int seen_int(int i) { int v[7] = {g.ndim, g.space_order, g.radius, g.adjoint, g.rec_toff, g.time_m, g.time_M};
  return v[i]; }
float seen_c(int d, int i) { return g_c[d][i]; }
float seen_dt(void) { return g.dt; }
''')
    so = tmp_path / 'libadj.so'
    subprocess.run(['gcc', '-shared', '-fPIC', '-Wl,-Bsymbolic', '-I', os.path.join(ROOT, 'include'), '-I',
                    str(tmp_path), '-o', str(so), str(tmp_path / 'IsoAdjOperator.c'), str(tmp_path / 'stub.c')],
                   check=True)
    lib = ctypes.CDLL(str(so))
    params = ci.signature(op._plan, 'IsoAdjOperator')
    objs = {p.name: ctypes.create_string_buffer(64) for p in params if p.ctype.startswith('struct dataobj')}
    argv = []
    for p in params:
        if p.ctype.startswith('struct dataobj'):
            argv.append(ctypes.cast(objs[p.name], ctypes.c_void_p))
        elif p.ctype == 'const float':
            argv.append(ctypes.c_float(0.5))
        elif p.ctype == 'const int':
            argv.append(ctypes.c_int({'time_m': 1, 'time_M': 7}.get(p.name, 0)))
        else:
            argv.append(ctypes.c_void_p(None))
    assert getattr(lib, 'IsoAdjOperator')(*argv) == 0
    lib.seen.restype = ctypes.c_void_p
    lib.seen_c.restype = ctypes.c_float
    lib.seen_dt.restype = ctypes.c_float
    addr = lambda n: ctypes.cast(objs[n], ctypes.c_void_p).value
    for i, n in enumerate(('v_vec', 'b_vec', 'vp_vec', 'damp_vec')):
        assert lib.seen(i) == addr(n), n
    # the adjoint injects the receiver data and samples the adjoint source (the reference's `src`)
    assert lib.seen(4) == addr('rec_vec') and lib.seen(5) == addr('src_vec')
    assert [lib.seen_int(i) for i in range(7)] == [3, 8, 4, 1, 0, 1, 7]
    assert lib.seen_dt() == np.float32(0.5)
    for d in range(3):
        want = np.float32(SA.sa_weights(4, 10.0))
        assert np.allclose([lib.seen_c(d, i) for i in range(4)], want, rtol=1e-6)


# ---------------------------------------------------------------------------------------------------------------
# the float64 restatement
# ---------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _golden_reference(name):
    g, model, geometry, solver = _golden_solver(name)
    so = int(g['so'])
    nt = int(g['nt'])
    c = [SA.sa_weights(so // 2, h) for h in model.spacing]
    B, V, W = [np.array(f.data_with_halo) for f in (model.b, model.vp, model.damp)]
    gp, ws = geometry.src.tabulate()
    src = dict(gp=gp, w=ws, r=geometry.src.r, data=g['src'])
    gp, ws = geometry.rec.tabulate()
    rec = dict(gp=gp, w=ws, r=geometry.rec.r, data=np.zeros_like(g['rec']))
    u0 = np.zeros((3,) + B.shape)
    dom = tuple(slice(so, -so) for _ in B.shape)
    u, tr = SA.sa_forward(u0, so, c, float(g['dt']), 1, nt - 2, B, V, W, src=src, rec=rec)
    v, tra = SA.sa_forward(u0, so, c, float(g['dt']), 1, nt - 2, B, V, W, src=dict(rec, data=g['rec']),
                           rec=dict(src, data=np.zeros_like(g['srca'])), adjoint=True)
    return g, model, dict(rec=tr, srca=tra, u=_sub(g, u[(nt - 1) % 3][dom]), v=_sub(g, v[0][dom]))


@pytest.mark.parametrize('name', GOLDENS)
def test_float64_vs_reference_golden(name):
    g, model, got = _golden_reference(name)
    lvl = TOL_LEVEL_2D if name.startswith('sa2d') else TOL
    assert rel_linf(got['rec'], g['rec']) < TOL
    assert rel_linf(got['srca'], g['srca']) < TOL
    assert rel_linf(got['u'], g['u']) < lvl
    assert rel_linf(got['v'], g['v']) < lvl


@pytest.mark.parametrize('name', GOLDENS)
def test_setup_w_over_q_matches_the_reference(name):
    g, model, _, _ = _golden_solver(name)
    assert rel_linf(_sub(g, model.damp.data), g['w']) < 1e-6


def _noise_case(so, nd=3, seed=5):
    c = dict(so=so)
    shape = (14, 15, 17)[:nd] if nd == 3 else (19, 23)
    alloc = tuple(n + 2 * so for n in shape)
    rng = np.random.default_rng(seed)
    c['shape'], c['spacing'] = shape, (10.0, 12.5, 8.0)[:nd]
    c['u'] = rng.standard_normal((3,) + alloc)
    c['b'] = rng.uniform(0.4, 1.2, alloc)
    c['vp'] = rng.uniform(1.5, 3.0, alloc)
    c['w'] = rng.uniform(0.0, 0.3, alloc)
    c['c'] = [SA.sa_weights(so // 2, h) for h in c['spacing']]
    return c


@pytest.mark.parametrize('mut', sorted(SA.MUTATIONS))
def test_mutations_move_the_result(mut):
    """Every mutation moves u by more than 100x the GPU tolerance on the white-noise case."""
    c = _noise_case(8)
    args = (c['u'], 8, c['c'], 0.9, 1, 3, c['b'], c['vp'], c['w'])
    ref, _ = SA.sa_forward(*args)
    bad, _ = SA.sa_forward(*args, mut=mut)
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
    the adjoint run with receiver traces d, sampled at the sources, with variable b, vp and w/Q."""
    c = _noise_case(so, nd)
    nt = 30
    s = _interior_sparse(c['shape'], c['spacing'], nt, 3, 1)
    d = _interior_sparse(c['shape'], c['spacing'], nt, 4, 2)
    z = np.zeros_like(c['u'])
    args = (so, c['c'], 0.5, 1, nt - 2, c['b'], c['vp'], c['w'])
    _, Fs = SA.sa_forward(z, *args, src=s, rec=dict(d, data=np.zeros_like(d['data'])))
    _, Ftd = SA.sa_forward(z, *args, src=d, rec=dict(s, data=np.zeros_like(s['data'])), adjoint=True)
    lhs = float(np.sum(Fs * d['data']))
    rhs = float(np.sum(s['data'] * Ftd))
    assert abs(lhs - rhs) / abs(lhs) < 1e-11


@pytest.fixture(scope='module')
def emu(tmp_path_factory):
    if shutil.which('nvcc') is None:
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp('emu') / 'libemu_sa.so'
    cmd = ['nvcc', '-O1', '-shared', '-Xcompiler', '-fPIC', '-I', os.path.join(ROOT, 'include'),
           '-I', os.path.join(ROOT, 'devito_b200', 'csrc'), os.path.join(ROOT, 'tests', 'support', 'emu_sa.cu'),
           '-o', str(out)]
    subprocess.run(cmd, check=True, capture_output=True)
    lib = ctypes.CDLL(str(out))
    lib.emu_sa_step.restype = ctypes.c_int
    return lib


@pytest.mark.parametrize('nd', [2, 3])
@pytest.mark.parametrize('so', [4, 8])
def test_emulated_point_body(emu, so, nd):
    """k_sa_generic's point body looped over an interior box on the CPU, one step, against float64."""
    c = _noise_case(so, nd)
    f32 = lambda x: np.ascontiguousarray(x, dtype=np.float32)
    u = f32(c['u'])
    b, vp, w = f32(c['b']), f32(c['vp']), f32(c['w'])
    dt = 0.9
    C = f32(np.float32(dt * dt) * vp * vp / b)
    lo = [1, 2, 4][:nd] if nd == 3 else [1, 4]
    hi = [n - 2 for n in c['shape']]
    out = u[2].copy()
    a3 = (1,) * (3 - nd) + u.shape[1:]
    lo3 = [0] * (3 - nd) + lo
    n3 = [1] * (3 - nd) + [h - l + 1 for l, h in zip(lo, hi)]
    r3 = [0] * (3 - nd) + [so // 2] * nd
    cw = np.zeros((3, 8), dtype=np.float32)
    for d in range(nd):
        cw[3 - nd + d, :so // 2] = c['c'][d]
    ip = lambda x: (ctypes.c_int * 3)(*x)
    fp = lambda x: x.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    rc = emu.emu_sa_step(fp(u[1]), fp(u[0]), fp(out), fp(b), fp(C), fp(w), ip(a3), ip(lo3), ip(n3), ip(r3), fp(cw),
                         ctypes.c_int(so), ctypes.c_float(dt))
    assert rc == 0
    want, _ = SA.sa_forward(u, so, c['c'], dt, 1, 1, b, vp, w, lo=lo, hi=hi)
    assert rel_linf(out, want[2]) < 1e-5


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('name', GOLDENS)
def test_forward_and_adjoint_vs_reference_golden(name):
    g, model, geometry, solver = _golden_solver(name)
    lvl = TOL_LEVEL_2D if name.startswith('sa2d') else TOL
    nt = int(g['nt'])
    rec, u, _ = solver.forward()
    assert rel_linf(rec.data, g['rec']) < TOL
    assert rel_linf(_sub(g, np.asarray(u.data)[(nt - 1) % 3]), g['u']) < lvl
    rec.data[:] = g['rec']
    srca, v, _ = solver.adjoint(rec)
    assert rel_linf(srca.data, g['srca']) < TOL
    assert rel_linf(_sub(g, np.asarray(v.data)[0]), g['v']) < lvl
    from devito_b200 import _lib
    # the 3-D golden's layout takes the TMA sweep, the 2-D one the generic kernel
    want = 'sa_tma<4>+adj' if name.startswith('sa3d') else 'sa_generic+adj'
    assert _lib.lib().b2_last_sweep_kernel().decode() == want


@pytest.mark.gpu
@pytest.mark.parametrize('shape', [(71, 61), (71, 61, 51)])
def test_adjoint_F_float32(shape):
    """The reference's test_adjoint_F (test_wavesolver_iso.py:87-107) in float32: r . F(s) = F^T(r) . s."""
    from devito_b200.seismic import acoustic_sa_setup
    solver = acoustic_sa_setup(shape=shape, space_order=8)
    src1, rec1 = solver.geometry.src, solver.geometry.rec
    rec2, _, _ = solver.forward(src1)
    rec1.data[:] = rec2.data[:]
    src2, _, _ = solver.adjoint(rec1)
    sum_s = np.dot(src1.data.reshape(-1).astype(np.float64), src2.data.reshape(-1).astype(np.float64))
    sum_r = np.dot(rec1.data.reshape(-1).astype(np.float64), rec2.data.reshape(-1).astype(np.float64))
    assert abs(sum_s - sum_r) / abs(sum_s + sum_r) < 1e-4


@pytest.mark.gpu
def test_bitwise_equalities():
    """Split [time_m, time_M] ranges equal one call; a host-staged apply equals the resident one; forward(save=True)
    equals the buffered run at the last three levels; no staging is left outstanding."""
    from devito_b200 import TimeFunction, _lib
    g, model, geometry, solver = _golden_solver('sa3d_so8')
    nt = geometry.nt
    rec_a, u_a, _ = solver.forward()
    rec_a, u_a = np.array(rec_a.data), np.array(u_a.data_with_halo)
    mk = lambda: TimeFunction(name='u', grid=model.grid, time_order=2, space_order=8)
    u = mk()
    rec = geometry.rec                    # a new receiver object: every split call must write into this one
    for lo, hi in ((1, 30), (31, 31), (32, nt - 2)):
        solver.forward(rec=rec, u=u, time_m=lo, time_M=hi)
    assert np.array_equal(np.array(rec.data), rec_a)
    assert np.array_equal(np.array(u.data_with_halo), u_a)
    u2 = mk()
    rec_b, _, _ = solver.forward(u=u2, resident=False)
    assert np.array_equal(np.array(rec_b.data), rec_a)
    assert np.array_equal(np.array(u2.data_with_halo), u_a)
    rec_s, us, _ = solver.forward(save=True)
    assert np.array_equal(np.array(rec_s.data), rec_a)
    for t in (nt - 3, nt - 2, nt - 1):
        assert np.array_equal(np.array(us.data_with_halo[t]), u_a[t % 3])
    assert _lib.lib().b2_staging_outstanding() == 0
