"""The one-thread-per-point CUDA kernels, executed on the CPU.

`devito_b200/csrc/b2_iso_point.cuh` holds the bodies of `k_iso_generic`, `k_ot4_w` and `k_iso_fs_fix`
as `__host__ __device__` functions; tests/support/emu_points.cu loops them over the grid as host code
(nvcc, no GPU). Comparing that with the oracle checks the very code the GPU runs — index arithmetic,
mirrored free-surface taps, the OT4 two-pass composition — before any GPU time is spent. It does not
cover launch geometry or the tiled TMA kernels; those are GPU tests."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import oracle as O
from helpers import rel_linf
import linear_cases as LC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.skipif(shutil.which('nvcc') is None, reason="nvcc not available")


@pytest.fixture(scope='module')
def emu(tmp_path_factory):
    out = tmp_path_factory.mktemp('emu') / 'libemu_points.so'
    cmd = ['nvcc', '-O1', '-shared', '-Xcompiler', '-fPIC', '-I', os.path.join(ROOT, 'include'),
           '-I', os.path.join(ROOT, 'devito_b200', 'csrc'), os.path.join(ROOT, 'tests', 'support', 'emu_points.cu'),
           '-o', str(out)]
    env = dict(os.environ)
    env.pop('CC', None)
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    lib = ctypes.CDLL(str(out))
    fp, ip = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int)
    lib.emu_iso_step.argtypes = [fp, ip, ctypes.c_int, ctypes.c_int, ctypes.c_int, fp, fp, fp, fp, ctypes.c_int,
                                 fp, ctypes.c_float, ctypes.c_float, ip, ip, ctypes.c_int, ctypes.c_int,
                                 ctypes.c_int, ctypes.c_int, ctypes.c_int, fp]
    lib.emu_iso_step.restype = ctypes.c_int
    lib.emu_born_step.argtypes = [fp, fp, fp, ip, ctypes.c_int, ip, ctypes.c_int, ctypes.c_int, fp, fp, fp, fp,
                                  ctypes.c_int, fp, ctypes.c_float, ctypes.c_float, ip, ip, ctypes.c_int,
                                  ctypes.c_int, ctypes.c_int]
    lib.emu_born_step.restype = ctypes.c_int
    lib.emu_snapshot.argtypes = [fp, ip, ctypes.c_int, fp, ip, ctypes.c_int, ip, ip]
    lib.emu_snapshot.restype = ctypes.c_int
    lib.emu_linear_steps.argtypes = [fp, ctypes.c_int, ctypes.c_int, ip, ctypes.c_int, ctypes.c_int, ip, ip, fp,
                                     ctypes.c_int, ip, ip, ctypes.c_int, ctypes.c_int]
    lib.emu_linear_steps.restype = ctypes.c_int
    return lib


def _fp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float)) if a is not None else None


def _ip(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))


def _initial(shape, so, seed):
    """Two smooth, non-trivial time levels (domain only; halo zero)."""
    rng = np.random.default_rng(seed)
    u = np.zeros((3,) + tuple(s + 2 * so for s in shape), dtype=np.float32)
    dom = (slice(so, -so),) * len(shape)
    grids = np.meshgrid(*[np.linspace(0, 1, s) for s in shape], indexing='ij')
    base = sum(np.sin((3 + i) * g * np.pi + rng.uniform(0, 1)) for i, g in enumerate(grids))
    u[(0,) + dom] = base
    u[(1,) + dom] = 0.9 * base + 0.05 * rng.standard_normal(shape)
    return u


def _run_emu(emu, u, so, w, dt, nsteps, damp, vp, param, param_kind, fs, ot4):
    nd = u.ndim - 1
    alloc3 = np.array(((1,) if nd == 2 else ()) + u.shape[1:], dtype=np.int32)
    lo = np.array(((0,) if nd == 2 else ()) + (0,) * nd, dtype=np.int32)
    hi = np.array(((0,) if nd == 2 else ()) + tuple(s - 2 * so - 1 for s in u.shape[1:]), dtype=np.int32)
    R = len(w[0]) - 1
    ws = [np.ascontiguousarray(x, dtype=np.float32) for x in w]
    if nd == 2:
        ws = [None] + ws
    W = np.zeros(int(np.prod(alloc3)), dtype=np.float32) if ot4 else None
    for time in range(1, nsteps + 1):
        rc = emu.emu_iso_step(_fp(u), _ip(alloc3), so, R, nd, _fp(ws[0]), _fp(ws[1]), _fp(ws[2]), _fp(damp),
                              param_kind, _fp(param), vp, dt, _ip(lo), _ip(hi), time % 3, (time - 1) % 3,
                              (time + 1) % 3, 1 if fs else 0, 1 if ot4 else 0, _fp(W))
        assert rc == 0
    return u


@pytest.mark.parametrize('case', ['plain', 'plain_vp_array', 'free_surface', 'free_surface_so4', 'ot4',
                                  'ot4_vp_array', 'plain_2d', 'free_surface_2d'])
def test_point_kernels_match_the_oracle(emu, case):
    fs = case.startswith('free_surface')
    ot4 = case.startswith('ot4')
    nd = 2 if case.endswith('2d') else 3
    so = 4 if case.endswith('so4') else 8
    shape = (22, 19, 17) if nd == 3 else (33, 29)
    h, vp, nsteps = 10.0, 1.5, 7
    dt = float(O.critical_dt(so, nd, h, 3.0))
    w = [O.fd2_weights(so, h)] * nd
    u_ref = _initial(shape, so, seed=3)
    u_emu = u_ref.copy()
    rng = np.random.default_rng(11)
    damp = np.pad((0.02 * rng.uniform(0, 1, shape)).astype(np.float32), so)
    param, kind = None, 0
    if case.endswith('vp_array'):
        param = np.pad(rng.uniform(1.5, 3.0, shape).astype(np.float32), so, mode='edge')
        kind = 1
    O.iso_forward(u_ref, so, w, dt, 1, nsteps, damp=damp, vp=vp, param=param, param_kind=kind,
                  free_surface=fs, ot4=ot4)
    _run_emu(emu, u_emu, so, w, dt, nsteps, damp, vp, param, kind, fs, ot4)
    dom = (slice(None),) + (slice(so, -so),) * nd
    assert np.abs(u_ref[dom]).max() > 0.1
    assert rel_linf(u_emu[dom], u_ref[dom]) < 1e-5
    if fs:
        assert not u_emu[dom][(nsteps + 1) % 3][..., 0].any()


@pytest.mark.parametrize('param', ['scalar', 'vp', 'm'])
def test_point_kernel_per_axis_spacing_and_sub_box_vs_float64(emu, param):
    """The generic point code with spacing (10, 12.5, 8), an interior update box that still reads the halo, and white
    noise in every time slot and in the halo, against the float64 reference (tests/ref64.py): a weight list or stride
    applied to the wrong axis in b2_iso_point.cuh, or a box bound off by one, fails here."""
    import kernel_cases as KC
    so = 8
    c = KC.iso_case(so, param, shape=(21, 26, 30), box=((1, 2, 3), (18, 22, 26)))
    _, w = KC.weights('iso', so)
    kind, pv = c['param']
    pk = 0 if np.ndim(pv) == 0 else (1 if kind == 'vp' else 2)
    u = c['u'].copy()
    alloc = np.array(u.shape[1:], dtype=np.int32)
    lo, hi = np.array(c['lo'], dtype=np.int32), np.array(c['hi'], dtype=np.int32)
    for time in range(1, KC.K + 1):
        rc = emu.emu_iso_step(_fp(u), _ip(alloc), so, so // 2, 3, _fp(w[0]), _fp(w[1]), _fp(w[2]), _fp(c['damp']), pk,
                              _fp(pv) if pk else None, float(pv) if pk == 0 else 1.0, c['dt'], _ip(lo), _ip(hi),
                              time % 3, (time - 1) % 3, (time + 1) % 3, 0, 0, None)
        assert rc == 0
    (ref,), _ = KC.reference(c)
    assert rel_linf(u, ref) < KC.TOL['iso']


@pytest.mark.parametrize('dmh', [0, 3])
def test_born_point_kernels_match_the_oracle(emu, dmh):
    so, shape, h, nsteps = 8, (21, 18, 16), 10.0, 6
    dt = float(O.critical_dt(so, 3, h, 3.0))
    w = [O.fd2_weights(so, h)] * 3
    rng = np.random.default_rng(5)
    u_ref = _initial(shape, so, seed=9)
    U_ref = 0.1 * _initial(shape, so, seed=10)
    u_emu, U_emu = u_ref.copy(), U_ref.copy()
    damp = np.pad((0.02 * rng.uniform(0, 1, shape)).astype(np.float32), so)
    vpa = np.pad(rng.uniform(1.5, 3.0, shape).astype(np.float32), so, mode='edge')
    dm = np.pad(rng.uniform(-0.05, 0.05, shape).astype(np.float32), dmh)
    O.born_forward(u_ref, U_ref, dm, so, w, dt, 1, nsteps, damp=damp, param=vpa, param_kind=1, dmhalo=dmh)
    alloc = np.array(u_emu.shape[1:], dtype=np.int32)
    dmalloc = np.array(dm.shape, dtype=np.int32)
    lo = np.zeros(3, dtype=np.int32)
    hi = np.array([s - 1 for s in shape], dtype=np.int32)
    ws = [np.ascontiguousarray(x, dtype=np.float32) for x in w]
    for time in range(1, nsteps + 1):
        rc = emu.emu_born_step(_fp(u_emu), _fp(U_emu), _fp(dm), _ip(dmalloc), dmh, _ip(alloc), so, 4, _fp(ws[0]),
                               _fp(ws[1]), _fp(ws[2]), _fp(damp), 1, _fp(vpa), 1.5, dt, _ip(lo), _ip(hi),
                               time % 3, (time - 1) % 3, (time + 1) % 3)
        assert rc == 0
    dom = (slice(None),) + (slice(so, -so),) * 3
    assert rel_linf(u_emu[dom], u_ref[dom]) < 1e-5
    assert rel_linf(U_emu[dom], U_ref[dom]) < 1e-5
    # the perturbation term matters in this set-up
    U_plain = 0.1 * _initial(shape, so, seed=10)
    O.iso_forward(U_plain, so, w, dt, 1, nsteps, damp=damp, param=vpa, param_kind=1)
    assert rel_linf(U_plain[dom], U_ref[dom]) > 1e-3


def test_snapshot_point_kernel(emu):
    """Copy of the iteration box between arrays of different halo width (so=8 wavefield -> so=2 snapshot)."""
    so, sh, shape = 8, 2, (9, 7, 11)
    rng = np.random.default_rng(2)
    slot = rng.standard_normal(tuple(s + 2 * so for s in shape)).astype(np.float32)
    snap = np.full(tuple(s + 2 * sh for s in shape), -7.0, dtype=np.float32)
    lo = np.array([1, 0, 2], dtype=np.int32)
    hi = np.array([7, 6, 9], dtype=np.int32)
    emu.emu_snapshot(_fp(slot), _ip(np.array(slot.shape, dtype=np.int32)), so, _fp(snap),
                     _ip(np.array(snap.shape, dtype=np.int32)), sh, _ip(lo), _ip(hi))
    box = tuple(slice(int(l), int(h) + 1) for l, h in zip(lo, hi))
    want = np.full_like(snap, -7.0)
    want[tuple(slice(b.start + sh, b.stop + sh) for b in box)] = slot[tuple(slice(b.start + so, b.stop + so) for b in box)]
    assert np.array_equal(snap, want)


def test_linear_point_kernel_runs_the_diffusion_example(emu):
    """BASELINE config 1 through the generic stencil kernel's point code: the operator's own taps
    (from the recogniser) applied by `linear_point` reproduce the reference's NumPy twin
    (examples/cfd/example_diffusion.py:61-83)."""
    from devito_b200 import Eq, Grid, Operator, TimeFunction, solve
    n, nt, a = 64, 20, 0.5
    g = Grid(shape=(n, n), extent=(2., 2.))
    u = TimeFunction(name='u', grid=g, time_order=1, space_order=2)
    hx, hy = g.spacing
    dt = 0.2 * hx * hy / a
    op = Operator([Eq(u.forward, solve(Eq(u.dt, a * u.laplace), u.forward), subdomain=g.interior)])
    args = op.arguments(time_M=nt - 1, dt=dt)
    init = np.zeros((n, n), dtype=np.float32)
    init[n // 4:n // 2, n // 4:n // 2] = 1.0
    so = 2
    f = np.zeros((2, n + 2 * so, n + 2 * so), dtype=np.float32)
    f[0, so:-so, so:-so] = init
    f[1, so:-so, so:-so] = init                       # cells outside the interior box are never written
    tshift = np.array([t for t, _, _ in args['taps']], dtype=np.int32)
    off = np.zeros((len(tshift), 3), dtype=np.int32)
    for i, (_, o, _) in enumerate(args['taps']):
        off[i, :2] = o
    coef = np.array([c for _, _, c in args['taps']], dtype=np.float32)
    emu.emu_linear_steps(_fp(f), 2, 2, _ip(np.array(f.shape[1:], dtype=np.int32)), so, len(tshift), _ip(tshift),
                         _ip(off), _fp(coef), op._plan['wshift'], _ip(np.array(args['lo'], dtype=np.int32)),
                         _ip(np.array(args['hi'], dtype=np.int32)), args['time_m'], args['time_M'])
    ref = init.astype(np.float64)
    for _ in range(nt):
        new = ref.copy()
        new[1:-1, 1:-1] = ref[1:-1, 1:-1] + a * dt * (
            (ref[2:, 1:-1] - 2 * ref[1:-1, 1:-1] + ref[:-2, 1:-1]) / hx ** 2 +
            (ref[1:-1, 2:] - 2 * ref[1:-1, 1:-1] + ref[1:-1, :-2]) / hy ** 2)
        ref = new
    assert rel_linf(f[nt % 2, so:-so, so:-so], ref) < 1e-5


@pytest.mark.parametrize('m', [m for m in LC.MATRIX if m[2] in ('fwd4', 'bwd3')], ids=LC.case_id)
def test_linear_point_kernel_vs_float64(emu, m):
    """Cases of the generic-update matrix (tests/test_linear_matrix.py) through `linear_point` on the CPU, with the
    taps and box the operator computes at apply, against tests/linear_ref.py: the 1-D and 3-D index arithmetic, the
    backward loop and the recogniser's taps, without a GPU."""
    c = LC.case(*m)
    op, _, _, _ = LC.build(c)
    _, _, over = LC.bounds(c)
    args = op.arguments(time_m=c['time_m'], time_M=c['time_M'], dt=LC.DEFAULTS['dt'], **over)
    taps = args['taps']
    tshift = np.array([t for t, _, _ in taps], dtype=np.int32)
    off = np.zeros((len(taps), 3), dtype=np.int32)
    for i, (_, o, _) in enumerate(taps):
        off[i, :c['nd']] = o
    coef = np.array([x for _, _, x in taps], dtype=np.float32)
    f = c['f'].copy()
    rc = emu.emu_linear_steps(_fp(f), f.shape[0], c['nd'], _ip(np.array(f.shape[1:], dtype=np.int32)), c['so'],
                              len(taps), _ip(tshift), _ip(off), _fp(coef), op._plan['wshift'],
                              _ip(np.array(args['lo'], dtype=np.int32)), _ip(np.array(args['hi'], dtype=np.int32)),
                              args['time_m'], args['time_M'])
    assert rc == 0
    LC.check(c, f, LC.reference(c))


def _emu_scheme(emu, c):
    """K steps of a KC scheme case through the point kernels (emu_iso_step / emu_born_step), no sparse points."""
    import kernel_cases as KC
    so = c['so']
    _, w = KC.weights('iso', so)
    kind, pv = c['param']
    pk = 0 if np.ndim(pv) == 0 else (1 if kind == 'vp' else 2)
    u = c['u'].copy()
    alloc = np.array(u.shape[1:], dtype=np.int32)
    lo, hi = np.array(c['lo'], dtype=np.int32), np.array(c['hi'], dtype=np.int32)
    par, vp = (_fp(pv) if pk else None), (float(pv) if pk == 0 else 1.0)
    if c['scheme'] == 'born':
        U = c['U'].copy()
        for time in range(1, KC.K + 1):
            rc = emu.emu_born_step(_fp(u), _fp(U), _fp(c['dm']), _ip(np.array(c['dm'].shape, dtype=np.int32)),
                                   c['dmh'], _ip(alloc), so, so // 2, _fp(w[0]), _fp(w[1]), _fp(w[2]), _fp(c['damp']),
                                   pk, par, vp, c['dt'], _ip(lo), _ip(hi), time % 3, (time - 1) % 3, (time + 1) % 3)
            assert rc == 0
        return dict(u=u, U=U)
    fs, ot4 = c['scheme'] == 'fs', c['scheme'] == 'ot4'
    W = np.zeros(int(np.prod(alloc)), dtype=np.float32) if ot4 else None
    for time in range(1, KC.K + 1):
        rc = emu.emu_iso_step(_fp(u), _ip(alloc), so, so // 2, 3, _fp(w[0]), _fp(w[1]), _fp(w[2]), _fp(c['damp']), pk,
                              par, vp, c['dt'], _ip(lo), _ip(hi), time % 3, (time - 1) % 3, (time + 1) % 3,
                              int(fs), int(ot4), _fp(W))
        assert rc == 0
    return dict(u=u)


@pytest.mark.parametrize('scheme,so,param,dmh', [
    ('fs', 4, 'scalar', 0), ('fs', 8, 'vp', 0), ('fs', 8, 'm', 0),
    ('ot4', 4, 'vp', 0), ('ot4', 8, 'scalar', 0), ('ot4', 8, 'm', 0),
    ('born', 8, 'vp', 0), ('born', 8, 'm', 3), ('born', 4, 'vp', 3),
])
def test_scheme_point_kernels_per_axis_spacing_vs_float64(emu, scheme, so, param, dmh):
    """`iso_fs_point`, `ot4_w_point` + `iso_point` and `born_src_point` with spacing (10, 12.5, 8), shape (21, 26, 32),
    white noise in every slot and halo, against tests/ref64.py. OT4 and Born run an interior box (which OT4 grows
    by R into the halo); the free surface needs z_m = 0, so its box is interior in x and y only. The vertical
    weights of the mirrored taps, of both OT4 Laplacians and of Born's U update are those of z only here."""
    import kernel_cases as KC
    shape = (21, 26, 32)
    box = ((1, 2, 0), (18, 22, 31)) if scheme == 'fs' else ((1, 2, 3), (18, 22, 26))
    c = KC.scheme_case(scheme, so, param, box=box, dmh=dmh, shape=shape)
    got = _emu_scheme(emu, c)
    want = KC.scheme_reference(c)
    assert rel_linf(got['u'], want['u']) < KC.TOL['iso']
    if scheme == 'born':
        assert rel_linf(got['U'], want['U']) < 1e-4
    if scheme == 'fs':
        assert not got['u'][(KC.K + 1) % 3][so + 1:so + 19, so + 2:so + 23, so].any()
