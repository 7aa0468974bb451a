"""2-D centred-TTI modelling: forward (`ForwardTTI`), adjoint (`AdjointTTI`), Born (`BornTTI`) and gradient
(`GradientTTI`) with the reference's `Gzz_centered_2d`.

CPU: recognition of the solver's four 2-D operators and refusal of look-alikes (phi on a 2-D grid, sin / cos swapped,
theta sampled at the output point); the C adapter passes ndim = 2; the float64 restatement (tests/tti2d_ref.py)
against the reference's goldens (oracle/make_golden_tti2d.py), its mutations, and the F / F^T dot test.
GPU: the goldens through the solver with the single-pass and the two-pass sweeps, the reference's 2-D
`test_adjoint_F` / `test_adjoint_J` / `test_gradientJ` in float32, restarts over split time ranges and host staging.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from helpers import load_golden, rel_linf
import tti2d_ref as T2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDENS = ['tti2d_so8', 'tti2d_so4_layers', 'tti2d_so8_varying']
TOL = 1e-4


def _last_kernel():
    from devito_b200 import _lib
    return _lib.lib().b2_last_sweep_kernel().decode()


def _solver(name):
    """The package's solver on the model of golden `name`."""
    from devito_b200.seismic import SeismicModel, demo_model, setup_geometry
    from devito_b200.seismic.tti import AnisotropicWaveSolver
    g = load_golden(name)
    so, shape, nbl = int(g['so']), tuple(int(x) for x in g['shape']), int(g['nbl'])
    if name.endswith('varying'):
        par = {k[4:]: g[k] for k in g if k.startswith('par_')}
        model = SeismicModel(space_order=so, origin=(0., 0.), shape=shape, dtype=np.float32, spacing=(10., 10.),
                             nbl=nbl, bcs="damp", **par)
    else:
        preset = 'constant-tti' if name == 'tti2d_so8' else 'layers-tti'
        kw = {} if preset == 'constant-tti' else {'nlayers': 3}
        model = demo_model(preset, spacing=(10., 10.), shape=shape, nbl=nbl, space_order=so, **kw)
    geometry = setup_geometry(model, float(g['tn']))
    return g, model, geometry, AnisotropicWaveSolver(model, geometry, space_order=so)


# ---------------------------------------------------------------------------------------------------------------
# recognition
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', GOLDENS)
def test_solver_operators_are_recognised(name):
    g, model, _, solver = _solver(name)
    assert float(np.float32(model.critical_dt)) == float(g['dt'])
    for op, want in ((solver.op_fwd(), 'ForwardTTI'), (solver.op_fwd(True), 'ForwardTTI'),
                     (solver.op_adj(), 'AdjointTTI'), (solver.op_jac(), 'BornTTI'),
                     (solver.op_jacadj(), 'GradientTTI')):
        assert (op.name, op.backend) == (want, 'cuda-sm90a'), op._why_not
        assert op._plan['grid'].dim == 2 and op._entry.flags['ndim'] == 2


LOOKALIKES = ['phi', 'sincos_swap', 'theta_at_output', 'inner_full_order', 'fwd_mix']


def _lookalike(kind):
    """A 2-D TTI pair (array-valued parameters) with one deviation from the reference's formulation."""
    from devito_b200 import Eq, Function, Grid, Operator, TimeFunction, cos, sin, solve, sqrt
    from devito_b200.seismic.tti import Gzz_centered_2d
    from types import SimpleNamespace
    so = 8
    grid = Grid(shape=(12, 14), extent=(110., 130.))
    x, z = grid.dimensions
    fn = lambda n: Function(name=n, grid=grid, space_order=so)
    vp, eps, delta, theta, damp = fn('vp'), fn('epsilon'), fn('delta'), fn('theta'), fn('damp')
    u = TimeFunction(name='u', grid=grid, time_order=2, space_order=so)
    v = TimeFunction(name='v', grid=grid, time_order=2, space_order=so)
    m, e2, sd = 1 / (vp * vp), 1 + 2 * eps, sqrt(1 + 2 * delta)
    model = SimpleNamespace(theta=theta, dim=2)

    def gzz(f):
        if kind in ('sincos_swap', 'theta_at_output', 'inner_full_order', 'phi'):
            o1 = so // 2 if kind != 'inner_full_order' else so
            st, ct = (cos(theta), sin(theta)) if kind == 'sincos_swap' else (sin(theta), cos(theta))
            gz = st * f.dx(fd_order=o1, x0=x + x.spacing / 2) + ct * f.dy(fd_order=o1, x0=z + z.spacing / 2)
            if kind == 'phi':
                gz = gz * cos(Function(name='phi', grid=grid, space_order=so))
            if kind == 'theta_at_output':
                return ct * gz.dy(fd_order=so // 2, x0=z - z.spacing / 2) + \
                    st * gz.dx(fd_order=so // 2, x0=x - x.spacing / 2)
            return (gz * ct).dy(fd_order=so // 2, x0=z - z.spacing / 2) + \
                (gz * st).dx(fd_order=so // 2, x0=x - x.spacing / 2)
        return Gzz_centered_2d(model, f)
    if kind == 'fwd_mix':            # a backward pair with the forward combination
        gxx = u.laplace - gzz(u)
        H0, Hz = e2 * gxx + sd * gzz(v), sd * gxx + gzz(v)
        eqs = [Eq(u.backward, solve(m * u.dt2 - H0 + damp * u.dt.T, u.backward)),
               Eq(v.backward, solve(m * v.dt2 - Hz + damp * v.dt.T, v.backward))]
    else:
        gxx = u.laplace - gzz(u)
        H0, Hz = e2 * gxx + sd * gzz(v), sd * gxx + gzz(v)
        eqs = [Eq(u.forward, solve(m * u.dt2 - H0 + damp * u.dt, u.forward)),
               Eq(v.forward, solve(m * v.dt2 - Hz + damp * v.dt, v.forward))]
    return Operator(eqs)


def test_lookalike_builder_accepts_the_reference_formulation():
    op = _lookalike('none')
    assert op.backend == 'cuda-sm90a', op._why_not


@pytest.mark.parametrize('kind', LOOKALIKES)
def test_lookalikes_are_refused(kind):
    from devito_b200 import InvalidOperator
    try:
        op = _lookalike(kind)
    except (InvalidOperator, NotImplementedError, KeyError, ValueError):
        return
    assert op.backend == 'numpy-interpreter', kind


def test_cinterface_passes_ndim_2(tmp_path):
    """The generated adapter of a 2-D ForwardTTI, compiled against a recording stub of b2_tti_forward, sets ndim = 2
    and the x / z weights in slots 0 and 1."""
    if shutil.which('gcc') is None:
        pytest.skip("gcc not available")
    from devito_b200 import cinterface as ci
    _, _, _, solver = _solver('tti2d_so4_layers')
    op = solver.op_fwd()
    ccode, hcode = ci.generate(op._plan, 'ForwardTTI')
    assert '  a.ndim = 2;' in ccode and 'a.w2[2]' not in ccode
    (tmp_path / 'ForwardTTI.c').write_text(ccode)
    (tmp_path / 'ForwardTTI.h').write_text(hcode)
    (tmp_path / 'stub.c').write_text('''#include "b200stencil.h"
static int g_nd = -1, g_w = 0;
int b2_tti_forward(const struct b2_tti_args *a) { g_nd = a->ndim; g_w = (a->w2[0] != 0) + (a->w2[1] != 0) +
  (a->w2[2] != 0); return 0; }
int seen_nd(void) { return g_nd; }
int seen_w(void) { return g_w; }
''')
    so = tmp_path / 'libfwd.so'
    subprocess.run(['gcc', '-shared', '-fPIC', '-Wl,-Bsymbolic', '-I', os.path.join(ROOT, 'include'), '-I',
                    str(tmp_path), '-o', str(so), str(tmp_path / 'ForwardTTI.c'), str(tmp_path / 'stub.c')],
                   check=True)
    lib = ctypes.CDLL(str(so))
    params = ci.signature(op._plan, 'ForwardTTI')
    objs = {p.name: ctypes.create_string_buffer(64) for p in params if p.ctype.startswith('struct dataobj')}
    argv = []
    for p in params:
        if p.ctype.startswith('struct dataobj'):
            argv.append(ctypes.cast(objs[p.name], ctypes.c_void_p))
        elif p.ctype == 'const float':
            argv.append(ctypes.c_float(1.0))
        elif p.ctype == 'const int':
            argv.append(ctypes.c_int(0))
        else:
            argv.append(ctypes.c_void_p(None))
    assert getattr(lib, 'ForwardTTI')(*argv) == 0
    assert (lib.seen_nd(), lib.seen_w()) == (2, 2)


# ---------------------------------------------------------------------------------------------------------------
# the float64 restatement against the reference
# ---------------------------------------------------------------------------------------------------------------
def _inputs(name):
    """Everything the restatement needs, taken from the package's (host-side) model and geometry."""
    from devito_b200.operator import half_node_first_derivative_weights, second_derivative_weights
    g, model, geometry, solver = _solver(name)
    so = int(g['so'])
    dt = float(g['dt'])
    hs = [float(h) for h in model.spacing]
    w2 = [second_derivative_weights(so, h) for h in hs]
    w1 = [half_node_first_derivative_weights(so, h) for h in hs]
    params = {}
    for k in ('vp', 'epsilon', 'delta', 'theta'):
        f = getattr(model, k)
        params[k] = np.array(f.data_with_halo, np.float64) if hasattr(f, 'data_with_halo') else float(f.data)
    params = {k: (v if np.ndim(v) else np.full(model.damp.data_with_halo.shape, v)) for k, v in params.items()}
    damp = np.array(model.damp.data_with_halo, np.float64)

    def sparse(sf, data):
        gp, w = sf.tabulate()
        return dict(gp=gp, w=w, r=sf.r, data=np.array(data, np.float64))
    return g, model, geometry, so, dt, w2, w1, params, damp, sparse


def _zeros(so, model, nt=3):
    return np.zeros((nt,) + tuple(s + 2 * so for s in model.grid.shape))


def restated(name, mut=None):
    """(forward rec, u_last, srca, p, born rec, du, grad) of the restatement, float64."""
    g, model, geometry, so, dt, w2, w1, P, damp, sparse = _inputs(name)
    nt = int(g['nt'])
    src = sparse(geometry.src, geometry.src.data)
    rec = sparse(geometry.rec, np.zeros_like(g['rec']))
    u = _zeros(so, model, nt)
    uf, vf, _, _, rec_f = T2.forward(u, u, so, w2, w1, dt, 1, nt - 2, damp, P, src=src, rec=rec, mut=mut)
    rin = sparse(geometry.rec, g['rec'])
    srca = sparse(geometry.src, np.zeros_like(g['srca']))
    z3 = _zeros(so, model)
    p, r, srca_t = T2.adjoint(z3, z3, so, w2, w1, dt, 1, nt - 2, damp, P, src=rin, rec=srca, mut=mut)
    grad = np.zeros(model.grid.shape)
    T2.adjoint(z3, z3, so, w2, w1, dt, 1, nt - 2, damp, P, src=rin, grad=grad, gh=0, usave=uf, vsave=vf, mut=mut)
    rb = sparse(geometry.rec, np.zeros_like(g['born_rec']))
    _, _, du, _, rec_b = T2.forward(z3, z3, so, w2, w1, dt, 1, nt - 2, damp, P, src=src, rec=rb, du=z3, dv=z3,
                                    dm=g['dm'], mut=mut)
    dom = lambda a: a[so:-so, so:-so]
    last = (nt - 1) % 3
    return dict(rec=rec_f, u_last=dom(uf[nt - 1]), srca=srca_t, p=dom(p[0]), born_rec=rec_b, du=dom(du[last]),
                grad=grad)


@pytest.fixture(scope='module')
def restatements():
    return {}


def _restated(cache, name, mut=None):
    if (name, mut) not in cache:
        cache[(name, mut)] = restated(name, mut)
    return cache[(name, mut)]


@pytest.mark.parametrize('name', GOLDENS)
def test_restatement_matches_the_reference(name, restatements):
    g = load_golden(name)
    got = _restated(restatements, name)
    for k in ('rec', 'u_last', 'srca', 'p', 'born_rec', 'du', 'grad'):
        assert rel_linf(got[k], g[k]) < TOL, (name, k, rel_linf(got[k], g[k]))


def _dot_problem(so, seed):
    rng = np.random.default_rng(seed)
    n = (20, 24)
    hs = (10., 8.)
    from devito_b200.operator import half_node_first_derivative_weights, second_derivative_weights
    w2 = [second_derivative_weights(so, h) for h in hs]
    w1 = [half_node_first_derivative_weights(so, h) for h in hs]
    A = tuple(x + 2 * so for x in n)
    gx, gz = np.meshgrid(np.linspace(0, 1, A[0]), np.linspace(0, 1, A[1]), indexing='ij')
    P = dict(vp=1.5 + 0.5 * gx + 0.3 * gz, epsilon=0.1 + 0.1 * gx * gz, delta=0.05 + 0.05 * gz,
             theta=0.3 + 0.6 * gx - 0.4 * gz)
    damp = 0.05 * rng.uniform(size=A)
    return rng, n, A, w2, w1, P, damp


def _undamp(damp, so, *sps):
    """No damping on the support cells: the injection adds dt^2/m after the division by m/dt^2 + damp/dt, so the
    forward and adjoint operators are exact transposes only where damp = 0 there (the reference's layout)."""
    n = [s - 2 * so for s in damp.shape]
    for sp in sps:
        damp[T2._Support(dict(sp, data=np.zeros((1, len(sp['gp'])))), [0, 0], [x - 1 for x in n], so).idx] = 0.0


@pytest.mark.parametrize('so', [4, 8])
def test_dot_test_F(so):
    """<F s, d> = <s, F^T d> for the float64 restatement, with source and receiver supports at random points."""
    rng, n, A, w2, w1, P, damp = _dot_problem(so, 1)
    dt, nt = 0.8, 24
    pts = lambda k: dict(gp=rng.integers(2, min(n) - 3, size=(k, 2)), w=[rng.uniform(size=(k, 2)) for _ in range(2)],
                         r=1)
    S, R = pts(2), pts(5)
    _undamp(damp, so, S, R)
    s = rng.standard_normal((nt, 2))
    d = rng.standard_normal((nt, 5))
    z = np.zeros((3,) + A)
    _, _, _, _, Fs = T2.forward(z, z, so, w2, w1, dt, 1, nt - 2, damp, P, src=dict(S, data=s),
                                rec=dict(R, data=np.zeros((nt, 5))))
    _, _, FTd = T2.adjoint(z, z, so, w2, w1, dt, 1, nt - 2, damp, P, src=dict(R, data=d),
                           rec=dict(S, data=np.zeros((nt, 2))))
    a, b = np.vdot(Fs, d), np.vdot(s, FTd)
    assert abs(a - b) < 1e-10 * max(abs(a), abs(b))


# ---------------------------------------------------------------------------------------------------------------
# GPU: the reference's goldens through the solver
# ---------------------------------------------------------------------------------------------------------------
def _sweep_name(so, arrays, kernel):
    if kernel == 1:
        return 'tti_two_pass'
    return f"tti2d{'_arr' if arrays else ''}<{so // 2}>"


@pytest.mark.gpu
@pytest.mark.parametrize('kernel', [0, 1])
@pytest.mark.parametrize('name', GOLDENS)
def test_goldens_through_the_solver(name, kernel):
    g, model, geometry, solver = _solver(name)
    so, nt = int(g['so']), int(g['nt'])
    arrays = name != 'tti2d_so8'
    sweep = _sweep_name(so, arrays, kernel)
    rec, u0, v0, _ = solver.forward(save=True, kernel=kernel)
    assert _last_kernel() == sweep
    assert rel_linf(rec.data, g['rec']) < TOL
    assert rel_linf(u0.data[nt - 1], g['u_last']) < TOL and rel_linf(v0.data[nt - 1], g['v_last']) < TOL
    rec.data[:] = g['rec']
    srca, p, r, _ = solver.adjoint(rec, kernel=kernel)
    assert _last_kernel() == sweep + '+adj'
    assert rel_linf(srca.data, g['srca']) < TOL
    assert rel_linf(p.data[0], g['p']) < TOL and rel_linf(r.data[0], g['r']) < TOL
    rec.data[:] = g['rec']
    dm, _ = solver.jacobian_adjoint(rec, u0, v0, kernel=kernel)
    assert _last_kernel() == sweep + '+adj'
    assert rel_linf(dm.data, g['grad']) < TOL
    rb, _, _, du, dv, _ = solver.jacobian(g['dm'], kernel=kernel)
    assert _last_kernel() in (sweep + '+born_v4', sweep + '+born_s')
    last = (nt - 1) % 3
    assert rel_linf(rb.data, g['born_rec']) < TOL
    assert rel_linf(du.data[last], g['du']) < TOL and rel_linf(dv.data[last], g['dv']) < TOL


@pytest.mark.gpu
@pytest.mark.parametrize('so', [4, 8])
def test_adjoint_F(so):
    """The reference's tests/test_adjoint.py::test_adjoint_F, `layers-tti` case in 2-D: shape (30, 35), spacing 15,
    nbl 10, tn 500; <F s, d> = <s, F^T d>. The reference runs float64; this backend is float32, so the bound is the
    1e-5 of the 3-D float32 port."""
    from devito_b200.seismic import demo_model, setup_geometry
    from devito_b200.seismic.tti import AnisotropicWaveSolver
    model = demo_model('layers-tti', spacing=(15., 15.), shape=(30, 35), nbl=10, space_order=so, nlayers=3)
    geometry = setup_geometry(model, 500.)
    solver = AnisotropicWaveSolver(model, geometry, space_order=so)
    rec, _, _, _ = solver.forward()
    srca, _, _, _ = solver.adjoint(rec=rec)
    term1 = np.dot(srca.data.reshape(-1).astype(np.float64), geometry.src.data.reshape(-1))
    term2 = np.linalg.norm(rec.data.astype(np.float64)) ** 2
    assert np.isclose((term1 - term2) / term1, 0., atol=1.e-5), (term1, term2)


@pytest.mark.gpu
@pytest.mark.parametrize('so', [4, 8])
def test_adjoint_J(so):
    """The reference's test_adjoint_J, TTI case in 2-D (tests/test_adjoint.py), ported as the 3-D port in
    test_zz_tti_adjoint.py: layers-tti (2 layers, vp 1.5 to 2) on (30, 35), m0 at constant vp 1.5, dm = m - m0;
    <J dm, J dm> = <dm, J^T (J dm)> through solver.jacobian and forward(save=True) + solver.jacobian_adjoint. The
    reference asserts 1e-12 in float64; this backend is float32, so the bound is the 3-D port's 1e-4."""
    from devito_b200.seismic import demo_model, setup_geometry
    from devito_b200.seismic.tti import AnisotropicWaveSolver
    shape, spacing, nbl = (30, 35), (10., 10.), 10 + so // 2
    model = demo_model('layers-tti', nlayers=2, vp_bottom=2, shape=shape, spacing=spacing, nbl=nbl, space_order=so)
    geometry = setup_geometry(model, 500.)
    solver = AnisotropicWaveSolver(model, geometry, space_order=so)
    model0 = demo_model('layers-tti', nlayers=2, vp_top=1.5, vp_bottom=1.5, shape=shape, spacing=spacing, nbl=nbl,
                        space_order=so, grid=model.grid)
    dm = (np.asarray(model.vp.data, np.float64) ** -2 - np.asarray(model0.vp.data, np.float64) ** -2).astype(np.float32)
    assert np.abs(dm).max() > 0
    du = solver.jacobian(dm, model=model0)[0]
    _, u0, v0, _ = solver.forward(save=True, model=model0)
    im, _ = solver.jacobian_adjoint(du, u0, v0, model=model0)
    term1 = np.dot(np.asarray(im.data, np.float64).reshape(-1), dm.astype(np.float64).reshape(-1))
    term2 = np.sum(np.asarray(du.data, np.float64) ** 2)
    assert term2 > 0
    assert abs(term1 - term2) < 1e-4 * abs(term1), (term1, term2)


@pytest.mark.gpu
def test_gradientJ():
    """The reference's tests/test_gradient.py::test_gradientJ, centred TTI in 2-D: shape (70, 80), spacing 20,
    tn 1000, nbl 10 + so/2, m0 a smoothed layered vp and dm = m - m0; |F(m0 + h dm) - F(m0)|_1 has slope 1 and
    |F(m0 + h dm) - F(m0) - h J dm|_1 slope 2 in h, over the reference's seven h, in float32."""
    from devito_b200 import Function
    from devito_b200.builtins import smooth
    from devito_b200.seismic import demo_model, setup_geometry
    from devito_b200.seismic.tti import AnisotropicWaveSolver
    so = 4
    model = demo_model('layers-tti', spacing=(20., 20.), shape=(70, 80), nbl=10 + so // 2, space_order=so, nlayers=3)
    geometry = setup_geometry(model, 1000.)
    wave = AnisotropicWaveSolver(model, geometry, space_order=so)
    v0 = Function(name='v0', grid=model.grid, space_order=so)
    smooth(v0, model.vp)
    v = np.array(model.vp.data)
    dm = (v ** -2 - np.array(v0.data) ** -2).astype(np.float32)
    rec0 = np.array(wave.forward(vp=v0)[0].data)
    Jdm = np.array(wave.jacobian(dm, vp=v0)[0].data)
    H = [0.5, 0.25, .125, 0.0625, 0.0312, 0.015625, 0.0078125]
    e1, e2 = np.zeros(7), np.zeros(7)
    for i, h in enumerate(H):
        vloc = Function(name='vloc', grid=model.grid, space_order=so)
        vloc.data[:] = np.sqrt(np.array(v0.data) ** 2 * v ** 2 / ((1 - h) * v ** 2 + h * np.array(v0.data) ** 2))
        d = np.array(wave.forward(vp=vloc)[0].data)
        delta = (d - rec0).reshape(-1).astype(np.float64)
        e1[i] = np.linalg.norm(delta, 1)
        e2[i] = np.linalg.norm(delta - h * Jdm.reshape(-1), 1)
    p1 = np.polyfit(np.log10(H), np.log10(e1), 1)
    p2 = np.polyfit(np.log10(H), np.log10(e2), 1)
    assert np.isclose(p1[0], 1.0, rtol=0.1), p1[0]
    assert np.isclose(p2[0], 2.0, rtol=0.1), p2[0]


@pytest.mark.gpu
def test_split_time_ranges_and_host_staging_are_bit_identical():
    _, model, geometry, solver = _solver('tti2d_so8_varying')
    rec, u, v, _ = solver.forward()
    whole = (np.array(u.data), np.array(v.data), np.array(rec.data))
    from devito_b200 import TimeFunction
    mk = lambda n: TimeFunction(name=n, grid=model.grid, time_order=2, space_order=solver.space_order)
    u2, v2 = mk('u'), mk('v')
    r2 = geometry.rec
    op = solver.op_fwd()
    kw = dict(model.physical_params())
    nt = geometry.nt
    half = nt // 2
    op.apply(src=geometry.src, rec=r2, u=u2, v=v2, dt=solver.dt, time_m=1, time_M=half, **kw)
    op.apply(src=geometry.src, rec=r2, u=u2, v=v2, dt=solver.dt, time_m=half + 1, time_M=nt - 2, **kw)
    assert np.array_equal(u2.data, whole[0]) and np.array_equal(v2.data, whole[1])
    assert np.array_equal(r2.data, whole[2])
    u3, v3 = mk('u'), mk('v')
    op.apply(src=geometry.src, rec=r2, u=u3, v=v3, dt=solver.dt, resident=False, **kw)
    assert np.array_equal(u3.data, whole[0]) and np.array_equal(v3.data, whole[1])


# ---------------------------------------------------------------------------------------------------------------
# mutations of the restatement, the J / J^T dot test and the emulated point body
# ---------------------------------------------------------------------------------------------------------------
def _noise_case(so, seed=5, n=(20, 24)):
    """White noise in every slot (halo included), parameters varying along both axes and from cell to cell, random
    sparse points and data, dm and the saved wavefields white noise."""
    rng, n, A, w2, w1, P, damp = _dot_problem(so, seed)
    # parameters that change from cell to cell, so that sampling one at the wrong point shows
    P = dict(P, theta=P['theta'] + 0.4 * rng.uniform(size=A), epsilon=P['epsilon'] + 0.2 * rng.uniform(size=A),
             delta=P['delta'] + 0.1 * rng.uniform(size=A))
    K, nt = 4, 8
    f = lambda: rng.standard_normal((3,) + A)
    pts = lambda k: dict(gp=rng.integers(1, min(n) - 2, size=(k, 2)), w=[rng.uniform(size=(k, 2)) for _ in range(2)],
                         r=1, data=rng.standard_normal((nt, k)))
    return dict(so=so, w2=w2, w1=w1, P=P, damp=damp, dt=0.8, K=K, u=f(), v=f(), du=f(), dv=f(),
                dm=0.05 * rng.standard_normal(n), usave=rng.standard_normal((nt,) + A),
                vsave=rng.standard_normal((nt,) + A), src=pts(2), rec=pts(5), n=n)


def _noise_run(c, mut=None):
    a = (c['so'], c['w2'], c['w1'], c['dt'], 1, c['K'], c['damp'], c['P'])
    u, v, du, dv, tr = T2.forward(c['u'], c['v'], *a, src=c['src'], rec=c['rec'], du=c['du'], dv=c['dv'], dm=c['dm'],
                                  mut=mut)
    grad = np.zeros(c['n'])
    p, r, ta = T2.adjoint(c['u'], c['v'], *a, src=c['rec'], rec=c['src'], grad=grad, usave=c['usave'],
                          vsave=c['vsave'], mut=mut)
    return dict(u=u, v=v, du=du, dv=dv, rec=tr, p=p, r=r, srca=ta, grad=grad)


@pytest.mark.parametrize('mut', sorted(T2.MUTATIONS))
def test_restatement_mutations_move_the_result(mut):
    """Each kind of kernel bug moves the fields, traces or gradient by more than 100 times the 1e-4 bound."""
    c = _noise_case(8)
    good, bad = _noise_run(c), _noise_run(c, mut)
    moved = max(rel_linf(bad[k], good[k]) for k in good)
    assert moved > 100 * TOL, (mut, moved)


@pytest.mark.parametrize('so', [4, 8])
def test_dot_test_J(so):
    """<J dm, dd> = <dm, J^T dd> for the float64 restatement: Born (`BornTTI`) against the gradient (`GradientTTI`).
    Exact when the damping is zero everywhere (the Born source is divided by m/dt^2 + damp/dt, the receivers are
    injected with dt^2/m) and the time range's ends carry no energy (the source is zero in its first two samples and
    the data in their last three), so that moving dt2 from u0 onto p by summation by parts leaves no boundary term."""
    rng, n, A, w2, w1, P, damp = _dot_problem(so, 2)
    damp[:] = 0.0
    dt, nt = 0.8, 24
    pts = lambda k: dict(gp=rng.integers(2, min(n) - 3, size=(k, 2)), w=[rng.uniform(size=(k, 2)) for _ in range(2)],
                         r=1)
    S, R = pts(1), pts(5)
    s = np.sin(np.arange(nt)[:, None] * 0.4)
    s[:2] = 0.0
    dm = rng.standard_normal(n)
    dd = rng.standard_normal((nt, 5))
    dd[-3:] = 0.0
    z3, zs = np.zeros((3,) + A), np.zeros((nt,) + A)
    u0, v0, _, _, _ = T2.forward(zs, zs, so, w2, w1, dt, 1, nt - 2, damp, P, src=dict(S, data=s))
    _, _, _, _, Jdm = T2.forward(z3, z3, so, w2, w1, dt, 1, nt - 2, damp, P, src=dict(S, data=s),
                                 rec=dict(R, data=np.zeros((nt, 5))), du=z3, dv=z3, dm=dm)
    grad = np.zeros(n)
    T2.adjoint(z3, z3, so, w2, w1, dt, 1, nt - 2, damp, P, src=dict(R, data=dd), grad=grad, usave=u0, vsave=v0)
    a, b = np.vdot(Jdm, dd), np.vdot(dm, grad)
    assert abs(a) > 0 and abs(a - b) < 1e-10 * max(abs(a), abs(b)), (a, b)


@pytest.fixture(scope='module')
def emu(tmp_path_factory):
    if shutil.which('nvcc') is None:
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp('emu') / 'libemu_tti2d.so'
    subprocess.run(['nvcc', '-O1', '-shared', '-Xcompiler', '-fPIC', '-I', os.path.join(ROOT, 'include'),
                    '-I', os.path.join(ROOT, 'devito_b200', 'csrc'),
                    os.path.join(ROOT, 'tests', 'support', 'emu_tti2d.cu'), '-o', str(out)], check=True)
    lib = ctypes.CDLL(str(out))
    fp, ip = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int)
    lib.emu_tti2d_step.argtypes = [fp, fp, ip, ctypes.c_int] + [fp] * 10 + [ip, ip] + [ctypes.c_int] * 4
    lib.emu_tti2d_step.restype = ctypes.c_int
    return lib


@pytest.mark.parametrize('adj', [0, 1])
@pytest.mark.parametrize('box', ['whole', 'interior'])
@pytest.mark.parametrize('so', [4, 8])
def test_emulated_point_body_matches_the_restatement(emu, so, box, adj):
    """One step of the point forms k_tti2d calls (b2_tti_point.cuh: Gz, the forward / adjoint update with the A form,
    the adjoint's mix), looped on the CPU by tests/support/emu_tti2d.cu, against the float64 restatement."""
    c = _noise_case(so, seed=11)
    n = c['n']
    lo, hi = ([0, 0], [n[0] - 1, n[1] - 1]) if box == 'whole' else ([2, 3], [n[0] - 4, n[1] - 2])
    P, dt = c['P'], c['dt']
    f32 = lambda a: np.ascontiguousarray(np.asarray(a, np.float32))
    md = 1.0 / (P['vp'] * P['vp']) / dt ** 2
    tab = [f32(x) for x in (np.sin(P['theta']), np.cos(P['theta']), 1 + 2 * P['epsilon'], np.sqrt(1 + 2 * P['delta']),
                            md, 1.0 / (md + c['damp'] / dt))]
    u, v = f32(c['u']), f32(c['v'])
    w = [f32(x) for x in (c['w2'][0], c['w2'][1], c['w1'][0], c['w1'][1])]
    fp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    ia = lambda x: (ctypes.c_int * len(x))(*x)
    t0, t2, t1 = (1, 2, 0) if adj else (1, 0, 2)
    assert emu.emu_tti2d_step(fp(u), fp(v), ia(u.shape[1:]), so, *[fp(x) for x in w], *[fp(x) for x in tab], ia(lo),
                              ia(hi), t0, t2, t1, adj) == 0
    a = (so, c['w2'], c['w1'], dt, 1, 1, c['damp'], P)
    ref = T2.adjoint(u, v, *a, lo=lo, hi=hi) if adj else T2.forward(u, v, *a, lo=lo, hi=hi)
    for got, want in ((u, ref[0]), (v, ref[1])):
        assert rel_linf(got[t1], want[t1]) < 1e-5, rel_linf(got[t1], want[t1])


# ---------------------------------------------------------------------------------------------------------------
# look-alikes of the 2-D Born, adjoint and gradient operators
# ---------------------------------------------------------------------------------------------------------------
BORN_LOOKALIKES = ['dt', 'sign', 'factor2', 'swapped', 'one_driven', 'dm_offcentre', 'other_params']


def _born_lookalike(kind):
    """The 2-D BornTTI equations with one deliberate difference."""
    from devito_b200 import Function, Operator, TimeFunction
    from devito_b200.seismic import demo_model, setup_geometry
    from devito_b200.seismic.tti import kernel_centered
    model = demo_model('layers-tti', shape=(16, 18), spacing=(10., 10.), nbl=4, space_order=4, nlayers=2)
    geometry = setup_geometry(model, 40.0)
    grid = model.grid
    dt = grid.stepping_dim.spacing
    mk = lambda n: TimeFunction(name=n, grid=grid, time_order=2, space_order=4)
    u0, v0, du, dv = mk('u0'), mk('v0'), mk('du'), mk('dv')
    dm = Function(name='dm', grid=grid, space_order=0 if kind != 'dm_offcentre' else 1)
    qu, qv = -dm * u0.dt2, -dm * v0.dt2
    lin_model = model
    if kind == 'dt':
        qu, qv = -dm * u0.dt, -dm * v0.dt
    elif kind == 'sign':
        qu, qv = dm * u0.dt2, dm * v0.dt2
    elif kind == 'factor2':
        qu, qv = -2 * dm * u0.dt2, -2 * dm * v0.dt2
    elif kind == 'swapped':
        qu, qv = -dm * v0.dt2, -dm * u0.dt2
    elif kind == 'one_driven':
        qv = 0
    elif kind == 'dm_offcentre':
        x = grid.dimensions[0]
        qu, qv = -dm.subs(x, x + 1) * u0.dt2, -dm.subs(x, x + 1) * v0.dt2
    elif kind == 'other_params':
        lin_model = demo_model('layers-tti', shape=(16, 18), spacing=(10., 10.), nbl=4, space_order=4, nlayers=2)
    src, rec = geometry.src, geometry.rec
    eqs = kernel_centered(model, u0, v0) + src.inject(field=(u0.forward, v0.forward), expr=src * dt ** 2 / model.m)
    eqs = eqs + kernel_centered(lin_model, du, dv, qu=qu, qv=qv) + rec.interpolate(expr=du + dv)
    return Operator(eqs, subs=model.spacing_map)


ADJ_LOOKALIKES = ['mix_at_output', 'mix_swap', 'img_sign', 'img_single', 'img_dt', 'img_buffered']


def _adj_lookalike(kind):
    """A 2-D backward TTI pair (array-valued parameters) with one deviation from the reference's formulation."""
    from devito_b200 import Eq, Function, Grid, Inc, Operator, TimeFunction, solve, sqrt
    from devito_b200.seismic.tti import Gzz_centered_2d
    from types import SimpleNamespace
    grid = Grid(shape=(12, 14), extent=(110., 130.))
    so = 4
    P = {}
    for i, n in enumerate(('vp', 'epsilon', 'delta', 'theta')):
        P[n] = Function(name=n, grid=grid, space_order=so)
        P[n].data[:] = 0.1 + 0.05 * i
    damp = Function(name='damp', grid=grid, space_order=so)
    model = SimpleNamespace(theta=P['theta'], grid=grid)
    mk = lambda n, save=None: TimeFunction(name=n, grid=grid, time_order=2, space_order=so, save=save)
    p, r = mk('p'), mk('r')
    m = 1 / (P['vp'] * P['vp'])
    e2, sd = 1 + 2 * P['epsilon'], sqrt(1 + 2 * P['delta'])
    gzz = lambda f: Gzz_centered_2d(model, f)
    gh = lambda f: f.laplace - gzz(f)
    if kind == 'mix_at_output':
        H0, Hz = e2 * gh(p) + sd * gh(r), sd * gzz(p) + gzz(r)
    elif kind == 'mix_swap':
        H0, Hz = gh(sd * p + r), gzz(e2 * p + sd * r)
    else:
        H0, Hz = gh(e2 * p + sd * r), gzz(sd * p + r)
    eqs = [Eq(p.backward, solve(m * p.dt2 - H0 + damp * p.dt.T, p.backward)),
           Eq(r.backward, solve(m * r.dt2 - Hz + damp * r.dt.T, r.backward))]
    if kind.startswith('img') or kind == 'grad':
        u0, v0 = mk('u0', 10), mk('v0', None if kind == 'img_buffered' else 10)
        dm = Function(name='dm', grid=grid)
        expr = {'img_sign': u0 * p.dt2 + v0 * r.dt2, 'img_single': -(u0 * p.dt2),
                'img_dt': -(u0 * p.dt + v0 * r.dt)}.get(kind, -(u0 * p.dt2 + v0 * r.dt2))
        eqs.append(Inc(dm, expr))
    return Operator(eqs)


def test_born_and_adjoint_lookalike_builders_accept_the_reference_formulation():
    for op in (_born_lookalike('none'), _adj_lookalike('none'), _adj_lookalike('grad')):
        assert op.backend == 'cuda-sm90a', op._why_not


@pytest.mark.parametrize('kind', BORN_LOOKALIKES)
def test_born_lookalikes_are_refused(kind):
    from devito_b200 import InvalidOperator
    try:
        op = _born_lookalike(kind)
    except (InvalidOperator, NotImplementedError, KeyError, ValueError):
        return
    assert op.backend == 'numpy-interpreter', kind


@pytest.mark.parametrize('kind', ADJ_LOOKALIKES)
def test_adjoint_and_imaging_lookalikes_are_refused(kind):
    from devito_b200 import InvalidOperator
    try:
        op = _adj_lookalike(kind)
    except (InvalidOperator, NotImplementedError, KeyError, ValueError):
        return
    assert op.backend == 'numpy-interpreter', kind


# ---------------------------------------------------------------------------------------------------------------
# GPU: every 2-D sweep variant against the float64 restatement
# ---------------------------------------------------------------------------------------------------------------
MATRIX = ([(so, preset, box, 0) for so in (4, 8) for preset in ('constant-tti', 'layers-tti')
           for box in ('whole', 'interior', 'tiny1x5', 'tiny3x1')] +
          [(so, preset, 'whole', 1) for so in (4, 8, 12) for preset in ('constant-tti', 'layers-tti')])
# update boxes (lo, hi) in (x, z) by grid shape; the tiny ones start at z = 4 (z_m % 4 == 0: the single-pass sweep,
# which has no size gate, takes them)
BOXES_2D = {
    'whole': lambda nx, nz: ([0, 0], [nx - 1, nz - 1]),
    'interior': lambda nx, nz: ([3, 4], [nx - 5, nz - 7]),
    'tiny1x5': lambda nx, nz: ([3, 4], [3, 8]),
    'tiny3x1': lambda nx, nz: ([3, 4], [5, 4]),
}


@pytest.mark.gpu
@pytest.mark.parametrize('so,preset,box,kernel', MATRIX)
def test_kernel_matrix_against_float64(so, preset, box, kernel):
    """Forward, adjoint, Born and gradient through the solver from white-noise fields (every slot, halo included)
    against tests/tti2d_ref.py, below 1e-4. kernel 0 takes the single-pass sweep on a z extent of three segments, the
    last one partial (1148 + 2 nbl points), and several x chunks, on the whole box, an interior box and boxes of
    1 x 5 and 3 x 1 points; kernel 1 (and so=12, which only the two-pass path runs) the two-pass sweep. Each case
    asserts the variant that ran."""
    from devito_b200 import Function, TimeFunction
    from devito_b200.operator import half_node_first_derivative_weights, second_derivative_weights
    from devito_b200.seismic import demo_model, setup_geometry
    from devito_b200.seismic.tti import AnisotropicWaveSolver
    kw = {'nlayers': 3} if preset == 'layers-tti' else {}
    model = demo_model(preset, spacing=(10., 8.), shape=(90, 1148), nbl=10, space_order=so, **kw)
    geometry = setup_geometry(model, 12.)
    solver = AnisotropicWaveSolver(model, geometry, space_order=so)
    arrays = preset == 'layers-tti'
    nx, nz = model.grid.shape
    lo, hi = BOXES_2D[box](nx, nz)
    lim = {} if box == 'whole' else dict(x_m=lo[0], x_M=hi[0], y_m=lo[1], y_M=hi[1])
    K, dt = 3, float(solver.dt)
    rng = np.random.default_rng(so + 7 * kernel + (box == 'whole'))
    hs = [float(h) for h in model.spacing]
    w2 = [second_derivative_weights(so, h) for h in hs]
    w1 = [half_node_first_derivative_weights(so, h) for h in hs]
    shp = model.damp.data_with_halo.shape
    P = {}
    for k in ('vp', 'epsilon', 'delta', 'theta'):
        f = getattr(model, k)
        P[k] = np.array(f.data_with_halo, np.float64) if hasattr(f, 'data_with_halo') else np.full(shp, float(f.data))
    damp = np.array(model.damp.data_with_halo, np.float64)
    tab = lambda sf, data: dict(gp=sf.tabulate()[0], w=sf.tabulate()[1], r=sf.r, data=np.array(data, np.float64))
    sweep = _sweep_name(so, arrays, 1 if so == 12 else kernel)

    def tf(name, save=None):
        f = TimeFunction(name=name, grid=model.grid, time_order=2, space_order=so, save=save)
        f.data_with_halo[:] = rng.standard_normal(f.data_with_halo.shape).astype(np.float32)
        return f
    src, rec = geometry.src, geometry.rec
    src.data[:] = rng.standard_normal(src.data.shape).astype(np.float32)
    a64 = (so, w2, w1, dt, 1, K, damp, P)
    run = dict(time_m=1, time_M=K, kernel=kernel, dt=dt, **lim)
    # forward
    u, v = tf('u'), tf('v')
    want = T2.forward(u.data_with_halo, v.data_with_halo, *a64, lo=lo, hi=hi, src=tab(src, src.data),
                      rec=tab(rec, np.zeros(rec.data.shape)))
    solver.forward(src=src, rec=rec, u=u, v=v, **run)
    assert _last_kernel() == sweep
    for got, w in ((u.data_with_halo, want[0]), (v.data_with_halo, want[1]), (rec.data[1:K + 1], want[4][1:K + 1])):
        assert rel_linf(got, w) < TOL, ('forward', rel_linf(got, w))
    # adjoint
    rec.data[:] = rng.standard_normal(rec.data.shape).astype(np.float32)
    p, r = tf('p'), tf('r')
    srca = geometry.new_src(name='srca', src_type=None)
    want = T2.adjoint(p.data_with_halo, r.data_with_halo, *a64, lo=lo, hi=hi, src=tab(rec, rec.data),
                      rec=tab(srca, np.zeros(srca.data.shape)))
    solver.adjoint(rec, srca=srca, p=p, r=r, **run)
    assert _last_kernel() == sweep + '+adj'
    for got, w in ((p.data_with_halo, want[0]), (r.data_with_halo, want[1]), (srca.data[1:K + 1], want[2][1:K + 1])):
        assert rel_linf(got, w) < TOL, ('adjoint', rel_linf(got, w))
    # Born
    u0, v0, du, dv = tf('u0'), tf('v0'), tf('du'), tf('dv')
    dm = Function(name='dm', grid=model.grid, space_order=0)
    dm.data[:] = (0.05 * rng.standard_normal(dm.data.shape)).astype(np.float32)
    want = T2.forward(u0.data_with_halo, v0.data_with_halo, *a64, lo=lo, hi=hi, src=tab(src, src.data),
                      rec=tab(rec, np.zeros(rec.data.shape)), du=du.data_with_halo, dv=dv.data_with_halo,
                      dm=np.array(dm.data))
    solver.jacobian(dm, src=src, rec=rec, u0=u0, v0=v0, du=du, dv=dv, **run)
    assert _last_kernel().startswith(sweep + '+born_')
    for got, w in ((u0.data_with_halo, want[0]), (du.data_with_halo, want[2]), (dv.data_with_halo, want[3]),
                   (rec.data[1:K + 1], want[4][1:K + 1])):
        assert rel_linf(got, w) < TOL, ('born', rel_linf(got, w))
    # gradient
    rec.data[:] = rng.standard_normal(rec.data.shape).astype(np.float32)
    us, vs = tf('u0', save=geometry.nt), tf('v0', save=geometry.nt)
    du, dv = tf('du'), tf('dv')
    grad = Function(name='dm', grid=model.grid)
    g64 = np.zeros(model.grid.shape)
    want = T2.adjoint(du.data_with_halo, dv.data_with_halo, *a64, lo=lo, hi=hi, src=tab(rec, rec.data), grad=g64,
                      usave=us.data_with_halo, vsave=vs.data_with_halo)
    solver.jacobian_adjoint(rec, us, vs, du=du, dv=dv, dm=grad, **run)
    assert _last_kernel() == sweep + '+adj'
    for got, w in ((du.data_with_halo, want[0]), (grad.data, g64)):
        assert rel_linf(got, w) < TOL, ('gradient', rel_linf(got, w))


@pytest.mark.gpu
def test_forced_single_pass_on_a_layout_that_does_not_qualify_fails():
    """kernel=2 on a z extent that is not a multiple of 4 fails with 210 and a message, instead of running another
    kernel."""
    from devito_b200 import ExecutionError
    from devito_b200.seismic import demo_model, setup_geometry
    from devito_b200.seismic.tti import AnisotropicWaveSolver
    model = demo_model('constant-tti', spacing=(10., 10.), shape=(40, 41), nbl=10, space_order=8)
    solver = AnisotropicWaveSolver(model, setup_geometry(model, 20.), space_order=8)
    with pytest.raises(ExecutionError, match='210.*does not qualify'):
        solver.forward(kernel=2)
    solver.forward(kernel=0)
    assert _last_kernel() == 'tti_two_pass'


@pytest.mark.gpu
@pytest.mark.parametrize('member', ['phi', 'phi_arr', 'halo'])
def test_2d_call_with_an_azimuth_or_halo_exchange_fails(member, monkeypatch):
    """A 2-D b2_tti_forward call with phi != 0, a phi array or a halo context returns 210 (the recogniser never builds
    one; the block is altered just before the call)."""
    from devito_b200 import ExecutionError
    from devito_b200.operator import Operator
    _, _, _, solver = _solver('tti2d_so4_layers')
    call = Operator._call

    def altered(self, L, symbol, a, args, dev, post=()):
        if member == 'phi':
            a.phi = 0.3
        elif member == 'phi_arr':
            a.phi_arr = a.vp_arr
        else:
            a.halo = ctypes.c_void_p(8)
        return call(self, L, symbol, a, args, dev, post)
    monkeypatch.setattr(Operator, '_call', altered)
    with pytest.raises(ExecutionError, match='210.*no azimuth'):
        solver.forward()
