"""Centred-TTI linearised (Born) modelling — the reference's `BornTTI` operator / `solver.jacobian(dm)`
(examples/seismic/tti/operators.py:532-586, tti/wavesolver.py:232-293).

CPU: recognition of the reference's formulation and refusal of look-alikes, the C adapter's new fields, the C oracle
against the reference goldens, the float64 reference against the oracle on the anisotropic kernel-matrix grid, the
sensitivity of that comparison to each kind of kernel bug, and the point body of the Born source term run on the CPU.
GPU: `b2_tti_args.born_du/born_dv/born_dm` against the goldens, dm = 0, the background pair against the forward
operator, linearity, the reference's Taylor test, restart and host staging. The sweep-variant matrix is
tests/test_tti_born_matrix.py.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from helpers import load_golden, rel_linf
import kernel_cases as KC
import ref64
import tti_born_ref as TB
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDENS = [('tti_born3d_so8', 'constant-tti', 8, {}), ('tti_born3d_so4_layers', 'layers-tti', 4, {'nlayers': 3})]
TOL = 1e-4
PNAMES = ('vp', 'epsilon', 'delta', 'theta', 'phi')


def _solver(name, preset, so, kw):
    from devito_b200.seismic import demo_model, setup_geometry
    from devito_b200.seismic.tti import AnisotropicWaveSolver
    g = load_golden(name)
    n, nbl = int(g['n']), int(g['nbl'])
    model = demo_model(preset, shape=(n,) * 3, spacing=(10.,) * 3, nbl=nbl, space_order=so, **kw)
    geometry = setup_geometry(model, float(g['tn']))
    assert geometry.nt == int(g['nt']) and np.float32(model.critical_dt) == g['dt']
    N = n + 2 * nbl
    c = N // 2
    assert np.array_equal(np.broadcast_to(np.asarray(model.vp.data), (N,) * 3)[c, c, :], g['vp_line'])
    g['dm'] = _golden_dm(N)
    assert abs(g['dm'].astype(np.float64).sum() - float(g['dm_sum'])) < 1e-9 * float(g['dm_sum'])
    return g, model, geometry, AnisotropicWaveSolver(model, geometry, space_order=so)


def _golden_dm(N):
    """The model perturbation of the goldens (oracle/make_golden_tti_born.py::dm_blob)."""
    ax = np.arange(N, dtype=np.float64)
    X, Y, Z = np.meshgrid(ax, ax, ax, indexing='ij')
    c = (N - 1) / 2.0
    return (0.05 * np.exp(-((X - c) ** 2 + (Y - c) ** 2 + (Z - c - 2) ** 2) / (2 * 4.0 ** 2))).astype(np.float32)


def _golden_view(g, a):
    """What the goldens hold of a wavefield given as (3, N, N, N) domain data: the last level written, on every
    second point."""
    return np.asarray(a)[int(g['slot'])][::2, ::2, ::2]


# ---------------------------------------------------------------------------------------------------------------
# recognition
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name,preset,so,kw', GOLDENS, ids=[x[0] for x in GOLDENS])
def test_jacobian_is_recognised(name, preset, so, kw):
    g, model, geometry, solver = _solver(name, preset, so, kw)
    op = solver.op_jac()
    assert op.name == 'BornTTI'
    assert op.backend == 'cuda-sm90a', op._why_not
    p = op._plan
    assert p['kind'] == 'tti'
    assert [p[k].name for k in ('u', 'v', 'born_du', 'born_dv', 'born_dm')] == ['u0', 'v0', 'du', 'dv', 'dm']
    assert p['src'].name == 'src' and p['rec'].name == 'rec' and p['rec_toff'] == 0
    args = op.arguments(dm=np.ascontiguousarray(g['dm']), dt=float(model.critical_dt))
    assert args['born_dm'].storage.host.shape == model.grid.shape
    text = str(op)
    for f in ('du', 'dv', 'dm'):
        assert f'a.born_{f} = (struct b2_dataobj *){f}_vec;' in text
    assert 'struct dataobj *restrict dm_vec' in text


def test_forward_equations_unchanged():
    """kernel_centered without qu / qv builds exactly the forward equations it built before."""
    from devito_b200 import TimeFunction, solve, sqrt
    from devito_b200.seismic import demo_model
    from devito_b200.seismic.tti import Gzz_centered, kernel_centered
    model = demo_model('layers-tti', shape=(12,) * 3, spacing=(10.,) * 3, nbl=4, space_order=4)
    u = TimeFunction(name='u', grid=model.grid, time_order=2, space_order=4)
    v = TimeFunction(name='v', grid=model.grid, time_order=2, space_order=4)
    d, e = sqrt(1 + 2 * model.delta), 1 + 2 * model.epsilon
    gxx = u.laplace - Gzz_centered(model, u)
    gzz = Gzz_centered(model, v)
    m, damp = model.m, model.damp
    want = [solve(m * u.dt2 - (e * gxx + d * gzz) + damp * u.dt, u.forward),
            solve(m * v.dt2 - (d * gxx + gzz) + damp * v.dt, v.forward)]
    got = kernel_centered(model, u, v)
    assert [str(x.rhs) for x in got] == [str(x) for x in want]


def _lookalike(kind):
    """The BornTTI equations with one deliberate difference."""
    from devito_b200 import Eq, Function, FreeSurface, Inc, Operator, TimeFunction
    from devito_b200.seismic import demo_model, setup_geometry
    from devito_b200.seismic.tti import kernel_centered
    model = demo_model('layers-tti', shape=(16,) * 3, spacing=(10.,) * 3, nbl=4, space_order=4, nlayers=2)
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
        lin_model = demo_model('layers-tti', shape=(16,) * 3, spacing=(10.,) * 3, nbl=4, space_order=4, nlayers=2)
    eqs = kernel_centered(model, u0, v0)
    if kind == 'backward':
        eqs = [Eq(e.lhs.subs(grid.stepping_dim, grid.stepping_dim - 2), e.rhs) for e in eqs]
    src, rec = geometry.src, geometry.rec
    eqs = eqs + src.inject(field=(u0.forward, v0.forward), expr=src * dt ** 2 / model.m)
    lin = kernel_centered(lin_model, du, dv, qu=qu, qv=qv)
    eqs = eqs + lin + rec.interpolate(expr=du + dv)
    if kind == 'increment':
        eqs.append(Inc(Function(name='grad', grid=grid), -u0 * dv.dt2))
    elif kind == 'snapshot':
        from devito_b200 import ConditionalDimension
        t_sub = ConditionalDimension('t_sub', parent=grid.time_dim, factor=2)
        us = TimeFunction(name='usave', grid=grid, time_order=2, space_order=4, save=10, time_dim=t_sub)
        eqs.append(Eq(us, u0))
    elif kind == 'free_surface':
        e = lin[0]
        eqs.append(FreeSurface(e, grid.subdomains['physdomain']))
    return Operator(eqs, subs=model.spacing_map)


def test_reference_formulation_through_lookalike_builder():
    op = _lookalike('none')
    assert op.backend == 'cuda-sm90a', op._why_not


LOOKALIKES = ['dt', 'sign', 'factor2', 'swapped', 'one_driven', 'dm_offcentre', 'other_params', 'backward',
              'increment', 'snapshot', 'free_surface']


@pytest.mark.parametrize('kind', LOOKALIKES)
def test_lookalikes_are_refused(kind):
    from devito_b200 import InvalidOperator
    try:
        op = _lookalike(kind)
    except (InvalidOperator, NotImplementedError, KeyError, ValueError):
        return              # refused outright (a free surface has no interpreter to fall back to)
    assert op.backend == 'numpy-interpreter', kind


def test_cinterface_recording_double_sees_the_born_fields(tmp_path):
    """The generated adapter, compiled against a recording stub of b2_tti_forward, passes the three new fields."""
    if shutil.which('gcc') is None:
        pytest.skip("gcc not available")
    from devito_b200.seismic import demo_model, setup_geometry
    from devito_b200.seismic.tti import JacobianOperator
    from devito_b200 import cinterface as ci
    model = demo_model('constant-tti', shape=(12,) * 3, spacing=(10.,) * 3, nbl=4, space_order=4)
    op = JacobianOperator(model, setup_geometry(model, 20.0), space_order=4)
    ccode, hcode = ci.generate(op._plan, 'BornTTI')
    (tmp_path / 'BornTTI.c').write_text(ccode)
    (tmp_path / 'BornTTI.h').write_text(hcode)
    (tmp_path / 'stub.c').write_text('''#include "b200stencil.h"
static const struct b2_tti_args *g_seen;
static void *g_du, *g_dv, *g_dm;
int b2_tti_forward(const struct b2_tti_args *a) { g_du = a->born_du; g_dv = a->born_dv; g_dm = a->born_dm;
  return 0; }
void *seen(int i) { return i == 0 ? g_du : (i == 1 ? g_dv : g_dm); }
''')
    so = tmp_path / 'libborn.so'
    # -Bsymbolic: the adapter calls the stub in its own library even when the real libb200stencil.so is already
    # loaded into the process with global symbols
    subprocess.run(['gcc', '-shared', '-fPIC', '-Wl,-Bsymbolic', '-I', os.path.join(ROOT, 'include'), '-I', str(tmp_path), '-o',
                    str(so), str(tmp_path / 'BornTTI.c'), str(tmp_path / 'stub.c')], check=True)
    lib = ctypes.CDLL(str(so))
    params = ci.signature(op._plan, 'BornTTI')
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
    assert getattr(lib, 'BornTTI')(*argv) == 0
    lib.seen.restype = ctypes.c_void_p
    for i, n in enumerate(('du_vec', 'dv_vec', 'dm_vec')):
        assert lib.seen(i) == ctypes.cast(objs[n], ctypes.c_void_p).value


# ---------------------------------------------------------------------------------------------------------------
# the C oracle against the reference, the float64 restatement against the oracle
# ---------------------------------------------------------------------------------------------------------------
def _sparse_tables(sf, data):
    gp, ws = sf.tabulate()
    return dict(data=np.ascontiguousarray(data, dtype=np.float32), gp=gp, w=ws, r=sf.r)


@pytest.mark.parametrize('name,preset,so,kw', GOLDENS, ids=[x[0] for x in GOLDENS])
def test_oracle_vs_reference_golden(name, preset, so, kw):
    g, model, geometry, _ = _solver(name, preset, so, kw)
    assert np.allclose(np.asarray(geometry.src.data)[:, 0], g['src'][:, 0])
    nt = int(g['nt'])
    dt = float(g['dt'])
    from devito_b200 import Function
    alloc = tuple(s + 2 * so for s in model.grid.shape)
    u, v, du, dv = (np.zeros((3,) + alloc, dtype=np.float32) for _ in range(4))
    src = _sparse_tables(geometry.src, g['src'])
    rec = _sparse_tables(geometry.rec, np.zeros_like(g['rec']))
    arrays = {}
    scal = {}
    for n in PNAMES:
        p = getattr(model, n)
        if isinstance(p, Function):
            assert p.space_order == so
            arrays[n] = np.ascontiguousarray(p.data_with_halo, dtype=np.float32)
            scal[n] = 0.0 if n != 'vp' else 1.0
        else:
            scal[n] = float(p.data)
    damp = np.ascontiguousarray(model.damp.data_with_halo, dtype=np.float32)
    assert damp.shape == alloc
    w2 = [O.fd2_weights(so, 10.0)] * 3
    w1 = [O.fd1_half_weights(so, 10.0)] * 3
    TB.oracle_tti_born_forward(u, v, du, dv, g['dm'], so, w2, w1, dt, 1, nt - 2, damp, scal['vp'], scal['epsilon'],
                               scal['delta'], scal['theta'], scal['phi'], src=src, rec=rec, arrays=arrays)
    dom = (slice(None),) + (slice(so, -so),) * 3
    for got, n in ((u, 'u0'), (v, 'v0'), (du, 'du'), (dv, 'dv')):
        assert rel_linf(_golden_view(g, got[dom]), g[n]) < TOL, n
    assert rel_linf(rec['data'], g['rec']) < TOL
    assert np.abs(g['du']).max() > 0 and np.abs(g['rec']).max() > 0


def born_case(so, arrays, box=None, dmh=0):
    import test_tti_born_matrix as M
    return M.born_case(so, arrays, box, dmh)


def _oracle_case(c, tables):
    so = c['so']
    _, (w2, w1) = KC.weights('tti', so)
    u, v, du, dv = (np.array(c[k]) for k in ('u', 'v', 'du', 'dv'))
    rec = dict(tables, data=np.zeros_like(tables['data']))
    P = c['params']
    arr = {n: np.asarray(x) for n, x in P.items() if np.ndim(x)}
    scal = {n: (float(x) if not np.ndim(x) else (1.0 if n == 'vp' else 0.0)) for n, x in P.items()}
    TB.oracle_tti_born_forward(u, v, du, dv, c['dm'], so, w2, w1, c['dt'], 1, KC.K, c['damp'], scal['vp'],
                               scal['epsilon'], scal['delta'], scal['theta'], scal['phi'], src=tables, rec=rec,
                               dmhalo=c['dmh'], lo=c['lo'], hi=c['hi'], arrays=arr)
    return dict(u0=u, v0=v, du=du, dv=dv, rec=rec['data'])


def _ref(c, tables, mut=None):
    (w2, w1), _ = KC.weights('tti', c['so'])
    rec = dict(tables, data=np.zeros_like(tables['data']))
    u, v, du, dv, tr = TB.tti_born_forward(c['u'], c['v'], c['du'], c['dv'], c['dm'], c['dmh'], c['so'], w2, w1,
                                           c['dt'], 1, KC.K, c['damp'], c['params'], lo=c['lo'], hi=c['hi'],
                                           src=tables, rec=rec, mut=mut)
    return dict(u0=u, v0=v, du=du, dv=dv, rec=tr)


def _tables(so):
    return KC.sparse_tables(KC.sparse_coordinates(), 'sinc' if so >= 8 else 'linear', KC.K + 2)


@pytest.mark.parametrize('box', ['full', 'sub'])
@pytest.mark.parametrize('arrays', [False, True], ids=['scalar', 'arrays'])
@pytest.mark.parametrize('so', [4, 8])
def test_float64_vs_oracle(so, arrays, box):
    c = born_case(so, arrays, KC.SUBBOX if box == 'sub' else None, dmh=3)
    tables = _tables(so)
    got = _oracle_case(c, tables)
    want = _ref(c, tables)
    for n in ('u0', 'v0', 'du', 'dv', 'rec'):
        err = rel_linf(got[n], want[n])
        assert err < TOL, f"{n}: {err:.2e}"


MUTATIONS = ['born_before_inject', 'born_dm_shift', 'tti_born_swap', 'w_xy', 'w_yz', 'transpose_xy', 'halo_zero',
             'shift_x', 'shift_z', 'c_at_output', 'tail_y', 'tail_z', 'swap_levels']


@pytest.mark.parametrize('mut', MUTATIONS)
def test_mutations_move_the_result(mut):
    """Each kind of kernel bug moves du, dv or the traces by at least 100 times the tolerance."""
    # rotation factors sampled at the wrong point only differ with array parameters; the halo is read across the
    # faces of the full box
    arrays = mut.startswith('shift') or mut == 'c_at_output'
    c = born_case(8, arrays, None if mut == 'halo_zero' else KC.SUBBOX, dmh=3)
    tables = _tables(8)
    good = _ref(c, tables)
    bad = _ref(c, tables, mut=mut)
    moved = max(rel_linf(bad[n], good[n]) for n in ('du', 'dv', 'rec'))
    assert moved > 100 * TOL, f"{mut}: {moved:.2e}"


# ---------------------------------------------------------------------------------------------------------------
# the point body of k_tti_born_src on the CPU (tests/support/emu_tti_born.cu)
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def emu(tmp_path_factory):
    if shutil.which('nvcc') is None:
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp('emu') / 'libemu_tti_born.so'
    cmd = ['nvcc', '-O1', '-shared', '-Xcompiler', '-fPIC', '-I', os.path.join(ROOT, 'include'),
           '-I', os.path.join(ROOT, 'devito_b200', 'csrc'), os.path.join(ROOT, 'tests', 'support', 'emu_tti_born.cu'),
           '-o', str(out)]
    subprocess.run(cmd, check=True, capture_output=True)
    lib = ctypes.CDLL(str(out))
    fp, ip = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int)
    lib.emu_tti_born_source.argtypes = [fp, fp, fp, fp, fp, ip, ctypes.c_int, ip, ctypes.c_int, fp, fp, fp,
                                        ctypes.c_float, ctypes.c_float, ip, ip, ctypes.c_int, ctypes.c_int,
                                        ctypes.c_int]
    lib.emu_tti_born_source.restype = ctypes.c_int
    return lib


def _fp(a):
    return None if a is None else a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def _ip(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))


@pytest.mark.parametrize('table', [False, True], ids=['den', 'A'])
@pytest.mark.parametrize('dmh', [0, 3])
@pytest.mark.parametrize('box', ['full', 'sub'])
@pytest.mark.parametrize('param', ['scalar', 'vp'])
def test_emulated_born_source(emu, param, box, dmh, table):
    """The Born source term on white noise, with the tabulated A or the denominator computed from m/dt^2 (scalar vp
    or a table of m/dt^2) and damp, against float64."""
    so = 8
    c = born_case(so, param == 'vp', KC.SUBBOX if box == 'sub' else None, dmh)
    vp = c['params']['vp']
    t0, t2, t1 = 1, 0, 2
    lo, hi = np.array(c['lo'], dtype=np.int32), np.array(c['hi'], dtype=np.int32)
    u, v = np.array(c['u']), np.array(c['v'])
    du, dv = np.array(c['du']), np.array(c['dv'])
    dt = c['dt']
    md = None
    if np.ndim(vp):
        md = (np.float32(1.0 / (dt * dt)) / (vp * vp)).astype(np.float32)
    damp = c['damp']
    A = None
    if table:
        mdv = md if md is not None else np.float32(1.0 / (float(vp) ** 2) / dt ** 2)
        A = (1.0 / (mdv + damp * np.float32(1.0 / dt))).astype(np.float32) * np.ones_like(damp)
    alloc = np.array(u.shape[1:], dtype=np.int32)
    dmalloc = np.array(c['dm'].shape, dtype=np.int32)
    rc = emu.emu_tti_born_source(_fp(u), _fp(v), _fp(du), _fp(dv), _fp(c['dm']), _ip(dmalloc), dmh, _ip(alloc), so,
                                 _fp(A), _fp(md), _fp(damp), float(vp) if not np.ndim(vp) else 1.0, dt, _ip(lo),
                                 _ip(hi), t0, t2, t1)
    assert rc == 0
    box_ = ref64._box(c['lo'], c['hi'], so)
    dmb = np.asarray(c['dm'], dtype=np.float64)[ref64._box(c['lo'], c['hi'], dmh)]
    m = 1.0 / np.asarray(vp, dtype=np.float64) ** 2
    den = (m[box_] if np.ndim(m) else m) / dt ** 2 + damp.astype(np.float64)[box_] / dt
    for f, got, base in ((c['du'], du, c['u']), (c['dv'], dv, c['v'])):
        b = base.astype(np.float64)
        want = f[2].astype(np.float64)
        want[box_] += -dmb * (b[t1][box_] - 2 * b[t0][box_] + b[t2][box_]) / dt ** 2 / den
        assert rel_linf(got[2], want) < 1e-6
        assert np.array_equal(got[:2], f[:2])


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
def _last_kernel():
    from devito_b200 import _lib
    return _lib.lib().b2_last_sweep_kernel().decode()


@pytest.mark.gpu
@pytest.mark.parametrize('name,preset,so,kw', GOLDENS, ids=[x[0] for x in GOLDENS])
def test_jacobian_vs_reference_golden(name, preset, so, kw):
    from devito_b200 import Function
    g, model, geometry, solver = _solver(name, preset, so, kw)
    rec, u0, v0, du, dv, _ = solver.jacobian(np.ascontiguousarray(g['dm']))
    assert '+born_' in _last_kernel()
    for f, n in ((u0, 'u0'), (v0, 'v0'), (du, 'du'), (dv, 'dv')):
        assert rel_linf(_golden_view(g, f.data), g[n]) < TOL, n
    assert rel_linf(rec.data, g['rec']) < TOL
    dmf = Function(name='dm', grid=model.grid, space_order=0)
    dmf.data[:] = g['dm']
    _, _, _, du2, dv2, _ = solver.jacobian(dmf)
    assert np.array_equal(np.asarray(du2.data), np.asarray(du.data))
    assert np.array_equal(np.asarray(dv2.data), np.asarray(dv.data))


def _small(preset='layers-tti', so=8):
    from devito_b200.seismic import demo_model, setup_geometry
    from devito_b200.seismic.tti import AnisotropicWaveSolver
    kw = {'nlayers': 3} if preset == 'layers-tti' else {}
    model = demo_model(preset, shape=(32, 36, 40), spacing=(10., 12.5, 8.), nbl=8, space_order=so, **kw)
    # long enough for the wavefield to cross the dm blob: du is then far from the subnormal range
    geometry = setup_geometry(model, 250.0)
    return model, AnisotropicWaveSolver(model, geometry, space_order=so)


def _blob(model, scale=0.05, shift=0.0):
    N = model.grid.shape
    X, Y, Z = np.meshgrid(*[np.arange(n, dtype=np.float64) for n in N], indexing='ij')
    c = [(n - 1) / 2.0 + shift for n in N]
    return (scale * np.exp(-((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2] - 2) ** 2) / 32.0)).astype(np.float32)


def _jac(solver, dm, **kw):
    rec, u0, v0, du, dv, _ = solver.jacobian(dm, **kw)
    return {n: np.array(f.data) for n, f in (('rec', rec), ('u0', u0), ('v0', v0), ('du', du), ('dv', dv))}


@pytest.mark.gpu
@pytest.mark.parametrize('preset', ['constant-tti', 'layers-tti'])
def test_zero_dm_and_background_equals_forward(preset):
    model, solver = _small(preset)
    dm = _blob(model)
    z = _jac(solver, np.zeros_like(dm))
    assert not z['du'].any() and not z['dv'].any() and not z['rec'].any()
    j = _jac(solver, dm)
    assert np.abs(j['du']).max() > 0 and np.abs(j['rec']).max() > 0
    rec, u, v, _ = solver.forward()
    assert np.array_equal(j['u0'], np.asarray(u.data)) and np.array_equal(j['v0'], np.asarray(v.data))
    assert np.array_equal(z['u0'], np.asarray(u.data))


@pytest.mark.gpu
def test_linearity():
    """J(2 dm) = 2 J(dm) and J(dm1 + dm2) = J(dm1) + J(dm2) up to float32 rounding. Doubling dm is exact only
    until the leading edge of the wavefield, where u.dt2 and du are subnormal, rounds differently; from there
    the differences grow like any rounding difference. The C oracle, in the reference's operation order, shows
    1.2e-5 (2 dm) and 1.9e-5 (dm1 + dm2) on this set-up, so the bound is 5e-5 for both."""
    model, solver = _small()
    dm1, dm2 = _blob(model), _blob(model, scale=-0.03, shift=3.0)
    j1, j2 = _jac(solver, dm1), _jac(solver, dm2)
    assert np.abs(j1['du']).max() > 1e-3 * np.abs(j1['u0']).max()
    j11 = _jac(solver, (2 * dm1).astype(np.float32))
    j12 = _jac(solver, (dm1 + dm2).astype(np.float32))
    for n in ('du', 'dv', 'rec'):
        assert rel_linf(j11[n], 2 * j1[n].astype(np.float64)) < 5e-5, n
        assert rel_linf(j12[n], j1[n].astype(np.float64) + j2[n]) < 5e-5, n


@pytest.mark.gpu
def test_restart_and_host_staging():
    """[time_m, k] then [k+1, time_M] equals one call bit for bit; resident=False equals resident bit for bit."""
    from devito_b200 import TimeFunction
    model, solver = _small()
    dm = _blob(model)
    one = _jac(solver, dm)
    nt = solver.geometry.nt
    mk = lambda n: TimeFunction(name=n, grid=model.grid, time_order=2, space_order=solver.space_order)
    u0, v0, du, dv = mk('u0'), mk('v0'), mk('du'), mk('dv')
    rec = solver.geometry.rec
    rec.data[:] = 0.0
    k = nt // 2
    solver.jacobian(dm, u0=u0, v0=v0, du=du, dv=dv, rec=rec, time_m=1, time_M=k)
    solver.jacobian(dm, u0=u0, v0=v0, du=du, dv=dv, rec=rec, time_m=k + 1, time_M=nt - 2)
    for f, n in ((u0, 'u0'), (v0, 'v0'), (du, 'du'), (dv, 'dv'), (rec, 'rec')):
        assert np.array_equal(np.asarray(f.data), one[n]), n
    staged = _jac(solver, dm, resident=False)
    for n in one:
        assert np.array_equal(staged[n], one[n]), n


@pytest.mark.gpu
def test_taylor():
    """The reference's Taylor test (tests/test_gradient.py::test_gradientJ, TTI case) in 3-D: with m0 a smoothed
    layered vp and dm = m - m0, |F(m0 + h dm) - F(m0)|_1 has slope 1 and |F(m0 + h dm) - F(m0) - h J dm|_1 slope 2
    in h."""
    from devito_b200 import Function
    from devito_b200.builtins import smooth
    from devito_b200.seismic import demo_model, setup_geometry
    from devito_b200.seismic.tti import AnisotropicWaveSolver
    so = 4
    model = demo_model('layers-tti', shape=(40, 40, 40), spacing=(15., 15., 15.), nbl=12, space_order=so, nlayers=3)
    geometry = setup_geometry(model, 600.0)
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
