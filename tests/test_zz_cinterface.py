"""`Operator.cinterface()`: the reference-style C symbol on top of libb200stencil.so.

Mirrors tests/test_cinterface.py:9-41 of the reference (files written, public structs only in the
header), then checks the adapter itself: compiled with gcc against a recording test double
(tests/support/stub_backend.c) it must hand `b2_iso_forward` / `b2_tti_forward` exactly the argument
block the Python host layer would build. The GPU test calls the adapter linked against the real
library with host arrays and compares with `Operator.apply`.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from devito_b200 import _lib as L_
from devito_b200.seismic import (AcousticWaveSolver, AnisotropicWaveSolver, demo_model,
                                 setup_geometry)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, 'include')
STUB_SRC = os.path.join(ROOT, 'tests', 'support', 'stub_backend.c')

needs_gcc = pytest.mark.skipif(shutil.which('gcc') is None, reason="gcc not available")


@pytest.fixture()
def jitdir(tmp_path, monkeypatch):
    monkeypatch.setenv('DEVITO_B200_JITDIR', str(tmp_path))
    return str(tmp_path)


def _iso_solver(so=8, n=16, nbl=6, preset='constant-isotropic'):
    model = demo_model(preset, shape=(n,) * 3, spacing=(10.,) * 3, nbl=nbl, space_order=so)
    geo = setup_geometry(model, tn=40.)
    return AcousticWaveSolver(model, geo, space_order=so)


def _tti_solver(so=8, n=16, nbl=6, preset='constant-tti'):
    model = demo_model(preset, shape=(n,) * 3, spacing=(10.,) * 3, nbl=nbl, space_order=so)
    geo = setup_geometry(model, tn=40.)
    return AnisotropicWaveSolver(model, geo, space_order=so)


def test_files_and_public_structs(jitdir):
    op = _iso_solver().op_fwd()
    ccode, hcode = op.cinterface(force=True)
    assert os.path.isfile(os.path.join(jitdir, 'Forward.c'))
    assert os.path.isfile(os.path.join(jitdir, 'Forward.h'))
    assert 'include "Forward.h"' in ccode
    # the public structs only appear in the header (reference tests/test_cinterface.py:31-39)
    assert 'struct dataobj\n{' in hcode and 'struct dataobj\n{' not in ccode
    assert 'struct profiler\n{' in hcode and 'struct profiler\n{' not in ccode
    # reference parameter order: Functions/Constants by name, bounds, dt, point ranges, time, timers
    proto = [ln for ln in hcode.splitlines() if ln.startswith('int Forward(')][0]
    order = ['damp_vec', 'rec_vec', 'rec_gp_vec', 'rec_wx_vec', 'src_vec', 'src_wz_vec', 'u_vec',
             'const float vp', 'x_M', 'x_m', 'z_m', 'const float dt', 'p_rec_M', 'p_src_m', 'time_M',
             'time_m', 'deviceid', 'struct profiler *timers']
    pos = [proto.index(tok) for tok in order]
    assert pos == sorted(pos)
    # not overwritten without force
    path = os.path.join(jitdir, 'Forward.h')
    with open(path, 'w') as f:
        f.write('/* kept */')
    op.cinterface()
    assert open(path).read() == '/* kept */'


def _cc(args, cwd):
    r = subprocess.run(['gcc'] + args, cwd=cwd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r


def _build_against_stub(jitdir, name):
    # one uniquely named double per test: the dynamic loader shares libraries by soname
    tag = f'stub_{name}_{os.path.basename(jitdir)}'.replace('-', '_')
    # the entry points are renamed on both sides so that the real library, when another test has
    # already loaded it with RTLD_GLOBAL, cannot interpose them
    ren = ['-Db2_iso_forward=double_b2_iso_forward', '-Db2_tti_forward=double_b2_tti_forward',
           '-Db2_sa_forward=double_b2_sa_forward']
    _cc(['-O1', '-shared', '-fPIC', '-Wall', '-Werror', '-I', INCLUDE] + ren + [STUB_SRC, '-o', f'lib{tag}.so'],
        jitdir)
    _cc(['-O1', '-shared', '-fPIC', '-Wall', '-Werror', '-I', INCLUDE, '-I', jitdir] + ren + [f'{name}.c',
         '-L', jitdir, f'-l{tag}', f'-Wl,-rpath,{jitdir}', '-lm', '-o', f'lib{name}_{tag}.so'], jitdir)
    stub = ctypes.CDLL(os.path.join(jitdir, f'lib{tag}.so'))
    lib = ctypes.CDLL(os.path.join(jitdir, f'lib{name}_{tag}.so'))
    return stub, lib


class _CProfiler(ctypes.Structure):
    _fields_ = [('section0', ctypes.c_double), ('section1', ctypes.c_double),
                ('section2', ctypes.c_double)]


def _dobj(arr, halo=None):
    return L_.make_dataobj(host=np.ascontiguousarray(arr), halo=halo)


def _flat_args(op, values, timers):
    """Positional ctypes arguments in the order of the generated prototype."""
    from devito_b200 import cinterface as ci
    out = []
    for p in ci.signature(op._plan, op.name):
        v = values[p.key] if p.key != 'timers' else timers
        if p.ctype.startswith('struct dataobj'):
            out.append(v.ptr)
        elif p.ctype == 'const float':
            out.append(ctypes.c_float(v))
        elif p.ctype == 'const int':
            out.append(ctypes.c_int(v))
        else:
            out.append(ctypes.byref(v))
    return out


def _sparse_values(sf, prefix, vals, keep):
    gp, ws = sf.tabulate()
    objs = [_dobj(sf.data), _dobj(gp)] + [_dobj(w) for w in ws]
    keep.extend(objs)
    vals[prefix] = objs[0]
    vals[prefix + '_gp'] = objs[1]
    for d, o in enumerate(objs[2:]):
        vals[f'{prefix}_w{"xyz"[d]}'] = o
    vals[f'p_{prefix}_m'] = 0
    vals[f'p_{prefix}_M'] = sf.npoint - 1


@needs_gcc
def test_iso_adapter_marshalling(jitdir):
    solver = _iso_solver(so=8)
    op = solver.op_fwd()
    op.cinterface(force=True)
    stub, lib = _build_against_stub(jitdir, 'Forward')
    p = op._plan
    u, damp, src, rec = p['u'], p['damp'], p['src'], p['rec']
    keep = []
    vals = {'u': _dobj(u.data_with_halo, u.halo), 'damp': _dobj(damp.data_with_halo, damp.halo),
            'vp': 1.5, 'dt': 1.25, 'time_m': 1, 'time_M': 7, 'deviceid': 3, 'devicerm': 1}
    for d, n in zip(p['grid'].dimensions, p['grid'].shape):
        vals[d.min_name], vals[d.max_name] = 2, n - 3
    _sparse_values(src, 'src', vals, keep)
    _sparse_values(rec, 'rec', vals, keep)
    timers = _CProfiler(1.0, 0.0, 0.0)
    lib.Forward.restype = ctypes.c_int
    stub.stub_set_rc(0)
    assert lib.Forward(*_flat_args(op, vals, timers)) == 0
    stub.stub_iso_seen.restype = ctypes.POINTER(L_.IsoArgs)
    a = stub.stub_iso_seen().contents
    assert (a.ndim, a.space_order, a.radius) == (3, 8, 4)
    for d in range(3):
        np.testing.assert_array_equal(np.ctypeslib.as_array(a.w[d], (5,)),
                                      np.asarray(p['w'][d], dtype=np.float32))
    assert ctypes.addressof(a.u.contents) == ctypes.addressof(vals['u'].obj)
    assert ctypes.addressof(a.damp.contents) == ctypes.addressof(vals['damp'].obj)
    assert a.u.contents.data == vals['u'].host.ctypes.data
    assert a.param_kind == 0 and not a.param
    assert a.vp == np.float32(1.5) and a.dt == np.float32(1.25)
    n = p['grid'].shape
    assert (a.x_m, a.x_M, a.y_m, a.y_M, a.z_m, a.z_M) == (2, n[0] - 3, 2, n[1] - 3, 2, n[2] - 3)
    assert (a.time_m, a.time_M) == (1, 7)
    assert (a.rec_toff, a.deviceid, a.adjoint) == (0, 3, 0)
    assert not a.halo and not a.grad and not a.usave
    s, r = a.src.contents, a.rec.contents
    assert (s.p_m, s.p_M, s.r) == (0, src.npoint - 1, 1)
    assert (r.p_m, r.p_M, r.r) == (0, rec.npoint - 1, 1)
    assert ctypes.addressof(s.data.contents) == ctypes.addressof(vals['src'].obj)
    assert ctypes.addressof(r.gp.contents) == ctypes.addressof(vals['rec_gp'].obj)
    assert ctypes.addressof(r.w[2].contents) == ctypes.addressof(vals['rec_wz'].obj)
    # section timers are accumulated into the caller's struct; the return code is passed through
    assert (timers.section0, timers.section1, timers.section2) == (2.5, 0.25, 0.125)
    stub.stub_set_rc(100)
    assert lib.Forward(*_flat_args(op, vals, timers)) == 100


@needs_gcc
def test_iso_adapter_array_velocity_and_adjoint(jitdir):
    solver = _iso_solver(so=4, preset='layers-isotropic')
    for op, adjoint in ((solver.op_fwd(), 0), (solver.op_adj(), 1)):
        ccode, hcode = op.cinterface(force=True)
        assert f'a.adjoint = {adjoint};' in ccode
        assert 'a.param_kind = B2_PARAM_VP;' in ccode and 'vp_vec' in hcode
        _cc(['-c', '-Wall', '-Werror', '-I', INCLUDE, '-I', jitdir, f'{op.name}.c', '-o', f'{op.name}.o'],
            jitdir)


@needs_gcc
def test_tti_adapter_marshalling(jitdir):
    solver = _tti_solver(so=8)
    op = solver.op_fwd()
    op.cinterface(force=True)
    stub, lib = _build_against_stub(jitdir, op.name)
    p = op._plan
    keep = []
    vals = {'u': _dobj(p['u'].data_with_halo, p['u'].halo), 'v': _dobj(p['v'].data_with_halo, p['v'].halo),
            'damp': _dobj(p['damp'].data_with_halo, p['damp'].halo),
            'vp': 1.5, 'epsilon': 0.3, 'delta': 0.2, 'theta': 0.7, 'phi': 0.35,
            'dt': 0.75, 'time_m': 1, 'time_M': 4, 'deviceid': 0, 'devicerm': 0}
    for d, n in zip(p['grid'].dimensions, p['grid'].shape):
        vals[d.min_name], vals[d.max_name] = 0, n - 1
    _sparse_values(p['src'], 'src', vals, keep)
    _sparse_values(p['rec'], 'rec', vals, keep)
    timers = _CProfiler()
    fn = getattr(lib, op.name)
    fn.restype = ctypes.c_int
    stub.stub_set_rc(0)
    assert fn(*_flat_args(op, vals, timers)) == 0
    stub.stub_tti_seen.restype = ctypes.POINTER(L_.TtiArgs)
    a = stub.stub_tti_seen().contents
    assert (a.space_order, a.radius) == (8, 4)
    for d in range(3):
        np.testing.assert_array_equal(np.ctypeslib.as_array(a.w2[d], (5,)),
                                      np.asarray(p['w2'][d], dtype=np.float32))
        np.testing.assert_array_equal(np.ctypeslib.as_array(a.w1[d], (4,)),
                                      np.asarray(p['w1'][d], dtype=np.float32))
    got = (a.vp, a.epsilon, a.delta, a.theta, a.phi, a.dt)
    assert got == tuple(float(np.float32(x)) for x in (1.5, 0.3, 0.2, 0.7, 0.35, 0.75))
    assert ctypes.addressof(a.v.contents) == ctypes.addressof(vals['v'].obj)
    assert not a.vp_arr and not a.theta_arr
    n = p['grid'].shape
    assert (a.x_M, a.y_M, a.z_M, a.time_M) == (n[0] - 1, n[1] - 1, n[2] - 1, 4)
    assert a.src.contents.p_M == 0 and a.rec.contents.p_M == p['rec'].npoint - 1


@needs_gcc
def test_adapter_links_against_the_library(jitdir):
    """The adapter resolves its one external symbol from libb200stencil.so and exports `Forward`."""
    op = _iso_solver().op_fwd()
    op.cinterface(force=True)
    libdir = os.path.dirname(L_.LIB_PATH)
    _cc(['-shared', '-fPIC', '-I', INCLUDE, '-I', jitdir, 'Forward.c', '-L', libdir, '-lb200stencil',
         f'-Wl,-rpath,{libdir}', '-lm', '-o', 'libForward.so'], jitdir)
    out = subprocess.run(['nm', '-D', os.path.join(jitdir, 'libForward.so')], capture_output=True, text=True).stdout
    assert ' T Forward' in out and ' U b2_iso_forward' in out


@pytest.mark.gpu
@needs_gcc
def test_adapter_runs_on_the_gpu(jitdir):
    """`Forward(...)` called like the reference calls its generated function (host arrays, flat
    argument list) == `Operator.apply` on the same inputs."""
    solver = _iso_solver(so=8, n=32, nbl=8)
    op = solver.op_fwd()
    p = op._plan
    u, damp, src, rec = p['u'], p['damp'], p['src'], p['rec']
    dt = solver.model.critical_dt
    # reference result through the Python host layer (host-staged, like the adapter call below)
    u.data_with_halo[:] = 0.
    rec.data[:] = 0.
    op.apply(dt=dt, resident=False)
    u_ref = np.array(u.data_with_halo)
    rec_ref = np.array(rec.data)
    assert np.abs(rec_ref).max() > 0
    # the same through the generated C symbol
    op.cinterface(force=True)
    libdir = os.path.dirname(L_.LIB_PATH)
    _cc(['-shared', '-fPIC', '-I', INCLUDE, '-I', jitdir, 'Forward.c', '-L', libdir, '-lb200stencil',
         f'-Wl,-rpath,{libdir}', '-lm', '-o', 'libForward.so'], jitdir)
    L_.lib()
    lib = ctypes.CDLL(os.path.join(jitdir, 'libForward.so'))
    uh = np.zeros_like(u_ref)
    rech = np.zeros_like(rec_ref)
    keep = []
    vals = {'u': _dobj(uh, u.halo), 'damp': _dobj(damp.data_with_halo, damp.halo),
            'vp': float(solver.model.vp.data if hasattr(solver.model.vp, 'data') else solver.model.vp),
            'dt': float(dt), 'time_m': 1, 'time_M': src.nt - 2, 'deviceid': 0, 'devicerm': 1}
    for d, n in zip(p['grid'].dimensions, p['grid'].shape):
        vals[d.min_name], vals[d.max_name] = 0, n - 1
    _sparse_values(src, 'src', vals, keep)
    _sparse_values(rec, 'rec', vals, keep)
    vals['rec'] = _dobj(rech)
    timers = _CProfiler()
    lib.Forward.restype = ctypes.c_int
    rc = lib.Forward(*_flat_args(op, vals, timers))
    assert rc == 0
    np.testing.assert_array_equal(vals['u'].host, u_ref)
    np.testing.assert_array_equal(vals['rec'].host, rec_ref)
    assert timers.section0 > 0


def test_ndarray_override_is_checked():
    """`op.apply(u=<ndarray>)`: a bare array stands in for the allocated data (reference
    devito/types/dense.py:913-926); shape/dtype are validated before anything runs."""
    from devito_b200.exceptions import InvalidArgument
    solver = _iso_solver(so=4)
    op = solver.op_fwd()
    u = op._plan['u']
    good = np.zeros(u.shape_allocated, dtype=np.float32)
    args = op.arguments(u=good, dt=1.0)
    assert args['fields'][0].storage.host is good and args['fields'][0] is not u
    with pytest.raises(InvalidArgument):
        op.arguments(u=np.zeros(u.shape, dtype=np.float32), dt=1.0)          # domain-only shape
    with pytest.raises(InvalidArgument):
        op.arguments(u=good.astype(np.float64), dt=1.0)


@pytest.mark.gpu
def test_ndarray_override_runs_in_place():
    solver = _iso_solver(so=8, n=32, nbl=8)
    op = solver.op_fwd()
    p = op._plan
    u, rec = p['u'], p['rec']
    dt = solver.model.critical_dt
    op.apply(dt=dt)
    u_ref, rec_ref = np.array(u.data_with_halo), np.array(rec.data)
    ua = np.zeros(u.shape_allocated, dtype=np.float32)
    ra = np.zeros(rec.data.shape, dtype=np.float32)
    op.apply(dt=dt, u=ua, rec=ra)
    np.testing.assert_array_equal(ua, u_ref)
    np.testing.assert_array_equal(ra, rec_ref)
