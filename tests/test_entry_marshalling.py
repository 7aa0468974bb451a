"""What each wave operator hands its C entry point, whichever way it is called.

`Operator.apply` (the Python host layer) and the adapter `Operator.cinterface()` writes both fill the argument
block of b2_iso_forward / b2_tti_forward / b2_sa_forward. Both run here without a GPU against the recording test
double tests/support/stub_backend.c, from the same inputs, and the two blocks are compared member by member and
by value (the Python layer frees its structs when `apply` returns). The override rules of `apply` are pinned too.
"""
import ctypes
import shutil
import types

import numpy as np
import pytest

from devito_b200 import _lib as L_
from devito_b200 import Constant, Function
from devito_b200.exceptions import InvalidArgument

import test_zz_cinterface as CI
import test_zz_born
import test_zz_freesurface
import test_zz_ot4
import test_zz_snapshots
import test_zz_tti_adjoint

pytestmark = pytest.mark.skipif(shutil.which('gcc') is None, reason="gcc not available")

STRUCTS = {'iso': L_.IsoArgs, 'tti': L_.TtiArgs, 'sa': L_.SaArgs}
SMALL = {'n': 12, 'nbl': 4, 'tn': 20.0, 'factor': 3}


# ---------------------------------------------------------------------------------------------------------------
# the operators
# ---------------------------------------------------------------------------------------------------------------
def _iso(case):
    if case == 'ot4':
        return test_zz_ot4._solver(SMALL, 'layers-isotropic', 4)[2].op_fwd()
    if case == 'free_surface':
        return test_zz_freesurface._solver(so=4, n=12, nbl=4, tn=20.0)[2].op_fwd()
    if case == 'snapshots':
        return test_zz_snapshots._operator(SMALL)[0]
    if case == 'born':
        return test_zz_born._solver(SMALL, so=4)[2].op_born()
    preset = 'constant-isotropic' if case == 'fwd_const' else 'layers-isotropic'
    solver = CI._iso_solver(so=4, n=12, nbl=4, preset=preset)
    return {'fwd_const': solver.op_fwd, 'fwd_layers': solver.op_fwd, 'adjoint': solver.op_adj,
            'gradient': solver.op_grad}[case]()


def _tti(case):
    preset = 'constant-tti' if case == 'fwd_const' else 'layers-tti'
    kw = {} if preset == 'constant-tti' else {'nlayers': 2}
    solver = test_zz_tti_adjoint._solver(preset, 4, kw, n=12, nbl=4, tn=20.0)[2]
    return {'fwd_const': solver.op_fwd, 'fwd_func': solver.op_fwd, 'adjoint': solver.op_adj,
            'born': solver.op_jac, 'gradient': solver.op_jacadj}[case]()


def _sa(case):
    from devito_b200.seismic import acoustic_sa_setup
    nd, which = int(case[0]), case[3:]
    solver = acoustic_sa_setup(shape=(13, 14, 15)[:nd], nbl=4, tn=20.0)
    return solver.op_fwd() if which == 'fwd' else solver.op_adj()


CASES = ([('iso', c) for c in ('fwd_const', 'fwd_layers', 'adjoint', 'ot4', 'free_surface', 'snapshots', 'born',
                               'gradient')] +
         [('tti', c) for c in ('fwd_const', 'fwd_func', 'adjoint', 'born', 'gradient')] +
         [('sa', c) for c in ('2d_fwd', '2d_adj', '3d_fwd', '3d_adj')])


def _operator(kind, case):
    op = {'iso': _iso, 'tti': _tti, 'sa': _sa}[kind](case)
    assert op.backend == 'cuda-sm90a' and op._plan['kind'] == kind, op._why_not
    return op


# ---------------------------------------------------------------------------------------------------------------
# the recording double, reached from the Python layer and from the generated adapter
# ---------------------------------------------------------------------------------------------------------------
def _stub_and_adapter(op, tmp_path, monkeypatch):
    """The recording double and the adapter linked against it; `_lib.lib()` returns the double too."""
    monkeypatch.setenv('DEVITO_B200_JITDIR', str(tmp_path))
    op.cinterface(force=True)
    stub, lib = CI._build_against_stub(str(tmp_path), op.name)
    fake = types.SimpleNamespace(b2_last_error=lambda: b'stub')
    for kind, st in STRUCTS.items():
        fn = getattr(stub, f'double_b2_{kind}_forward')
        fn.argtypes, fn.restype = [ctypes.POINTER(st)], ctypes.c_int
        setattr(fake, f'b2_{kind}_forward', fn)
        getattr(stub, f'stub_{kind}_deep').restype = ctypes.POINTER(st)
    monkeypatch.setattr(L_, 'lib', lambda: fake)
    return stub, getattr(lib, op.name)


def _obj_value(p):
    """A recorded dataobj by value: extents, halo, contents, whether a device copy came along."""
    if not p:
        return None
    o = p.contents
    rank = next(i for i in range(8) if o.size[i] == 0)
    return {'size': tuple(o.size[i] for i in range(rank)),
            'hsize': tuple(o.hsize[i] for i in range(2 * rank)) if o.hsize else None,
            'data': ctypes.string_at(o.data, o.nbytes) if o.data else None, 'nbytes': o.nbytes,
            'dmap': bool(o.dmap)}


def _sparse_value(p):
    if not p:
        return None
    s = p.contents
    return {'data': _obj_value(s.data), 'gp': _obj_value(s.gp), 'w': [_obj_value(s.w[d]) for d in range(3)],
            'p_m': s.p_m, 'p_M': s.p_M, 'r': s.r}


def _recorded(stub, kind):
    """The last block the double received, every member by value (the timers excepted)."""
    a = getattr(stub, f'stub_{kind}_deep')().contents
    nw = a.ndim if kind != 'tti' else 3
    count = {'w': a.radius + 1, 'w2': a.radius + 1, 'w1': a.radius, 'c': a.radius}
    out = {}
    for name, ctype in STRUCTS[kind]._fields_:
        v = getattr(a, name)
        if name == 'timers':
            continue
        if name in count:
            out[name] = [tuple(v[d][i] for i in range(count[name])) for d in range(nw)]
        elif ctype is ctypes.POINTER(L_.Dataobj):
            out[name] = _obj_value(v)
        elif ctype is ctypes.POINTER(L_.Sparse):
            out[name] = _sparse_value(v)
        else:
            out[name] = v
    return out


def _plan_objects(plan):
    """Every Function, Constant and sparse function the recogniser put in the plan, by name."""
    out = {}

    def walk(v):
        if isinstance(v, dict):
            for x in v.values():
                walk(x)
        elif isinstance(v, (tuple, list)):
            for x in v:
                walk(x)
        elif isinstance(v, (Function, Constant)) or getattr(v, 'is_SparseTimeFunction', False):
            out[v.name] = v
    walk(plan)
    return out


def _fill(op, seed=7):
    """Seeded values in every dense array the operator takes, so that contents are compared, not zeros."""
    rng = np.random.default_rng(seed)
    for f in _plan_objects(op._plan).values():
        if isinstance(f, Function):
            f.data_with_halo[:] = rng.uniform(0.5, 1.5, size=f.data_with_halo.shape).astype(np.float32)


def _adapter_values(op, args, dt):
    """The flat arguments of the adapter: copies of the same arrays, the same scalars."""
    p = op._plan
    vals, keep = {'dt': dt, 'time_m': args['time_m'], 'time_M': args['time_M'], 'deviceid': 0, 'devicerm': 1}, []
    for d, lo, hi in zip(p['grid'].dimensions, args['lo'], args['hi']):
        vals[d.min_name], vals[d.max_name] = lo, hi
    for f in _plan_objects(p).values():
        if getattr(f, 'is_SparseTimeFunction', False):
            CI._sparse_values(f, f.name, vals, keep)
            vals[f'p_{f.name}_M'] = f.npoint - 1
        elif isinstance(f, Function):
            vals[f.name] = CI._dobj(np.array(f.data_with_halo), f.halo)
        else:
            vals[f.name] = float(f.data)
    return vals, keep


def _both(op, stub, adapter, dt):
    """(block built by Operator.apply, block built by the adapter) from the same inputs."""
    kind = op._plan['kind']
    _fill(op)
    args = op.arguments(dt=dt)
    vals, keep = _adapter_values(op, args, dt)
    summary = op.apply(dt=dt, resident=False)
    assert summary.time > 0
    py = _recorded(stub, kind)
    adapter.restype = ctypes.c_int
    assert adapter(*CI._flat_args(op, vals, CI._CProfiler())) == 0
    return py, _recorded(stub, kind)


def _compare(py, ad):
    assert set(py) == set(ad)
    for k in py:
        if isinstance(py[k], float):
            assert np.float32(py[k]) == np.float32(ad[k]), k
        else:
            assert py[k] == ad[k], k


ARRAYS = {'iso': ('u', 'damp', 'param', 'grad', 'usave', 'born_U', 'born_dm', 'snap'),
          'tti': ('u', 'v', 'damp', 'vp_arr', 'epsilon_arr', 'delta_arr', 'theta_arr', 'phi_arr', 'born_du',
                  'born_dv', 'born_dm', 'grad', 'usave', 'vsave'),
          'sa': ('u', 'b', 'vp', 'damp')}

EXPECT = {
    ('iso', 'fwd_const'): dict(param_kind=0, adjoint=0, ot4=0, free_surface=0, set={'u', 'damp'}),
    ('iso', 'fwd_layers'): dict(param_kind=1, vp=1.0, adjoint=0, set={'u', 'damp', 'param'}),
    ('iso', 'adjoint'): dict(param_kind=1, adjoint=1, set={'u', 'damp', 'param'}),
    ('iso', 'ot4'): dict(param_kind=1, ot4=1, adjoint=0, set={'u', 'damp', 'param'}),
    ('iso', 'free_surface'): dict(param_kind=1, free_surface=1, set={'u', 'damp', 'param'}),
    ('iso', 'snapshots'): dict(param_kind=0, snap_factor=3, snap_toff=0, set={'u', 'damp', 'snap'}),
    ('iso', 'born'): dict(param_kind=1, set={'u', 'damp', 'param', 'born_U', 'born_dm'}),
    ('iso', 'gradient'): dict(param_kind=1, adjoint=1, set={'u', 'damp', 'param', 'grad', 'usave'}),
    ('tti', 'fwd_const'): dict(adjoint=0, set={'u', 'v', 'damp'}),
    ('tti', 'fwd_func'): dict(adjoint=0, vp=1.0, set={'u', 'v', 'damp', 'vp_arr', 'epsilon_arr', 'delta_arr',
                                                       'theta_arr', 'phi_arr'}),
    ('tti', 'adjoint'): dict(adjoint=1, set={'u', 'v', 'damp', 'vp_arr', 'epsilon_arr', 'delta_arr', 'theta_arr',
                                              'phi_arr'}),
    ('tti', 'born'): dict(adjoint=0, set={'u', 'v', 'damp', 'vp_arr', 'epsilon_arr', 'delta_arr', 'theta_arr',
                                           'phi_arr', 'born_du', 'born_dv', 'born_dm'}),
    ('tti', 'gradient'): dict(adjoint=1, set={'u', 'v', 'damp', 'vp_arr', 'epsilon_arr', 'delta_arr', 'theta_arr',
                                               'phi_arr', 'grad', 'usave', 'vsave'}),
    ('sa', '2d_fwd'): dict(ndim=2, adjoint=0, set={'u', 'b', 'vp', 'damp'}),
    ('sa', '2d_adj'): dict(ndim=2, adjoint=1, set={'u', 'b', 'vp', 'damp'}),
    ('sa', '3d_fwd'): dict(ndim=3, adjoint=0, set={'u', 'b', 'vp', 'damp'}),
    ('sa', '3d_adj'): dict(ndim=3, adjoint=1, set={'u', 'b', 'vp', 'damp'}),
}


@pytest.mark.parametrize('kind,case', CASES, ids=[f'{k}-{c}' for k, c in CASES])
def test_apply_and_adapter_build_the_same_block(kind, case, tmp_path, monkeypatch):
    op = _operator(kind, case)
    stub, adapter = _stub_and_adapter(op, tmp_path, monkeypatch)
    p = op._plan
    # an injection written with a literal dt**2 (the snapshot operator) takes that dt
    dt = float(np.float32(np.sqrt(p['inject_dt2']) if p.get('inject_literal') else 0.5))
    py, ad = _both(op, stub, adapter, dt)
    _compare(py, ad)
    want = dict(EXPECT[(kind, case)])
    assert {k for k in ARRAYS[kind] if py[k] is not None} == want.pop('set')
    for k, v in want.items():
        assert py[k] == v, k
    assert py['dt'] == np.float32(dt) and py['rec_toff'] == p['rec_toff']
    assert (py['src'] is None) == (p['src'] is None) and (py['rec'] is None) == (p['rec'] is None)
    assert not any(py[k]['dmap'] for k in ARRAYS[kind] if py[k] is not None)
    assert py['u']['size'] == p['u'].data_with_halo.shape


# ---------------------------------------------------------------------------------------------------------------
# the override rules of `apply`, per kind
# ---------------------------------------------------------------------------------------------------------------
def test_ndarray_wavefield_is_used_and_written_back(tmp_path, monkeypatch):
    op = _operator('iso', 'fwd_const')
    stub, _ = _stub_and_adapter(op, tmp_path, monkeypatch)
    u = op._plan['u']
    arr = np.random.default_rng(3).uniform(size=u.shape_allocated).astype(np.float32)
    before = arr.tobytes()
    op.apply(dt=0.5, resident=False, u=arr)
    assert _recorded(stub, 'iso')['u']['data'] == before
    assert arr.ravel()[0] == stub.stub_calls()
    assert arr.tobytes()[4:] == before[4:]


def test_iso_function_for_a_constant_velocity_switches_to_an_array(tmp_path, monkeypatch):
    op = _operator('iso', 'fwd_const')
    stub, _ = _stub_and_adapter(op, tmp_path, monkeypatch)
    p = op._plan
    assert p['m_role'][0] == 'vp_c'
    vp = Function(name='vp', grid=p['grid'], space_order=p['so'])
    vp.data_with_halo[:] = 1.25
    op.apply(dt=0.5, resident=False, vp=vp)
    a = _recorded(stub, 'iso')
    assert a['param_kind'] == 1 and a['vp'] == 1.0
    assert a['param']['data'] == np.full(vp.data_with_halo.shape, 1.25, np.float32).tobytes()
    op.apply(dt=0.5, resident=False, vp=2.0)
    a = _recorded(stub, 'iso')
    assert a['param_kind'] == 0 and a['param'] is None and a['vp'] == 2.0


def test_sa_number_for_a_function_buoyancy_is_a_value(tmp_path, monkeypatch):
    op = _operator('sa', '3d_fwd')
    stub, _ = _stub_and_adapter(op, tmp_path, monkeypatch)
    assert op._plan['b_role'][0] == 'f'
    op.apply(dt=0.5, resident=False, b=0.75)
    a = _recorded(stub, 'sa')
    assert a['b'] is None and a['b_value'] == 0.75 and a['vp'] is not None and a['vp_value'] == 1.0


def test_tti_parameters_keep_the_kind_they_were_built_with(tmp_path, monkeypatch):
    for case, value in (('fwd_const', 'function'), ('fwd_func', 0.3)):
        op = _operator('tti', case)
        (tmp_path / case).mkdir()
        stub, _ = _stub_and_adapter(op, tmp_path / case, monkeypatch)
        p = op._plan
        if value == 'function':
            value = Function(name='theta', grid=p['grid'], space_order=p['so'])
        with pytest.raises(InvalidArgument):
            op.apply(dt=0.5, resident=False, theta=value)
    assert stub.stub_calls() == 0


# ---------------------------------------------------------------------------------------------------------------
# every consumer reads the same objects (the reference plugin overrides `parameters` by name)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind,case', CASES, ids=[f'{k}-{c}' for k, c in CASES])
def test_parameters_are_what_the_adapter_takes(kind, case):
    from devito_b200 import cinterface as ci
    op = _operator(kind, case)
    p = op._plan
    names = {f.name for f in op.parameters}
    sparse = {f'{sf.name}_{x}' for sf in (p['src'], p['rec']) if sf is not None for x in ('gp', 'wx', 'wy', 'wz')}
    head = {q.key for q in ci.signature(p, op.name) if q.ctype.startswith('struct dataobj') or q.key != 'dt'
            and q.ctype == 'const float'} - sparse
    assert names == head
    assert names == set(_plan_objects(p))
    if (kind, case) == ('tti', 'gradient'):
        assert {'usave', 'vsave', 'grad'} <= {s.member for s in op._entry.arrays}
        assert {'u0', 'v0'} <= names
    if (kind, case) == ('tti', 'born'):
        assert {'born_du', 'born_dv', 'born_dm'} <= {s.member for s in op._entry.arrays}
        assert {'du', 'dv', 'dm'} <= names
