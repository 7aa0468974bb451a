"""`b2_system_forward` (`devito_b200.system.LinearSystem.apply`) against the float64 tap-table interpreter
(tests/system_ref.py), on the GPU.

* The fixture systems of oracle/make_golden_system.py (the reference's elastic and viscoelastic runs, with the tables
  refplugin built): host-staged coefficient arrays, and device-resident ones through `make_dataobj(dev_ptr=...)` as
  the plugin passes them. Compared with the interpreter (TOL) and with the reference's stored outputs (TOL_REF).
* The synthetic systems of tests/system_cases.py, in three modes: host-staged, device-resident coefficients, and the
  taps shuffled after `Stage` sorted them by coefficient array (every tap reloads the cached coefficient).
* Malformed calls: each returns B2_ERR_INVALID (210) and leaves the fields and traces untouched.
* Every call, run or refused, releases every staging buffer it took (`b2_staging_outstanding`).

The reference package is never read here.
"""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest

from helpers import load_golden, rel_linf
import system_cases as SC
import system_ref as SR

pytestmark = pytest.mark.gpu

TOL = 1e-5
TOL_REF = 2e-5
B2_ERR_INVALID = 210
_interp = {}


def _sparse_obj(sp, keep):
    from devito_b200 import _lib as L_
    data = np.array(sp['data'], dtype=np.float32)
    ns = SimpleNamespace(data=L_.make_dataobj(host=data), gp=L_.make_dataobj(host=np.ascontiguousarray(sp['gp'],
                                                                                                    dtype=np.int32)),
                         ws=[L_.make_dataobj(host=np.ascontiguousarray(w, dtype=np.float32)) for w in sp['w']],
                         p_m=int(sp['p_m']), p_M=int(sp['p_M']), r=int(sp['r']))
    keep[id(sp)] = (ns, data)
    return ns


def _build(system, fields, coefs, mode, seed=0):
    """(LinearSystem, field holders, host field arrays, coefficient objects, traces by sparse id, keep-alive)."""
    from devito_b200 import _lib as L_
    from devito_b200.system import LinearSystem, Stage, Tap
    rng = np.random.default_rng(seed)
    F = [np.array(f, dtype=np.float32) for f in fields]
    fobjs = [L_.make_dataobj(host=f) for f in F]
    stages = []
    for out, ots, taps, *ext in system['stages']:
        st = Stage(out, ots, [Tap(*t) for t in taps], ext[0] if ext else 0)
        if mode == 'shuffled':
            st.taps = [st.taps[i] for i in rng.permutation(len(st.taps))]
        stages.append(st)
    sps = {}

    def sp(q):
        return sps[id(q['sp'])][0] if id(q['sp']) in sps else _sparse_obj(q['sp'], sps)
    keep = []
    inj = []
    for q in system['injections']:
        pobj = None
        if q['param'] is not None:
            pobj = L_.make_dataobj(host=np.ascontiguousarray(q['param'], dtype=np.float32))
            keep.append(pobj)
        inj.append((sp(q), q['fields'], q['tshift'], q['scale'], q['kind'], pobj))
    itp = [(sp(q), q['field'], q['tshift']) for q in system['interpolations']]
    cobjs = [np.ascontiguousarray(c, dtype=np.float32) for c in coefs]
    if mode == 'device':
        import torch
        ts = [torch.from_numpy(c).cuda() for c in cobjs]
        torch.cuda.synchronize()
        cobjs = [L_.make_dataobj(dev_ptr=t.data_ptr(), shape=t.shape) for t in ts]
        keep.append(ts)
    ls = LinearSystem(system['nd'], system['halo'], len(F), stages, inj, itp)
    return ls, fobjs, F, cobjs, {k: d for k, (_, d) in sps.items()}, keep


def _execute(system, fields, coefs, lo, hi, tm, tM, mode):
    from devito_b200 import _lib as L_
    ls, fobjs, F, cobjs, traces, keep = _build(system, fields, coefs, mode)
    ls.apply(fobjs, cobjs, lo, hi, tm, tM)
    assert L_.lib().b2_staging_outstanding() == 0
    return F, traces


def _interpreted(name):
    if name not in _interp:
        if name.startswith('sys_'):
            g = load_golden(name)
            case = SR.from_fixture(g)
        else:
            case = SC.synthetic(name)
        F, tr = SR.run(*case)
        _interp[name] = (case, F, tr)
    return _interp[name]


@pytest.mark.parametrize('mode', ['host', 'device'])
@pytest.mark.parametrize('name', SC.FIXTURES)
def test_fixture_system(name, mode):
    g = load_golden(name)
    case, F64, tr64 = _interpreted(name)
    system = case[0]
    F, tr = _execute(*case, mode)
    got = SR.fixture_outputs(g, system, F, tr)
    want = SR.fixture_outputs(g, system, F64, tr64)
    nf = len(g['field_names'])
    ref = list(g['ref_fields']) + [g[f'ref_trace{i}'] for i in range(len(got[1]))]
    got, want = list(got[0]) + got[1], list(want[0]) + want[1]
    e64 = [rel_linf(a, b) for a, b in zip(got, want)]
    eref = [rel_linf(a, b) for a, b in zip(got, ref)]
    print(f'{name} {mode}: vs float64 fields {max(e64[:nf]):.1e} traces {max(e64[nf:]):.1e}; '
          f'vs reference fields {max(eref[:nf]):.1e} traces {max(eref[nf:]):.1e}')
    assert max(e64) < TOL, e64
    assert max(eref) < TOL_REF, eref


@pytest.mark.parametrize('mode', ['host', 'device', 'shuffled'])
@pytest.mark.parametrize('name', list(SC.SYNTHETIC))
def test_synthetic_system(name, mode):
    case, F64, tr64 = _interpreted(name)
    system = case[0]
    F, tr = _execute(*case, mode)
    a, b = SC.outputs(system, F, tr)
    a64, b64 = SC.outputs(system, F64, tr64)
    ef = [rel_linf(x, y) for x, y in zip(a, a64)]
    et = [rel_linf(x, y) for x, y in zip(b, b64)]
    print(f'{name} {mode}: fields {max(ef):.1e} traces {max(et):.1e}')
    assert max(ef) < TOL and max(et) < TOL, (ef, et)


# ---------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------
_H = 2


def _small(nd, stages=None, coefs=None):
    """A small valid system: field 0 two-slot, field 1 one-slot; an update of 0, a scratch stage of 1; one source into
    field 0, one receiver of field 1. Returns (system, fields, coefs, lo, hi)."""
    shape = (12, 10, 9)[3 - nd:]
    alloc = tuple(s + 2 * _H for s in shape)
    rng = np.random.default_rng(5)
    T = [2, 1]
    fields = [rng.standard_normal((t,) + alloc).astype(np.float32) for t in T]
    z = (0,) * nd
    x1 = (1,) + (0,) * (nd - 1)
    if stages is None:
        stages = [(0, 1, [(0, 0, x1, 0.5, 0), (1, 0, z, 0.25, -1)]), (1, 0, [(0, 1, x1, 1.0, -1)])]
    if coefs is None:
        coefs = [rng.uniform(0.5, 1.5, shape).astype(np.float32)]
    pos = np.array([[s / 2 + 0.3 for s in shape]]) * np.array(SC.spacing_of(nd))
    from oracle import oracle as O
    gp, ws = O.tabulate(pos, (0.0,) * nd, SC.spacing_of(nd), 1, 'linear')
    sp = dict(data=rng.standard_normal((4, 1)).astype(np.float32), gp=gp.astype(np.int32), w=ws, r=1, p_m=0, p_M=0)
    system = dict(nd=nd, halo=_H, T=T, stages=stages,
                  injections=[dict(sp=sp, fields=[0], tshift=1, scale=0.5, kind=0, param=None)],
                  interpolations=[dict(sp=sp, field=1, tshift=0)])
    return system, fields, coefs, (0,) * nd, tuple(s - 1 for s in shape)


def _refused(system, fields, coefs, lo, hi, edit=None):
    from devito_b200 import _lib as L_
    ls, fobjs, F, cobjs, traces, keep = _build(system, fields, coefs, 'host')
    F0 = [f.copy() for f in F]
    tr0 = {k: v.copy() for k, v in traces.items()}
    a, timers, hold = ls.arguments(fobjs, cobjs, lo, hi, 0, 2)
    if edit is not None:
        edit(a)
    rc = L_.lib().b2_system_forward(ctypes.byref(a))
    assert rc == B2_ERR_INVALID, (rc, L_.lib().b2_last_error().decode())
    assert L_.lib().b2_staging_outstanding() == 0
    assert all(np.array_equal(f, f0) for f, f0 in zip(F, F0))
    assert all(np.array_equal(traces[k], tr0[k]) for k in tr0)
    return L_.lib().b2_last_error().decode()


def test_small_system_runs():
    """The base of the refusals is itself valid and agrees with the interpreter."""
    for nd in (2, 3):
        system, fields, coefs, lo, hi = _small(nd)
        F, tr = _execute(system, fields, coefs, lo, hi, 0, 2, 'host')
        F64, tr64 = SR.run(system, fields, coefs, lo, hi, 0, 2)
        a, b = SC.outputs(system, F, tr)
        a64, b64 = SC.outputs(system, F64, tr64)
        assert max(rel_linf(x, y) for x, y in zip(a + b, a64 + b64)) < TOL


@pytest.mark.parametrize('nd', [2, 3])
def test_refuses_shifted_read_of_the_written_level(nd):
    z, x1 = (0,) * nd, (0,) * (nd - 1) + (1,)
    # a one-slot field: every level is the written one (tshift 1 != out_tshift 0 still names the same slot)
    msg = _refused(*_small(nd, stages=[(1, 0, [(1, 1, x1, 1.0, -1), (0, 0, z, 1.0, -1)])]))
    assert 'level it writes' in msg
    msg = _refused(*_small(nd, stages=[(1, 0, [(1, 0, x1, 1.0, -1)])]))
    assert 'level it writes' in msg
    # a two-slot field read at the level it writes
    msg = _refused(*_small(nd, stages=[(0, 1, [(0, 1, x1, 1.0, -1)])]))
    assert 'level it writes' in msg


def _set_inject(attr, value, j=None):
    def edit(a):
        if j is None:
            setattr(a.inject[0], attr, value)
        else:
            getattr(a.inject[0], attr)[j] = value
    return edit


SPARSE_EDITS = {
    'inject_nfields_0': _set_inject('nfields', 0),
    'inject_nfields_4': _set_inject('nfields', 4),
    'inject_field_high': _set_inject('fields', 2, 0),
    'inject_field_negative': _set_inject('fields', -1, 0),
    'inject_third_field_high': lambda a: (_set_inject('nfields', 3)(a), _set_inject('fields', 0, 1)(a),
                                          _set_inject('fields', 7, 2)(a)),
    'param_kind_3': _set_inject('param_kind', 3),
    'param_kind_negative': _set_inject('param_kind', -1),
    'interp_field_high': lambda a: setattr(a.interp[0], 'field', 2),
    'interp_field_negative': lambda a: setattr(a.interp[0], 'field', -1),
    # the sparse tables themselves, refused before any of them is staged
    'interp_p_M_high': lambda a: setattr(a.interp[0].s.contents, 'p_M', 1),      # = npoint_total
    'inject_no_weight_table': lambda a: a.inject[0].s.contents.w.__setitem__(1, None),
}
_SPARSE_MSG = {'interp_p_M_high': 'point range', 'inject_no_weight_table': 'weight table'}


@pytest.mark.parametrize('edit', list(SPARSE_EDITS))
def test_refuses_bad_sparse_indices(edit):
    msg = _refused(*_small(3), edit=SPARSE_EDITS[edit])
    if edit in _SPARSE_MSG:
        assert _SPARSE_MSG[edit] in msg
    else:
        assert 'injection' in msg or 'interpolation' in msg


@pytest.mark.parametrize('side', [-1, 1])
@pytest.mark.parametrize('axis', [0, 1, 2])
@pytest.mark.parametrize('nd', [2, 3])
def test_refuses_offset_leaving_the_allocation(nd, axis, side):
    if axis >= nd:
        pytest.skip('2-D grids have two axes')
    off = [0] * nd
    off[axis] = side * (_H + 1)
    msg = _refused(*_small(nd, stages=[(0, 1, [(0, 0, tuple(off), 1.0, -1)])]))
    assert 'leaves the allocated array' in msg
    # an offset of one halo fits the box, but not the box widened by one cell
    off[axis] = side * _H
    msg = _refused(*_small(nd, stages=[(1, 0, [(0, 0, tuple(off), 1.0, -1)], 1)]))
    assert 'leaves the allocated array' in msg


@pytest.mark.parametrize('nd', [2, 3])
def test_refuses_coefficient_array_of_another_shape(nd):
    shape = (12, 10, 9)[3 - nd:]
    for d in range(nd):
        for delta in (-1, 1):
            s = list(shape)
            s[d] += delta
            msg = _refused(*_small(nd, coefs=[np.ones(s, dtype=np.float32)]))
            assert "grid's shape" in msg
    # the second array disagrees with the first
    msg = _refused(*_small(nd, coefs=[np.ones(shape, dtype=np.float32), np.ones(shape[:-1] + (shape[-1] + 2,),
                                                                               dtype=np.float32)]))
    assert "grid's shape" in msg


def test_refuses_too_many_fields():
    from devito_b200 import _lib as L_

    def edit(a):
        ptrs = [a.fields[i % 2] for i in range(SC.MAX_FIELDS + 1)]
        a.fields = (ctypes.POINTER(L_.Dataobj) * len(ptrs))(*ptrs)
        a.nfields = len(ptrs)
    msg = _refused(*_small(3), edit=edit)
    assert 'fields' in msg


def test_refuses_bad_box_widening():
    z = (0,) * 3
    assert 'malformed' in _refused(*_small(3, stages=[(1, 0, [(0, 0, z, 1.0, -1)], _H + 1)]))
    assert 'malformed' in _refused(*_small(3, stages=[(1, 0, [(0, 0, z, 1.0, -1)], -1)]))
    assert 'malformed' in _refused(*_small(3, stages=[(1, 0, [(0, 0, z, 1.0, 0)], 1)]))    # coefficient array
