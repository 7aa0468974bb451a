"""The float64 tap-table interpreter (tests/system_ref.py) against the reference's own elastic and viscoelastic runs,
and the reach of its mutations. CPU only.

The fixtures (oracle/make_golden_system.py) hold the inputs refplugin builds for `b2_system_forward` from the
reference's equations and the reference's outputs of the same run. The interpreter reproduces every field's last level
and every trace within TOL (rel L-inf; measured: at most 5.5e-6, the memory variable r_xz of the viscoelastic case;
traces at most 2.2e-6). Before the scratch stage of `div(v)` was widened into the halo, the receiver just outside the
top face (rec2's last trace) differed from the reference by 2.4e-4 .. 5.4e-4 of the trace maximum.

Each mutation (a kernel bug the tests must see) moves the outputs by at least 100 x TOL in the cases CLAIMS names.
Where a mutation cannot move a case, it is claimed elsewhere:
- coef_no_origin: the fixtures iterate the full domain (origin 0); claimed on the interior-box synthetic cases;
- inject_two: 2-D injects into two fields; claimed on the 3-D fixture and every synthetic case;
- vp_m_swap: the elastic sources have scalar scales; claimed on the synthetic cases;
- swap_xy_2d: claimed on the 2-D cases only;
- guard_narrow: the fixtures' edge receiver moves rec2 by only 4.6e-5 .. 5.4e-4 (5 .. 54 x TOL); claimed on the
  synthetic cases, whose fields hold white noise in the halo.
"""
import numpy as np
import pytest

from helpers import load_golden, rel_linf
import system_cases as SC
import system_ref as SR

TOL = 1e-5
_2D = [n for n in SC.FIXTURES if '2d' in n]
CLAIMS = {
    'coef_shifted': SC.FIXTURES + list(SC.SYNTHETIC),
    'coef_no_origin': ['s3_interior_t3', 's2_interior_t3'],
    'tap_slot_out_T': SC.FIXTURES + list(SC.SYNTHETIC),
    'inject_first': SC.FIXTURES + list(SC.SYNTHETIC),
    'inject_two': ['sys_el3d_so4'] + list(SC.SYNTHETIC),
    'vp_m_swap': list(SC.SYNTHETIC),
    'interp_tshift1': SC.FIXTURES + list(SC.SYNTHETIC),
    'swap_xy_2d': _2D + ['s2_full', 's2_interior_t3'],
    'guard_narrow': list(SC.SYNTHETIC),
}
_cache = {}


def _fixture_run(name, mut=None):
    key = (name, mut)
    if key not in _cache:
        g = load_golden(name)
        s, f, c, lo, hi, tm, tM = SR.from_fixture(g)
        F, tr = SR.run(s, f, c, lo, hi, tm, tM, mut=mut)
        fl, trs = SR.fixture_outputs(g, s, F, tr)
        _cache[key] = list(fl) + trs
    return _cache[key]


def _synthetic_run(name, mut=None):
    key = (name, mut)
    if key not in _cache:
        s, f, c, lo, hi, tm, tM = SC.synthetic(name)
        F, tr = SR.run(s, f, c, lo, hi, tm, tM, mut=mut)
        a, b = SC.outputs(s, F, tr)
        _cache[key] = a + b
    return _cache[key]


def _run(name, mut=None):
    return _fixture_run(name, mut) if name.startswith('sys_') else _synthetic_run(name, mut)


def test_every_mutation_is_claimed():
    assert set(CLAIMS) == set(SR.MUTATIONS)
    assert all(CLAIMS.values())


@pytest.mark.parametrize('name', SC.FIXTURES)
def test_fixture_matches_reference(name):
    g = load_golden(name)
    out = _fixture_run(name)
    nf = len(g['field_names'])
    ref = list(g['ref_fields']) + [g[f'ref_trace{i}'] for i in range(len(out) - nf)]
    errs = [rel_linf(a, b) for a, b in zip(out, ref)]
    print(name, 'fields', ['%.1e' % e for e in errs[:nf]], 'traces', ['%.1e' % e for e in errs[nf:]])
    assert max(errs) < TOL, errs
    # the run must not be trivial: every field and trace carries the wave
    assert all(np.abs(b).max() > 0 for b in ref)


@pytest.mark.parametrize('name', SC.FIXTURES)
def test_fixture_tables(name):
    """What the plugin built: one scratch field (div(v)) filled by the last stage, widened by the receivers' radius
    into the halo; the updates write level t + 1 of two-slot fields; the source goes into the stress diagonal."""
    g = load_golden(name)
    nd, nref = int(g['nd']), len(g['field_names'])
    assert list(g['T']) == [2] * nref + [1]
    assert list(g['stage_tshift']) == [1] * (len(g['stage_out']) - 1) + [0]
    assert int(g['stage_out'][-1]) == nref and int(g['stage_ext'][-1]) == int(g['sp2_r']) == 1
    assert not g['stage_ext'][:-1].any()
    assert int(g['itp_field'][1]) == nref and str(g['field_names'][g['itp_field'][0]]).endswith('_' + 'xyz'[nd - 1] * 2)
    assert int(g['inj_nfields'][0]) == nd
    assert g['coefs'].shape[1:] == tuple(int(a) - 2 * int(g['halo']) for a in g['alloc'])


@pytest.mark.parametrize('name,mut', [(n, m) for m, names in CLAIMS.items() for n in names])
def test_mutation_is_seen(name, mut):
    base, bad = _run(name), _run(name, mut)
    d = max(rel_linf(a, b) for a, b in zip(bad, base))
    print(f'{name} {mut}: {d / TOL:.0f} x TOL')
    assert d >= 100 * TOL, d
