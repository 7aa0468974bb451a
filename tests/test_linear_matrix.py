"""The generic constant-coefficient update (`b2_linear_forward`, DESIGN §3.3e) against float64 (tests/linear_ref.py).

Each case builds its equation from a seeded tap table (tests/linear_cases.py) with Constants, spacings and `dt` in
its coefficients, starts from white noise in every slot and halo cell and runs K = 6 steps on 1-D, 2-D and 3-D grids
with anisotropic spacing. The box of every slot must be within 1e-5 of float64; every other cell, halo included, and
every slot not written must be bit-identical to the input. tests/test_linear_ref.py shows that the kinds of bug this
could hide move these cases by at least 100 times that bound.
"""
import numpy as np
import pytest

import linear_cases as LC

pytestmark = pytest.mark.gpu


def _apply(c, op, **kw):
    _, _, over = LC.bounds(c)
    kw = dict(dict(dt=LC.DEFAULTS['dt'], time_m=c['time_m'], time_M=c['time_M']), **over, **kw)
    op.apply(**kw)


def _run(c, **kw):
    op, u, _, _ = LC.build(c)
    assert op.backend == 'cuda-sm90a' and op._plan['kind'] == 'linear'
    _apply(c, op, **kw)
    return np.array(u.data_with_halo)


@pytest.mark.parametrize('m', LC.MATRIX, ids=LC.case_id)
def test_matrix(m):
    c = LC.case(*m)
    LC.check(c, _run(c), LC.reference(c))


def test_overrides_at_apply_equal_values_on_the_objects():
    """`a=`, `b=`, `dt=` and `h_x=` at apply: the same result as a grid of that spacing with the Constants set, and
    that of float64 at those values, with `a` in many taps."""
    c = LC.case(2, 'cloud', 'fwd2', 'interior')
    o = LC.OVERRIDES
    op, u, _, _ = LC.build(c)
    assert op.backend == 'cuda-sm90a'
    _apply(c, op, **o)
    over = np.array(u.data_with_halo)
    op2, u2, (a, b), _ = LC.build(c, grid_spacing=(o['h_x'],) + LC.spacing(2)[1:])
    a.data, b.data = o['a'], o['b']
    _apply(c, op2, dt=o['dt'])
    assert np.array_equal(over, np.array(u2.data_with_halo))
    want = LC.reference(c, LC.values(2, **o))
    LC.check(c, over, want)
    assert LC.box_error(c, want, LC.reference(c)) > 100 * LC.TOL       # the overrides matter


@pytest.mark.parametrize('times', ['fwd4', 'bwd3'])
def test_split_time_range_is_bit_identical(times):
    c = LC.case(3, 'cloud', times, 'custom')
    op, u, _, _ = LC.build(c)
    mid = c['time_m'] + 2
    parts = [(c['time_m'], mid), (mid + 1, c['time_M'])]
    for m, M in (parts if c['wshift'] > 0 else parts[::-1]):
        _apply(c, op, time_m=m, time_M=M)
    assert np.array_equal(np.array(u.data_with_halo), _run(c))


@pytest.mark.parametrize('times', ['fwd2', 'bwd3'])
def test_host_staged_call_is_bit_identical(times):
    c = LC.case(2, 'star', times, 'custom')
    got = _run(c, resident=False)
    assert np.array_equal(got, _run(c))
    LC.check(c, got, LC.reference(c))


def test_field_override():
    """`u=` another TimeFunction of the same layout: that one is updated, the operator's own is untouched."""
    from devito_b200 import TimeFunction
    c = LC.case(3, 'star', 'fwd4', 'interior')
    op, u, _, g = LC.build(c)
    other = dict(c, f=np.random.default_rng(9).standard_normal(c['f'].shape).astype(np.float32))
    v = TimeFunction(name='v', grid=g, time_order=c['time_order'], space_order=c['so'])
    v.data_with_halo[:] = other['f']
    _apply(c, op, u=v)
    assert np.array_equal(np.array(u.data_with_halo), c['f'])
    LC.check(other, np.array(v.data_with_halo), LC.reference(other))


@pytest.mark.parametrize('shape', [(65600, 2, 3), (262200, 3)], ids=['3d-x-stride', '2d-y-stride'])
def test_launch_limits(shape):
    """More than 65 535 x-planes (3-D: the grid-stride loop over x) and more than 4 x 65 535 rows along the kernel's
    y (2-D: x; the grid-stride loop over y), about 11 MB and 7 MB per slot."""
    c = LC.case(len(shape), ('star', 2), 'fwd1', 'whole', shape=shape)
    LC.check(c, _run(c), LC.reference(c))
