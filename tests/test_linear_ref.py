"""The float64 restatement of the generic update (tests/linear_ref.py) and the recogniser's tap tables, on the CPU.

1. Sensitivity: every mutation of linear_ref.MUTATIONS moves every matrix case it applies to by at least 100 times the
   GPU bound, so a kernel with that kind of bug fails tests/test_linear_matrix.py.
2. The bound is justified: a float32 NumPy run of the 64-tap, 4-level cases stays within a tenth of it.
3. The recogniser's taps, evaluated at apply, are the test's own tables at the test's values of the Constants, `dt`
   and the spacings, including values overridden at apply.
4. Updates the kernel cannot run exactly are not recognised: a level read that shares the written slot, 65 taps,
   5 levels.
"""
import numpy as np
import pytest

import linear_cases as LC
import linear_ref as LR
from helpers import rel_linf


def _applies(mut, c):
    if mut == 'axes_reversed':
        return c['nd'] > 1
    if mut == 'backward_ascending':
        return c['wshift'] < 0
    if mut == 'drop_last_tap':
        return len(c['table']) == 64
    if mut == 'halo_zero':
        return LC.reaches_halo(c)
    return True


@pytest.mark.parametrize('mut', sorted(LR.MUTATIONS))
def test_mutation_moves_every_matrix_case(mut):
    moved = {}
    for m in LC.MATRIX:
        c = LC.case(*m)
        if _applies(mut, c):
            moved[LC.case_id(m)] = LC.box_error(c, LC.reference(c, mut=mut), LC.reference(c))
    assert moved
    weak = {k: v for k, v in moved.items() if v < 100 * LC.TOL}
    assert not weak, weak


@pytest.mark.parametrize('nd', [1, 2, 3])
def test_float32_run_is_within_a_tenth_of_the_bound(nd):
    c = LC.case(nd, 'cloud', 'fwd4', 'whole')
    assert len(c['table']) == 64 and len({s for s, *_ in c['table']}) == 4
    err = LC.box_error(c, LC.reference(c, dtype=np.float32), LC.reference(c))
    assert 0 < err < LC.TOL / 10


def test_reference_is_jacobi_and_writes_only_the_box():
    """One step by hand: every level read before the write, the halo as stored, nothing outside the box."""
    rng = np.random.default_rng(1)
    f = rng.standard_normal((2, 9, 7))
    taps = [(0, (0, 0), 0.5), (0, (1, 0), 0.25), (0, (0, -1), -0.125), (0, (-1, 1), 2.0)]
    got = LR.run(f, 1, taps, 1, (0, 2), (6, 3), 4, 4)
    want = f.copy()
    for x in range(1, 8):
        for y in range(3, 5):
            want[1, x, y] = sum(c * f[0, x + o[0], y + o[1]] for _, o, c in taps)
    assert np.array_equal(got, want)


@pytest.mark.parametrize('m', LC.MATRIX, ids=LC.case_id)
def test_recogniser_taps_are_the_table(m):
    c = LC.case(*m)
    op, _, _, _ = LC.build(c)
    assert op.backend == 'cuda-sm90a' and op._plan['kind'] == 'linear'
    assert op._plan['wshift'] == c['wshift']
    lo, hi, over = LC.bounds(c)
    for v, kw in ((LC.values(c['nd']), dict(dt=LC.DEFAULTS['dt'])),
                  (LC.values(c['nd'], **LC.OVERRIDES), LC.OVERRIDES)):
        args = op.arguments(time_m=c['time_m'], time_M=c['time_M'], **over, **kw)
        want = LC.coefficients(c['table'], c['nd'], v)
        got = args['taps']
        assert [(s, tuple(o)) for s, o, _ in got] == [(s, o) for s, o, _ in want]
        np.testing.assert_allclose([x for *_, x in got], [x for *_, x in want], rtol=1e-6, atol=0)
        assert (args['lo'], args['hi']) == (lo, hi)
    distinct = {(s, o) for s, o, _, _ in c['table']}
    assert len(op._plan['taps']) == len(distinct)
    if m[1] == 'merge':
        assert len(distinct) < len(c['table'])


def test_constant_override_reaches_every_tap():
    """A Constant in several taps: its value at apply overrides all of them, as setting `.data` does."""
    from devito_b200 import Constant, Eq, Grid, Operator, TimeFunction
    g = Grid(shape=(16, 16))
    u = TimeFunction(name='u', grid=g, time_order=1, space_order=2)
    a, b = Constant(name='a', value=0.5), Constant(name='b', value=0.25)
    op = Operator(Eq(u.forward, u + b * u.dx + a * u.laplace))
    assert op.backend == 'cuda-sm90a'
    over = op.arguments(time_M=3, a=0.625, b=0.0)['taps']
    a.data, b.data = 0.625, 0.0
    assert over == op.arguments(time_M=3)['taps']
    h2 = float(g.spacing[0]) ** 2
    assert rel_linf([c for *_, c in over], [0.625 / h2] * 2 + [1 - 4 * 0.625 / h2] + [0.625 / h2] * 2) < 1e-6


@pytest.mark.parametrize('time_order,wshift,reads', [(2, 1, -2), (1, -1, 1), (3, 1, -3), (2, -1, 2)])
def test_a_level_in_the_written_slot_is_not_recognised(time_order, wshift, reads):
    """(t + reads) and (t + wshift) are the same slot modulo time_order + 1: the kernel would read cells that other
    threads of the same launch are writing."""
    from devito_b200 import Eq, Grid, Operator, TimeFunction
    g = Grid(shape=(12, 10))
    t, (x, _) = g.stepping_dim, g.dimensions
    q = TimeFunction(name='q', grid=g, time_order=time_order, space_order=2)
    lhs = q.forward if wshift > 0 else q.backward
    ok = Operator(Eq(lhs, 0.5 * q.subs(x, x + 1) + 0.25 * q.subs(t, t + reads - wshift)))
    assert ok.backend == 'cuda-sm90a'                     # the same update one level away is fine
    op = Operator(Eq(lhs, 0.5 * q.subs(x, x + 1) + 0.25 * q.subs(t, t + reads)))
    assert op.backend == 'numpy-interpreter'
    assert 'written time slot' in op._why_not


def test_taps_and_levels_beyond_the_kernel_stay_on_the_interpreter():
    from devito_b200 import Eq, Grid, Operator, TimeFunction
    g = Grid(shape=(12, 10))
    t, (x, y) = g.stepping_dim, g.dimensions
    u = TimeFunction(name='u', grid=g, time_order=1, space_order=4)
    offs = [(i, j) for i in range(-4, 5) for j in range(-4, 5)][:65]

    def star(n):
        return sum((0.01 * (k + 1) * u.subs(x, x + i).subs(y, y + j) for k, (i, j) in enumerate(offs[:n])),
                   0.0 * u)
    assert Operator(Eq(u.forward, star(64))).backend == 'cuda-sm90a'
    assert Operator(Eq(u.forward, star(65))).backend == 'numpy-interpreter'
    v = TimeFunction(name='v', grid=g, time_order=5, space_order=2)
    assert Operator(Eq(v.forward, sum(0.1 * v.subs(t, t - k) for k in range(4)))).backend == 'cuda-sm90a'
    assert Operator(Eq(v.forward, sum(0.1 * v.subs(t, t - k) for k in range(5)))).backend == 'numpy-interpreter'
