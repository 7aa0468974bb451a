"""The two-level isotropic sweep (`iso_tma2<4,scalar>`: one pass advances u[t] to u[t+1] and u[t+2]) against the
float64 reference (tests/ref64.py) on an anisotropic, non-cubic grid.

The pass is taken for so = 8 with a scalar vp when every time slot is zero outside the update box and no source
support reaches outside it; B2_ISO2=2 lets it run on these small grids and B2_ISO_LX cuts x into chunks. The
grid has partial z and y tiles (148 = 2*64 + 20, 45 = 2*16 + 13), the sub-boxes end on a partial float4 along z
(138, 141 and 139 points: tails of 2, 1 and 3), the source straddles a tile edge in y and z and an x-chunk edge, and every time slot, halo included, is compared. Each case asserts which sweep kernel ran, and two
layouts that must fall back to the one-step kernel (a non-zero halo, a source reaching into the halo) check that.
"""
import functools

import numpy as np
import pytest

from helpers import rel_linf
import kernel_cases as KC
import ref64

pytestmark = pytest.mark.gpu

SO = 8
SHAPE = (70, 45, 148)
LX = 32                                      # x-chunk length: chunks [0, 32), [32, 64), [64, 70)
TWO, ONE = 'iso_tma2<4,scalar>', 'iso_tma<4,scalar>'
# source between cells 31|32 (x-chunk edge), 15|16 (y-tile edge), 63|64 (z-tile edge); receivers elsewhere
SRC = np.array([[31.5, 15.4, 63.6]])
REC = np.array([[31.5, 15.4, 63.6], [10.2, 40.7, 140.3], [60.9, 3.3, 2.5], [45.0, 30.0, 100.25]])
NT = 9


def _lib():
    from devito_b200 import _lib as L
    return L.lib()


def _tables(pts, seed):
    coords = (pts * np.array(KC.SPACING)).astype(np.float32)
    t = KC.sparse_tables(coords, 'linear', NT)
    t['data'] = np.random.default_rng(seed).standard_normal(t['data'].shape).astype(np.float32)
    return coords, t


@functools.lru_cache(maxsize=None)
def _setup(rec_toff, src_pts=None):
    from devito_b200 import Constant, Eq, Grid, Function, Operator, SparseTimeFunction, TimeFunction, solve
    grid = Grid(shape=SHAPE, extent=tuple((n - 1) * h for n, h in zip(SHAPE, KC.SPACING)))
    u = TimeFunction(name='u', grid=grid, time_order=2, space_order=SO)
    damp = Function(name='damp', grid=grid, space_order=SO)
    vp = Constant(name='vp', value=2.0)
    m = 1 / vp ** 2
    scoords, stab = _tables(SRC if src_pts is None else np.array(src_pts), 5)
    rcoords, rtab = _tables(REC, 6)
    src = SparseTimeFunction(name='src', grid=grid, npoint=len(scoords), nt=NT, interpolation='linear', r=1,
                             coordinates=scoords)
    src.data[:] = stab['data']
    rec = SparseTimeFunction(name='rec', grid=grid, npoint=len(rcoords), nt=NT, interpolation='linear', r=1,
                             coordinates=rcoords)
    dt = grid.stepping_dim.spacing
    eqs = [Eq(u.forward, solve(m * u.dt2 - u.laplace + damp * u.dt, u.forward))]
    eqs += src.inject(field=u.forward, expr=src * dt ** 2 / m)
    eqs += rec.interpolate(expr=u.forward if rec_toff else u)
    op = Operator(eqs)
    assert op.backend == 'cuda-sm90a'
    return op, u, damp, rec, stab, rtab


def _case(box, halo_noise=False):
    """u: white noise inside the box, zero elsewhere (unless halo_noise); damp: white noise everywhere."""
    rng = np.random.default_rng(1)
    a = tuple(n + 2 * SO for n in SHAPE)
    lo, hi = box
    u = np.zeros((3,) + a, dtype=np.float32) if not halo_noise else rng.standard_normal((3,) + a).astype(np.float32)
    sl = tuple(slice(l + SO, h + SO + 1) for l, h in zip(lo, hi))
    u[(slice(None),) + sl] = rng.standard_normal((3,) + tuple(h - l + 1 for l, h in zip(lo, hi)))
    damp = (0.1 * rng.uniform(0.0, 1.0, a)).astype(np.float32)
    return u, damp


FULL = ((0, 0, 0), tuple(n - 1 for n in SHAPE))
SUB = ((2, 3, 4), (SHAPE[0] - 3, SHAPE[1] - 2, SHAPE[2] - 7))             # nz = 138
TAIL1 = ((1, 0, 0), (SHAPE[0] - 2, SHAPE[1] - 1, SHAPE[2] - 8))           # nz = 141
TAIL3 = ((0, 2, 4), (SHAPE[0] - 1, SHAPE[1] - 3, SHAPE[2] - 6))           # nz = 139
BOXES = {'full': FULL, 'sub': SUB, 'tail1': TAIL1, 'tail3': TAIL3}


def _run(monkeypatch, box, ranges, rec_toff=0, halo_noise=False, src_pts=None):
    monkeypatch.setenv('B2_ISO2', '2')
    monkeypatch.setenv('B2_ISO_LX', str(LX))
    op, u, damp, rec, stab, rtab = _setup(rec_toff, src_pts)
    u0, d = _case(box, halo_noise)
    u.data_with_halo[:] = u0
    damp.data_with_halo[:] = d
    rec.data[:] = 0.0
    lo, hi = box
    bounds = dict(x_m=lo[0], x_M=hi[0], y_m=lo[1], y_M=hi[1], z_m=lo[2], z_M=hi[2])
    dt = float(KC.O.critical_dt(SO, 3, min(KC.SPACING), 2.5))
    kernels = []
    for t0, t1 in ranges:
        op.apply(time_m=t0, time_M=t1, dt=dt, **bounds)
        kernels.append(_lib().b2_last_sweep_kernel().decode())
    w64, _ = KC.weights('iso', SO)
    rec_t = dict(rtab, data=np.zeros_like(rtab['data']))
    want, traces = ref64.iso_forward(u0, SO, w64, dt, ranges[0][0], ranges[-1][1], damp=d, param=('vp', 2.0),
                                     lo=lo, hi=hi, src=stab, rec=rec_t, rec_toff=rec_toff)
    got = np.array(u.data_ro_with_halo)
    assert np.abs(got).max() > 0.5
    assert rel_linf(got, want) < KC.TOL['iso']               # all three slots, halo included
    assert rel_linf(np.array(rec.data), traces) < KC.TOL['iso']
    return kernels


@pytest.mark.parametrize('nsteps', [4, 5])
@pytest.mark.parametrize('box', list(BOXES))
def test_two_level_matches_float64(monkeypatch, nsteps, box):
    lo, hi = BOXES[box]
    assert box == 'full' or (hi[2] - lo[2] + 1) % 4 != 0
    ks = _run(monkeypatch, BOXES[box], [(1, nsteps)])
    assert ks == [TWO]


@pytest.mark.parametrize('rec_toff', [0, 1])
def test_two_level_receivers(monkeypatch, rec_toff):
    assert _run(monkeypatch, FULL, [(1, 4)], rec_toff=rec_toff) == [TWO]


def test_two_level_restart_over_sub_ranges(monkeypatch):
    # 1..2 (one pass), 3..5 (one step, one pass), 6..6 (one step: the one-step kernel)
    assert _run(monkeypatch, FULL, [(1, 2), (3, 5), (6, 6)]) == [TWO, TWO, ONE]


def test_falls_back_on_a_nonzero_halo(monkeypatch):
    assert _run(monkeypatch, SUB, [(1, 4)], halo_noise=True) == [ONE]


def test_falls_back_when_a_source_reaches_the_halo(monkeypatch):
    # a support cell at x = -1: outside the update box
    assert _run(monkeypatch, FULL, [(1, 4)], src_pts=((-0.5, 20.2, 70.3),)) == [ONE]


def test_two_level_reports_sparse_sections(monkeypatch):
    # the pass's injection and interpolation launches are sampled like the one-step loop's
    monkeypatch.setenv('B2_ISO2', '2')
    op, u, damp, rec, _, _ = _setup(0)
    u0, d = _case(FULL)
    u.data_with_halo[:] = u0
    damp.data_with_halo[:] = d
    dt = float(KC.O.critical_dt(SO, 3, min(KC.SPACING), 2.5))
    summary = op.apply(time_m=1, time_M=6, dt=dt)
    assert _lib().b2_last_sweep_kernel().decode() == TWO
    assert summary['section0'].time > 0 and summary['section1'].time > 0 and summary['section2'].time > 0
