"""The isotropic TMA sweep with a scalar velocity takes the update coefficient A = 1/(m/dt^2 + damp/dt) of every
x-plane whose damp repeats the centre plane's, bit for bit over the update box, from one tile it pins per CTA
instead of streaming it (b2_iso.cu::k_iso_tma). These cases check that rule and its bookkeeping against float64
(tests/ref64.py) on the anisotropic, non-cubic grid of tests/kernel_cases.py.

The damping field is a sum of per-axis profiles, like the reference's absorbing layer, so that every x-plane outside
the x-layers repeats. A few interior planes are then perturbed inside the box (one on an x-chunk boundary of
B2_ISO_LX=12), so the repeated set is not contiguous, and one plane only outside the box's rows, where the rule still
counts it as repeated. `b2_last_iso_coef_reuse` must equal the count numpy finds by the same rule.
"""
import ctypes
import functools

import numpy as np
import pytest

from helpers import rel_linf
import kernel_cases as KC
import ref64

pytestmark = pytest.mark.gpu

LAYER = 4                     # absorbing-layer width (points) of the per-axis profiles


def _lib():
    from devito_b200 import _lib
    return _lib.lib()


def _profile(n, so):
    """A ramp over the LAYER points next to each end of the domain, and the halo; zero inside."""
    i = np.arange(n + 2 * so, dtype=np.float64) - so
    d = np.maximum(np.maximum(LAYER - i, i - (n - 1 - LAYER)), 0.0) / LAYER
    return (0.08 * d * d).astype(np.float32)


# x-planes perturbed inside the box, and the one perturbed outside the box's rows, per grid
PERTURBED = {KC.SHAPE: ((9, 12, 24), 17),                      # 12, 24: first planes of B2_ISO_LX=12 chunks
             KC.MULTI: ((2, 5, 10), 7)}


def layered_damp(shape, so, lo):
    """sum of per-axis profiles (float32, x + y + z), then perturbed planes; lo: the box's lower corner"""
    p = [_profile(n, so) for n in shape]
    damp = (p[0][:, None, None] + p[1][None, :, None]) + p[2][None, None, :]
    y, z = so + lo[1] + 3, so + lo[2] + 5                        # inside every box used below
    inside, outside = PERTURBED[shape]
    for x in inside:
        damp[so + x, y, z] += np.float32(1e-3)
    damp[so + outside, so + lo[1] - 1, z] += np.float32(1e-3)   # outside the box's rows: still repeated
    return damp


def expected_reuse(damp, so, lo, hi):
    """the rule: planes of the box whose damp equals the centre plane's bit for bit over the box's rows and columns"""
    o = [so + l for l in lo]
    n = [h - l + 1 for l, h in zip(lo, hi)]
    box = damp[o[0]:o[0] + n[0], o[1]:o[1] + n[1], o[2]:o[2] + n[2]].view(np.uint32)
    ref = damp[o[0] + n[0] // 2, o[1]:o[1] + n[1], o[2]:o[2] + n[2]].view(np.uint32)
    return int(np.count_nonzero((box == ref[None]).all(axis=(1, 2))))


@functools.lru_cache(maxsize=None)
def _setup(so, adjoint, shape=KC.SHAPE):
    from devito_b200 import Constant, Eq, Function, Grid, Operator, TimeFunction, solve
    c = KC.iso_case(so, 'scalar', shape=shape)
    grid = Grid(shape=shape, extent=tuple((n - 1) * h for n, h in zip(shape, KC.SPACING)))
    u = TimeFunction(name='v' if adjoint else 'u', grid=grid, time_order=2, space_order=so)
    damp = Function(name='damp', grid=grid, space_order=so)
    m = 1 / Constant(name='vp', value=float(c['param'][1])) ** 2
    nxt = u.backward if adjoint else u.forward
    pde = m * u.dt2 - u.laplace + damp * (u.dt.T if adjoint else u.dt)
    op = Operator([Eq(nxt, solve(pde, nxt))])
    assert op.backend == 'cuda-sm90a'
    return op, u, damp, c


def _apply(so, adjoint, box, white=False, shape=KC.SHAPE, **kw):
    """(u after time 1..K, damp, lo, hi, case)"""
    op, u, damp, c = _setup(so, adjoint, shape)
    lo, hi = box if box is not None else ((0, 0, 0), tuple(n - 1 for n in shape))
    d = c['damp'] if white else layered_damp(shape, so, lo)
    damp.data_with_halo[:] = d
    u.data_with_halo[:] = c['u']
    bounds = dict(x_m=lo[0], x_M=hi[0], y_m=lo[1], y_M=hi[1], z_m=lo[2], z_M=hi[2])
    op.apply(time_m=1, time_M=KC.K, dt=c['dt'], **bounds, **kw)
    assert _lib().b2_last_sweep_kernel().decode() == f'iso_tma<{so // 2},scalar>'
    return np.array(u.data_ro_with_halo), d, lo, hi, c


def _last_call_streamed():
    prof = (ctypes.c_double * 5)()
    _lib().b2_last_call_profile(prof)
    return prof[4] == 1.0


BOXES = {'full': None, 'sub': KC.SUBBOX}


@pytest.mark.parametrize('lx', [None, '12'])
@pytest.mark.parametrize('box', ['full', 'sub'])
@pytest.mark.parametrize('adjoint', [False, True], ids=['forward', 'adjoint'])
@pytest.mark.parametrize('so', [4, 8, 12, 16])
def test_reuse_matches_float64(so, adjoint, box, lx, monkeypatch):
    if lx:
        monkeypatch.setenv('B2_ISO_LX', lx)
    got, d, lo, hi, c = _apply(so, adjoint, BOXES[box])
    want, _ = ref64.iso_forward(c['u'], so, [ref64.fd2_weights(so, h) for h in KC.SPACING], c['dt'], 1, KC.K,
                                damp=d, param=c['param'], lo=lo, hi=hi, adjoint=adjoint)
    assert np.abs(got).max() > 0.5
    assert rel_linf(got, want) < KC.TOL['iso']
    n = expected_reuse(d, so, lo, hi)
    assert 0 < n < hi[0] - lo[0] + 1 - 3                        # the three perturbed planes are streamed
    assert _lib().b2_last_iso_coef_reuse() == n


@pytest.mark.parametrize('adjoint', [False, True], ids=['forward', 'adjoint'])
def test_reuse_on_several_tiles(adjoint):
    """kernel_cases.MULTI (13, 44, 300) at so = 8: 3 x 3 yz-tiles of 16 x 128, the last of each partial. The layered
    damp differs from tile to tile (its y and z ramps), so a CTA that took its pinned A from another tile than its
    own would change the answer."""
    got, d, lo, hi, c = _apply(8, adjoint, None, shape=KC.MULTI)
    want, _ = ref64.iso_forward(c['u'], 8, [ref64.fd2_weights(8, h) for h in KC.SPACING], c['dt'], 1, KC.K,
                                damp=d, param=c['param'], lo=lo, hi=hi, adjoint=adjoint)
    assert np.abs(got).max() > 0.5
    assert rel_linf(got, want) < KC.TOL['iso']
    n = expected_reuse(d, 8, lo, hi)
    assert 0 < n < hi[0] - lo[0] + 1 - 3
    assert _lib().b2_last_iso_coef_reuse() == n


@pytest.mark.parametrize('box', ['full', 'sub'])
def test_streamed_loop_equals_reuse(box, monkeypatch):
    """The streamed time loop tabulates A chunk by chunk and streams every tile: the same bits."""
    resident, d, lo, hi, _ = _apply(8, False, BOXES[box])
    assert _lib().b2_last_iso_coef_reuse() == expected_reuse(d, 8, lo, hi) > 0
    monkeypatch.setenv('B2_STREAM', '2')
    monkeypatch.setenv('B2_STREAM_W', '12')
    streamed, *_ = _apply(8, False, BOXES[box], resident=False)
    assert _last_call_streamed()
    assert _lib().b2_last_iso_coef_reuse() == 0
    assert np.array_equal(streamed, resident)


def test_white_noise_damp_reuses_the_centre_plane_only():
    got, d, lo, hi, c = _apply(8, False, None, white=True)
    want, _ = ref64.iso_forward(c['u'], 8, [ref64.fd2_weights(8, h) for h in KC.SPACING], c['dt'], 1, KC.K,
                                damp=d, param=c['param'], lo=lo, hi=hi)
    assert rel_linf(got, want) < KC.TOL['iso']
    assert _lib().b2_last_iso_coef_reuse() == 1
