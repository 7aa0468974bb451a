"""Parity at BASELINE.json's full sizes (iso so=8 1024^3, TTI so=8 768^3) through a size-independent property:
LOCALITY. After K explicit steps a point source has influenced only the cells within K*radius of
its support, so the wavefield in a window around each source must equal a run of the CPU oracle on
a small grid that holds just that window (same local damping values, same source signature). Five
sources are placed where the full-size launch configuration is most exposed — the grid centre, an
x-chunk boundary of the sweep kernel, a corner of the absorbing layer, and the far y / x-z edges —
and everything outside their windows must still be exactly zero.

The CPU twin runs the same check with the oracle on both sides (a 200^3 "big" grid), which
validates the window arithmetic of this test itself without a GPU.
"""
import numpy as np
import pytest

from oracle import oracle as O
from helpers import rel_linf

SO, R, H, VP = 8, 4, 10.0, 1.5
K = 6                      # time steps: support radius K*R - R + 2 = 22 cells  <  WIN/2 - R
WIN = 64                   # window edge; the source's base cell sits at window index 31
BASE = 31


def _signature(nt, npoint):
    """A different, O(1) time series per source (first K+2 samples matter)."""
    t = np.arange(nt, dtype=np.float64)[:, None]
    p = np.arange(npoint, dtype=np.float64)[None, :]
    return (np.cos(0.9 * t + 0.7 * p) * (1.0 + 0.25 * p)).astype(np.float32)


def _coords(bases, origin):
    """Physical coordinates putting source `i` half-way between cells bases[i] and bases[i]+1."""
    return (np.asarray(origin, dtype=np.float64)[None, :] + (np.asarray(bases) + 0.5) * H).astype(np.float32)


TTI = dict(epsilon=0.3, delta=0.2, theta=0.7, phi=0.35)     # preset `constant-tti`


def _oracle_run(kind, u, v, damp, dt, src):
    w2 = [O.fd2_weights(SO, H)] * 3
    if kind == 'iso':
        O.iso_forward(u, SO, w2, dt, 1, K, damp=damp, vp=VP, src=src)
    else:
        w1 = [O.fd1_half_weights(SO, H)] * 3
        O.tti_forward(u, v, SO, w2, w1, dt, 1, K, damp, VP, TTI['epsilon'], TTI['delta'], TTI['theta'],
                      TTI['phi'], src=src)


def _small_run(kind, damp_window, sig, dt):
    """Oracle on the WIN^3 window: zero initial state, no absorbing layer of its own. Returns the
    domain part of u (iso) or of u and v stacked (TTI)."""
    n = WIN
    u = np.zeros((3, n + 2 * SO, n + 2 * SO, n + 2 * SO), dtype=np.float32)
    v = np.zeros_like(u)
    damp = np.zeros(u.shape[1:], dtype=np.float32)
    damp[SO:-SO, SO:-SO, SO:-SO] = damp_window
    c = np.full((1, 3), (BASE + 0.5) * H, dtype=np.float32)
    gp, ws = O.tabulate(c, (0., 0., 0.), (np.float32(H),) * 3, 1, 'linear')
    src = dict(data=np.ascontiguousarray(sig.reshape(-1, 1)), gp=gp, w=ws, r=1)
    _oracle_run(kind, u, v, damp, dt, src)
    dom = (slice(None), slice(SO, -SO), slice(SO, -SO), slice(SO, -SO))
    return u[dom] if kind == 'iso' else np.concatenate([u[dom], v[dom]])


def _check_windows(kind, window_of, damp_window_of, count_nonzero_total, bases, sig, dt):
    """window_of(lo) -> (3 [iso] or 6 [TTI: u then v], WIN, WIN, WIN) block of the big run's DOMAIN
    starting at cell `lo`. Tolerances: BASELINE.json north_star (1e-5 iso, 1e-4 TTI)."""
    nz = 0
    tol = 1e-5 if kind == 'iso' else 1e-4
    for i, b in enumerate(bases):
        lo = tuple(int(x) - BASE for x in b)
        small = _small_run(kind, damp_window_of(lo), sig[:, i], dt)
        big = window_of(lo)
        assert big.shape == small.shape
        assert np.abs(small).max() > 1e-3
        err = rel_linf(big, small)
        assert err < tol, f"source {i} at {b}: window differs from the oracle, rel L-inf {err:.3e}"
        # the wave has not reached the rim of the window
        rim = np.ones(big.shape[1:], dtype=bool)
        rim[R:-R, R:-R, R:-R] = False
        assert not big[:, rim].any()
        nz += int(np.count_nonzero(big))
    assert count_nonzero_total() == nz, "the wavefield is non-zero outside the source windows"


def _dt(kind):
    return float(O.critical_dt(SO, 3, H, VP, eps_max=TTI['epsilon'] if kind == 'tti' else None))


@pytest.mark.parametrize('kind,n', [('iso', 160), ('tti', 120)])
def test_window_locality_oracle_twin(kind, n):
    """CPU: oracle on a 200^3 / 160^3 grid vs oracle on the windows — validates the test's own
    arithmetic."""
    nbl = 20
    N = n + 2 * nbl
    spacing = (np.float32(H),) * 3
    origin = tuple(np.float32(-nbl * H) for _ in range(3))
    dt = _dt(kind)
    bases = [(36, 36, 36), (N - 50, 120, 100), (100, N - 1 - 36, 40)][:3 if kind == 'iso' else 2]
    nt = K + 3
    sig = _signature(nt, len(bases))
    gp, ws = O.tabulate(_coords(bases, origin), origin, spacing, 1, 'linear')
    assert [tuple(g) for g in gp] == bases
    damp = O.damp_field((N, N, N), nbl, spacing, SO)
    u = np.zeros((3, N + 2 * SO, N + 2 * SO, N + 2 * SO), dtype=np.float32)
    v = np.zeros_like(u)
    _oracle_run(kind, u, v, damp, dt, dict(data=sig, gp=gp, w=ws, r=1))
    fields = [u] if kind == 'iso' else [u, v]

    def window_of(lo):
        return np.concatenate([f[:, SO + lo[0]:SO + lo[0] + WIN, SO + lo[1]:SO + lo[1] + WIN,
                                 SO + lo[2]:SO + lo[2] + WIN] for f in fields])

    def damp_window_of(lo):
        return damp[SO + lo[0]:SO + lo[0] + WIN, SO + lo[1]:SO + lo[1] + WIN, SO + lo[2]:SO + lo[2] + WIN]

    _check_windows(kind, window_of, damp_window_of, lambda: sum(int(np.count_nonzero(f)) for f in fields),
                   bases, sig, dt)


def _full_size_bases(N, xchunk):
    """Source cells for the full-size runs: where the launch configuration is most exposed."""
    return [(N // 2 - 1, N // 2 - 1, N // 2 - 1),          # grid centre
            (xchunk - 1, 300, N - 324),                    # straddles a boundary between x-chunks of the sweep
                                                           # kernel (on 132 SMs: 4 x 256 planes at 1024^3,
                                                           # 3 x 256 at 768^3)
            (36, 36, 36),                                  # inside the absorbing corner (damp != 0)
            (N - xchunk - 1, N - 1 - 36, 200),             # far y edge, another x-chunk boundary
            (N - 1 - 36, 500, N - 1 - 36)]                 # far x / z edges


@pytest.mark.gpu
@pytest.mark.parametrize('kind,n', [('iso', 944), ('tti', 688)])
def test_window_locality_full_size(kind, n):
    """GPU: the BASELINE.json sizes — iso so=8 at 1024^3 (headline) and TTI so=8 at 768^3 (C4), both
    including the 40-cell absorbing layers."""
    import torch
    from devito_b200 import TimeFunction
    from devito_b200.seismic import (AcousticWaveSolver, AnisotropicWaveSolver, PointSource, demo_model,
                                     setup_geometry)
    nbl = 40
    N = n + 2 * nbl
    preset = 'constant-isotropic' if kind == 'iso' else 'constant-tti'
    extra = dict(bcs='damp') if kind == 'iso' else {}        # the TTI preset already asks for it
    model = demo_model(preset, shape=(n,) * 3, spacing=(H,) * 3, nbl=nbl, space_order=SO, **extra)
    geometry = setup_geometry(model, tn=30.)
    cls = AcousticWaveSolver if kind == 'iso' else AnisotropicWaveSolver
    solver = cls(model, geometry, space_order=SO)
    dt = float(model.critical_dt)
    assert dt == _dt(kind)
    origin = tuple(float(o) for o in model.grid.origin)
    assert origin == (-nbl * H,) * 3
    bases = _full_size_bases(N, 256)
    coords = _coords(bases, origin)
    src = PointSource(name='src', grid=model.grid, time_range=geometry.time_axis, coordinates=coords)
    assert src.nt >= K + 2
    sig = _signature(src.nt, len(bases))
    src.data[:] = sig
    gp, _ = src.tabulate()
    assert [tuple(int(c) for c in g) for g in gp] == bases
    names = ['u'] if kind == 'iso' else ['u', 'v']
    fields = {nm: TimeFunction(name=nm, grid=model.grid, time_order=2, space_order=SO) for nm in names}
    solver.forward(src=src, time_m=1, time_M=K, **fields)
    if kind == 'iso':
        # the headline's kernel: an even step count, 5 linear sources (40 injection entries), a zero halo, 13.5 GB of u
        from devito_b200 import _lib
        assert _lib.lib().b2_last_sweep_kernel().decode() == 'iso_tma2<4,scalar>'
    devs = [fields[nm].storage.dev for nm in names]
    for dev in devs:
        assert isinstance(dev, torch.Tensor) and dev.is_cuda
        assert tuple(dev.shape) == (3,) + (N + 2 * SO,) * 3
    damp = model.damp.data_ro_domain

    def window_of(lo):
        return np.concatenate([dev[:, SO + lo[0]:SO + lo[0] + WIN, SO + lo[1]:SO + lo[1] + WIN,
                                   SO + lo[2]:SO + lo[2] + WIN].cpu().numpy() for dev in devs])

    def damp_window_of(lo):
        return np.asarray(damp[lo[0]:lo[0] + WIN, lo[1]:lo[1] + WIN, lo[2]:lo[2] + WIN])

    _check_windows(kind, window_of, damp_window_of,
                   lambda: sum(int(torch.count_nonzero(dev).item()) for dev in devs), bases, sig, dt)
