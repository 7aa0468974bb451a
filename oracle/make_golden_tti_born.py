"""Golden vectors of the reference's centred-TTI linearised modelling, `AnisotropicWaveSolver.jacobian(dm)`
(examples/seismic/tti/wavesolver.py:232-293, operator `BornTTI`, tti/operators.py:532-586), run by the REFERENCE
itself with its own CPU backend, like oracle/make_golden.py:

  PYTHONPATH=oracle/refshim:/root/reference DEVITO_LANGUAGE=openmp DEVITO_ARCH=gcc \
  DEVITO_SAFE_MATH=1 DEVITO_LOGGING=ERROR python oracle/make_golden_tti_born.py

The model perturbation is the smooth Gaussian blob of `dm_blob` (tests rebuild it from the same formula). To keep the
fixtures small they hold the full receiver traces and, of u0, v0, du and dv, the last time level written, on every
second point of the domain along each axis.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, save  # noqa: E402


def dm_blob(N):
    """(N, N, N) float32 Gaussian blob, amplitude 0.05, width 4 cells, 2 cells below the centre."""
    ax = np.arange(N, dtype=np.float64)
    X, Y, Z = np.meshgrid(ax, ax, ax, indexing='ij')
    c = (N - 1) / 2.0
    return (0.05 * np.exp(-((X - c) ** 2 + (Y - c) ** 2 + (Z - c - 2) ** 2) / (2 * 4.0 ** 2))).astype(np.float32)


def tti_born(name, so, n, nbl, tn, preset='constant-tti', **kw):
    from examples.seismic import demo_model, setup_geometry
    from examples.seismic.tti import AnisotropicWaveSolver
    model = demo_model(preset, spacing=(10., 10., 10.), shape=(n, n, n), nbl=nbl, space_order=so,
                       dtype=np.float32, **kw)
    geometry = setup_geometry(model, tn)
    solver = AnisotropicWaveSolver(model, geometry, space_order=so)
    dm = dm_blob(n + 2 * nbl)
    rec, u0, v0, du, dv, _ = solver.jacobian(dm)
    nt = geometry.nt
    slot = (nt - 1) % 3
    sub = lambda f: np.array(f.data[slot][::2, ::2, ::2])
    c = (n + 2 * nbl) // 2
    vp = np.broadcast_to(model.vp.data, (n + 2 * nbl,) * 3)
    save(name, so=so, n=n, nbl=nbl, tn=tn, dt=np.float32(model.critical_dt), nt=nt, slot=slot,
         src=np.array(geometry.src.data), rec=np.array(rec.data), u0=sub(u0), v0=sub(v0), du=sub(du), dv=sub(dv),
         vp_line=np.array(vp[c, c, :], dtype=np.float32), dm_sum=np.float64(dm.astype(np.float64).sum()))


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    tti_born('tti_born3d_so8', so=8, n=20, nbl=8, tn=120.0)
    tti_born('tti_born3d_so4_layers', so=4, n=20, nbl=8, tn=120.0, preset='layers-tti', nlayers=3)
