"""Golden vectors of the reference's self-adjoint variable-density visco-acoustic modelling,
`SaIsoAcousticWaveSolver.forward` and `.adjoint` (examples/seismic/self_adjoint/wavesolver.py, operators
`IsoFwdOperator` / `IsoAdjOperator`), run by the REFERENCE itself with its own CPU backend, like oracle/make_golden.py:

  PYTHONPATH=oracle/refshim:/root/reference DEVITO_LANGUAGE=openmp DEVITO_ARCH=gcc \
  DEVITO_SAFE_MATH=1 DEVITO_LOGGING=ERROR python oracle/make_golden_sa.py

vp and b vary smoothly along every axis (`smooth_vp_b`; tests rebuild them from the same formula), so that a buoyancy
sampled at the wrong offset changes the answer; the reference's own example has b = 1 everywhere. The adjoint is run
on the forward's receiver data. To keep the fixtures small they hold the full traces and, of u and v, the last time
level written and the w/Q field on every second point (every point in 2-D).
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, save  # noqa: E402


def smooth_vp_b(shape):
    """vp (km/s) and b = 1/rho on the unpadded `shape`, smooth and different along every axis."""
    axes = [np.linspace(0.0, 1.0, n) for n in shape]
    grids = np.meshgrid(*axes, indexing='ij')
    vp = 1.5 + 0.6 * grids[-1] + 0.2 * np.sin(2.5 * grids[0])
    rho = 1.0 + 0.8 * grids[-1] ** 2 + 0.3 * np.cos(3.0 * grids[0])
    if len(shape) == 3:
        vp = vp + 0.15 * np.cos(2.0 * grids[1])
        rho = rho + 0.25 * np.sin(3.5 * grids[1])
    return vp.astype(np.float32), (1.0 / rho).astype(np.float32)


def sa(name, shape, nbl, tn, so=8):
    from examples.seismic import Model, setup_geometry
    from examples.seismic.self_adjoint import SaIsoAcousticWaveSolver, setup_w_over_q
    vp, b = smooth_vp_b(shape)
    omega = 2.0 * np.pi * 0.010

    def init_damp(func, nbl):
        setup_w_over_q(func, omega, 0.1, 1000.0, nbl, sigma=0)
    model = Model(origin=(0.,) * len(shape), shape=shape, vp=vp, b=b, spacing=(10.,) * len(shape), nbl=nbl,
                  space_order=so, bcs=init_damp, dtype=np.float32)
    geometry = setup_geometry(model, tn)
    solver = SaIsoAcousticWaveSolver(model, geometry, space_order=so)
    rec, u, _ = solver.forward()
    srca, v, _ = solver.adjoint(rec)
    nt = geometry.nt
    step = 2 if len(shape) == 3 else 1
    sub = lambda a: np.array(a[(slice(None, None, step),) * len(shape)])
    save(name, so=so, shape=np.array(shape), nbl=nbl, tn=tn, dt=np.float32(solver.dt), nt=nt, step=step,
         src=np.array(geometry.src.data), rec=np.array(rec.data), srca=np.array(srca.data),
         u=sub(u.data[(nt - 1) % 3]), v=sub(v.data[0]), w=sub(model.damp.data))


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    sa('sa3d_so8', (24, 24, 24), nbl=10, tn=150.0)
    sa('sa2d_so8', (71, 61), nbl=10, tn=500.0)
