"""Golden vectors of the reference's centred-TTI adjoint and gradient, `AnisotropicWaveSolver.adjoint(rec)` (operator
`AdjointTTI`) and `forward(save=True)` followed by `jacobian_adjoint(rec, u0, v0)` (operator `GradientTTI`,
examples/seismic/tti/operators.py `AdjointOperator` / `JacobianAdjOperator`), run by the REFERENCE itself with its
own CPU backend, like oracle/make_golden_tti_born.py:

  PYTHONPATH=oracle/refshim:/root/reference DEVITO_LANGUAGE=openmp DEVITO_ARCH=gcc \
  DEVITO_SAFE_MATH=1 DEVITO_LOGGING=ERROR python oracle/make_golden_tti_adj.py

The receiver data fed to both is the reference's own forward `rec`. The fixtures hold that input, the adjoint
source `srca`, the last level written of p and r (slot 0: the loop ends writing level time_m - 1 = 0) on every
second point of the domain along each axis, and the whole gradient `dm`.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, save  # noqa: E402


def tti_adj(name, so, n, nbl, tn, preset='constant-tti', **kw):
    from examples.seismic import demo_model, setup_geometry
    from examples.seismic.tti import AnisotropicWaveSolver
    model = demo_model(preset, spacing=(10., 10., 10.), shape=(n, n, n), nbl=nbl, space_order=so,
                       dtype=np.float32, **kw)
    geometry = setup_geometry(model, tn)
    solver = AnisotropicWaveSolver(model, geometry, space_order=so)
    rec, u0, v0, _ = solver.forward(save=True)
    rec_in = np.array(rec.data)
    srca, p, r, _ = solver.adjoint(rec)
    rec.data[:] = rec_in
    dm, _ = solver.jacobian_adjoint(rec, u0, v0)
    sub = lambda f: np.array(f.data[0][::2, ::2, ::2])
    save(name, so=so, n=n, nbl=nbl, tn=tn, dt=np.float32(model.critical_dt), nt=geometry.nt, rec=rec_in,
         srca=np.array(srca.data), p=sub(p), r=sub(r), dm=np.array(dm.data))


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    tti_adj('tti_adj3d_so8', so=8, n=20, nbl=8, tn=120.0)
    tti_adj('tti_adj3d_so4_layers', so=4, n=20, nbl=8, tn=120.0, preset='layers-tti', nlayers=3)
