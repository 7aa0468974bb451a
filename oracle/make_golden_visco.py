"""Golden vectors of the reference's second-order SLS viscoacoustic modelling, `ViscoacousticWaveSolver.forward` and
`.adjoint` with `kernel='sls', time_order=2` (examples/seismic/viscoacoustic/operators.py:124-192, wavesolver.py),
run by the REFERENCE itself with its own CPU backend, like oracle/make_golden.py:

  PYTHONPATH=oracle/refshim:/root/reference DEVITO_LANGUAGE=openmp DEVITO_ARCH=gcc \
  DEVITO_SAFE_MATH=1 DEVITO_LOGGING=ERROR python oracle/make_golden_visco.py

vp, b and qp vary smoothly along every axis (`smooth_vp_b_qp`; tests rebuild them from the same formula), so that a
buoyancy sampled at the wrong offset or a quality factor taken at the wrong point changes the answer. The solver
switches the model's damping field to the "mask" profile (1 inside, below 1 in the absorbing layers); the fixtures
keep it. The adjoint is run on the forward's receiver data. To keep the fixtures small they hold the full traces and,
of p, r, pa and ra, the last time level written on every second point (every point in 2-D).
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, save  # noqa: E402
from make_golden_sa import smooth_vp_b  # noqa: E402


def smooth_vp_b_qp(shape):
    """vp (km/s), b = 1/rho and qp on the unpadded `shape`, smooth and different along every axis."""
    vp, b = smooth_vp_b(shape)
    axes = [np.linspace(0.0, 1.0, n) for n in shape]
    grids = np.meshgrid(*axes, indexing='ij')
    qp = 30.0 + 40.0 * grids[-1] + 10.0 * np.sin(2.0 * grids[0])
    if len(shape) == 3:
        qp = qp + 8.0 * np.cos(3.0 * grids[1])
    return vp, b, qp.astype(np.float32)


def visco(name, shape, nbl, tn, so=8):
    from examples.seismic import Model, setup_geometry
    from examples.seismic.viscoacoustic import ViscoacousticWaveSolver
    vp, b, qp = smooth_vp_b_qp(shape)
    model = Model(origin=(0.,) * len(shape), shape=shape, vp=vp, b=b, qp=qp, spacing=(10.,) * len(shape), nbl=nbl,
                  space_order=so, bcs="mask", dtype=np.float32)
    geometry = setup_geometry(model, tn)
    solver = ViscoacousticWaveSolver(model, geometry, space_order=so, kernel='sls', time_order=2)
    from devito import NODE, TimeFunction
    p, r, pa, ra = (TimeFunction(name=n, grid=model.grid, time_order=2, space_order=so, staggered=NODE)
                    for n in ('p', 'r', 'pa', 'r'))
    rec, _, _, _ = solver.forward(p=p, r=r)
    srca, _, _, _ = solver.adjoint(rec, pa=pa, r=ra)
    nt = geometry.nt
    step = 2 if len(shape) == 3 else 1
    sub = lambda a: np.array(a[(slice(None, None, step),) * len(shape)])
    last = (nt - 1) % 3
    save(name, so=so, shape=np.array(shape), nbl=nbl, tn=tn, dt=np.float32(solver.dt), nt=nt, step=step,
         f0=np.float32(geometry._f0), src=np.array(geometry.src.data), rec=np.array(rec.data),
         srca=np.array(srca.data), p=sub(p.data[last]), r=sub(r.data[last]), pa=sub(pa.data[0]),
         ra=sub(ra.data[0]), damp=sub(model.damp.data))


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    visco('visco3d_so8', (24, 24, 24), nbl=10, tn=150.0)
    visco('visco2d_so8', (71, 61), nbl=10, tn=500.0)
