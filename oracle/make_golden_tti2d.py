"""Golden vectors of the reference's 2-D centred-TTI operators, run by the REFERENCE itself with its own CPU backend,
like oracle/make_golden_tti_adj.py:

  PYTHONPATH=oracle/refshim:/root/reference DEVITO_LANGUAGE=openmp DEVITO_ARCH=gcc \
  DEVITO_SAFE_MATH=1 DEVITO_LOGGING=ERROR python oracle/make_golden_tti2d.py

For one model `AnisotropicWaveSolver` (examples/seismic/tti/wavesolver.py) runs `forward(save=True)` (`ForwardTTI`),
`adjoint(rec)` (`AdjointTTI`), `jacobian(dm)` (`BornTTI`) and `jacobian_adjoint(rec, u0, v0)` (`GradientTTI`), all
with `Gzz_centered_2d`. The fixtures hold the forward receivers and last levels of u, v, the adjoint source and the
last levels of p, r, the Born receivers and last levels of du, dv, and the gradient, all on the whole grid (2-D
fixtures are small). The `varying` model has vp, epsilon, delta and theta varying along both axes (the `layers-tti`
preset varies along z only, so it cannot show where theta is sampled along x); its parameter arrays are stored.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, save  # noqa: E402


def dm_blob(shape):
    """float32 Gaussian blob of amplitude 0.05 and width 4 cells, 2 cells below the centre."""
    X, Z = np.meshgrid(*[np.arange(m, dtype=np.float64) for m in shape], indexing='ij')
    cx, cz = (shape[0] - 1) / 2.0, (shape[1] - 1) / 2.0
    return (0.05 * np.exp(-((X - cx) ** 2 + (Z - cz - 2) ** 2) / (2 * 4.0 ** 2))).astype(np.float32)


def varying_parameters(shape):
    gx, gz = np.meshgrid(*[np.linspace(0., 1., m, dtype=np.float32) for m in shape], indexing='ij')
    return dict(vp=(1.5 + 0.7 * gx + 0.9 * gz).astype(np.float32),
                epsilon=(0.25 * gx * gz + 0.05).astype(np.float32),
                delta=(0.12 * gx + 0.06 * gz + 0.02).astype(np.float32),
                theta=(0.2 + 0.9 * gx * gz + 0.3 * gx - 0.2 * gz).astype(np.float32))


def tti2d(name, so, shape, nbl, tn, preset=None, **kw):
    from examples.seismic import SeismicModel, demo_model, setup_geometry
    from examples.seismic.tti import AnisotropicWaveSolver
    spacing = (10., 10.)
    extra = {}
    if preset is None:
        par = varying_parameters(shape)
        model = SeismicModel(space_order=so, origin=(0., 0.), shape=shape, dtype=np.float32, spacing=spacing,
                             nbl=nbl, bcs="damp", **par)
        extra = {'par_' + k: v for k, v in par.items()}
    else:
        model = demo_model(preset, spacing=spacing, shape=shape, nbl=nbl, space_order=so, dtype=np.float32, **kw)
    geometry = setup_geometry(model, tn)
    solver = AnisotropicWaveSolver(model, geometry, space_order=so)
    nt = geometry.nt
    last = (nt - 1) % 3
    rec, u0, v0, _ = solver.forward(save=True)
    rec_f = np.array(rec.data)
    u_last, v_last = np.array(u0.data[nt - 1]), np.array(v0.data[nt - 1])
    srca, p, r, _ = solver.adjoint(rec)
    srca_a, p0, r0 = np.array(srca.data), np.array(p.data[0]), np.array(r.data[0])
    rec.data[:] = rec_f
    g, _ = solver.jacobian_adjoint(rec, u0, v0)
    grad = np.array(g.data)
    dm = dm_blob(model.grid.shape)
    rb, _, _, du, dv, _ = solver.jacobian(dm)
    save(name, so=so, shape=np.array(shape), nbl=nbl, tn=tn, dt=np.float32(model.critical_dt), nt=nt,
         src_coords=np.array(geometry.src.coordinates.data), rec_coords=np.array(geometry.rec.coordinates.data),
         rec=rec_f, u_last=u_last, v_last=v_last, srca=srca_a, p=p0, r=r0, grad=grad, dm=dm,
         born_rec=np.array(rb.data), du=np.array(du.data[last]), dv=np.array(dv.data[last]), **extra)


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    tti2d('tti2d_so8', so=8, shape=(40, 44), nbl=10, tn=150.0, preset='constant-tti')
    tti2d('tti2d_so4_layers', so=4, shape=(40, 44), nbl=10, tn=150.0, preset='layers-tti', nlayers=3)
    tti2d('tti2d_so8_varying', so=8, shape=(36, 40), nbl=10, tn=150.0)
