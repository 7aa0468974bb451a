"""Propagation cases shared by tests/dist_worker.py (decomposed over N ranks) and tests/test_distributed.py
(the same case on one GPU): each returns {name: array}; arrays named in SLABBED are split along their
x axis under decomposition and re-assembled by the test."""
import numpy as np

SO, NBL, TN = 8, 10, 150.0
# name -> axis of the array that is decomposed (None: replicated / merged, e.g. receiver traces)
AXIS = {'u': 1, 'v': 1, 'U': 1, 'usave': 1, 'grad': 0, 'rec': None}


def shape_for(nranks):
    return (24 * nranks - 4, 28, 28)                     # 24 owned planes per rank incl. absorbing layers


def run_case(kind, nranks, topology=None):
    import devito_b200 as dv
    from devito_b200.seismic import (demo_model, setup_geometry, AcousticWaveSolver, AnisotropicWaveSolver)
    n = shape_for(nranks)
    kw = dict(spacing=(10., 10., 10.), shape=n, nbl=NBL, space_order=SO)
    if topology is not None:
        kw['topology'] = topology
    if kind in ('iso', 'tti'):
        preset = 'constant-isotropic' if kind == 'iso' else 'constant-tti'
        cls = AcousticWaveSolver if kind == 'iso' else AnisotropicWaveSolver
        model = demo_model(preset, **kw)
        out = cls(model, setup_geometry(model, TN), space_order=SO).forward()
        res = {'rec': out[0].data, 'u': out[1].data}
        if kind == 'tti':
            res['v'] = out[2].data
        return res, model
    if kind == 'ttiarr':                                   # array-valued vp / eps / delta / theta / phi, varying along every axis
        from devito_b200.seismic import SeismicModel
        gx, gy, gz = np.meshgrid(*[np.linspace(0., 1., m, dtype=np.float32) for m in n], indexing='ij')
        model = SeismicModel(space_order=SO, vp=(1.5 + 0.6 * gx + 0.5 * gy + 0.9 * gz).astype(np.float32),
                             origin=(0., 0., 0.), shape=n, dtype=np.float32, spacing=(10., 10., 10.), nbl=NBL,
                             epsilon=(0.25 * gx * gz + 0.05).astype(np.float32), delta=(0.12 * gy + 0.02).astype(np.float32),
                             theta=(0.2 + 0.9 * gx * gy + 0.3 * gz).astype(np.float32),
                             phi=(0.1 + 0.8 * gy * gz - 0.4 * gx).astype(np.float32), bcs="damp",
                             **({'topology': topology} if topology is not None else {}))
        out = AnisotropicWaveSolver(model, setup_geometry(model, TN), space_order=SO).forward()
        return {'rec': out[0].data, 'u': out[1].data, 'v': out[2].data}, model
    if kind == 'iso12':                                    # so=12: the one-row sweep kernel with the fused halo step
        kw12 = dict(kw, space_order=12, nbl=14)
        model = demo_model('constant-isotropic', **kw12)
        rec, u, _ = AcousticWaveSolver(model, setup_geometry(model, TN), space_order=12).forward()
        return {'rec': rec.data, 'u': u.data}, model
    if kind == 'stream':                                   # host-staged apply: streamed loop, skewed along y when decomposed
        import os
        model = demo_model('constant-isotropic', **kw)
        solver = AcousticWaveSolver(model, setup_geometry(model, TN, interpolation='sinc'), space_order=SO)
        if topology is not None:
            os.environ['B2_STREAM'], os.environ['B2_STREAM_W'] = '2', '16'
            rec, u, _ = solver.forward(resident=False)
            import ctypes
            from devito_b200 import _lib
            prof = (ctypes.c_double * 5)()
            _lib.lib().b2_last_call_profile(prof)
            assert prof[4] == 1.0, "the decomposed host-staged apply did not stream"
        else:
            rec, u, _ = solver.forward()
        return {'rec': rec.data, 'u': u.data}, model
    if kind == 'fs':                                       # free surface + layered velocity
        model = demo_model('layers-isotropic', fs=True, nlayers=3, **kw)
        rec, u, _ = AcousticWaveSolver(model, setup_geometry(model, TN), space_order=SO).forward()
        return {'rec': rec.data, 'u': u.data}, model
    if kind == 'ot4':                                      # 4th order in time: the halo is 2*radius planes wide
        model = demo_model('constant-isotropic', **kw)
        rec, u, _ = AcousticWaveSolver(model, setup_geometry(model, TN), space_order=SO, kernel='OT4').forward()
        return {'rec': rec.data, 'u': u.data}, model
    if kind == 'born':                                     # two wavefields stepped together
        model = demo_model('layers-isotropic', nlayers=2, **kw)
        solver = AcousticWaveSolver(model, setup_geometry(model, TN), space_order=SO)
        gshape = tuple(s + 2 * NBL for s in n)
        rng = np.random.default_rng(11)
        dm_glb = (1e-2 * rng.standard_normal(gshape)).astype(np.float32)
        dm = dv.Function(name='dm', grid=model.grid, space_order=0)
        lo, hi = model.grid.distributor.x_range if model.grid.distributor.is_parallel else (0, gshape[0])
        dm.data[:] = dm_glb[lo:hi]
        rec, u, U, _ = solver.jacobian(dm)
        return {'rec': rec.data, 'u': u.data, 'U': U.data}, model
    if kind == 'grad':                                     # saved forward field + adjoint run + imaging condition
        model = demo_model('constant-isotropic', **kw)
        solver = AcousticWaveSolver(model, setup_geometry(model, TN), space_order=SO)
        rec, u, _ = solver.forward(save=True)
        grad, _ = solver.jacobian_adjoint(rec, u)
        return {'rec': rec.data, 'grad': grad.data}, model
    if kind == 'snap':                                     # time-subsampled snapshots
        from devito_b200 import ConditionalDimension, Eq, Operator, TimeFunction, solve
        model = demo_model('constant-isotropic', **kw)
        geometry = setup_geometry(model, TN)
        factor = 4
        nsnaps = (geometry.nt + factor - 1) // factor
        t_sub = ConditionalDimension('t_sub', parent=model.grid.time_dim, factor=factor)
        usave = TimeFunction(name='usave', grid=model.grid, time_order=2, space_order=2, save=nsnaps, time_dim=t_sub)
        u = TimeFunction(name='u', grid=model.grid, time_order=2, space_order=SO)
        pde = model.m * u.dt2 - u.laplace + model.damp * u.dt
        src, rec = geometry.src, geometry.rec
        dt = model.critical_dt
        op = Operator([Eq(u.forward, solve(pde, u.forward))] + src.inject(field=u.forward, expr=src * dt ** 2 / model.m) +
                      [Eq(usave, u)] + rec.interpolate(expr=u), subs=model.spacing_map)
        op(time=geometry.nt - 2, dt=dt)
        return {'rec': rec.data, 'u': u.data, 'usave': usave.data}, model
    raise ValueError(kind)


TOL = {'ttiarr': 1e-4, 'iso12': 1e-5, 'stream': 1e-5, 'iso': 1e-5, 'tti': 1e-4, 'fs': 1e-5, 'ot4': 1e-5, 'born': 1e-4, 'grad': 1e-4, 'snap': 1e-5}
