"""Golden vectors of the staggered-grid system executor `b2_system_forward`: the reference's elastic and viscoelastic
forward runs (examples/seismic/elastic, examples/seismic/viscoelastic, `layers-*` presets), run by the REFERENCE itself
with its own CPU backend, like oracle/make_golden_tti_adj.py:

  PYTHONPATH=oracle/refshim:/root/reference:. DEVITO_LANGUAGE=openmp DEVITO_ARCH=gcc \
  DEVITO_SAFE_MATH=1 DEVITO_LOGGING=ERROR python oracle/make_golden_system.py

Each fixture `tests/golden/sys_*.npz` holds two things from ONE `solver.forward()`:

* the executor's inputs exactly as `devito_b200/refplugin.py` hands them to `LinearSystem.apply`: the stage and tap
  tables (flat, each tap's scalar coefficient already evaluated for dt and the spacings), the float32 coefficient
  arrays `_eval_coef` tabulated, the slot count of every field (the scratch field of `div(v)` has one), the sparse
  tables (base cells, weights, radius, point range, traces), the injections and interpolations, the time range and
  the iteration box;
* the reference's outputs of that run: every receiver trace (rec1 = tau_zz, rec2 = div(v)) and the last time level
  written of every field (domain only; every second point along each axis in 3-D).

So this script is also what checks the plugin's extraction (`_restate_system`, `_eval_coef`, `_apply_system`):
tests/test_system_ref.py runs the float64 tap-table interpreter (tests/system_ref.py) on the captured inputs and
compares with the captured outputs. Rerun it whenever refplugin changes.

The geometry adds one receiver just outside the top face of the grid (base cell -1 along the last axis): the support
of its linear interpolation reaches a halo cell, where the reference evaluates `div(v)` from the fields' halo.
"""
import ctypes
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, save  # noqa: E402


def _arr(obj, ndim, ctype=ctypes.c_float):
    """Copy of the array behind a `struct dataobj` holder (host data)."""
    o = obj.obj
    shape = tuple(int(o.size[i]) for i in range(ndim))
    return np.ctypeslib.as_array(ctypes.cast(o.data, ctypes.POINTER(ctype)), shape).copy()


def _capture(system, fields, coefs, lo, hi, time_m, time_M, cap):
    nd = system.ndim
    cap.update(nd=nd, halo=system.halo, lo=np.array(lo), hi=np.array(hi), time_m=time_m, time_M=time_M)
    cap['T'] = np.array([int(f.obj.size[0]) for f in fields])
    cap['alloc'] = np.array([int(fields[0].obj.size[d + 1]) for d in range(nd)])
    cap['coefs'] = np.stack([np.asarray(c, dtype=np.float32) for c in coefs]) if coefs else np.zeros((0,))
    cap['stage_out'] = np.array([s.out_field for s in system.stages])
    cap['stage_tshift'] = np.array([s.out_tshift for s in system.stages])
    cap['stage_ntaps'] = np.array([len(s.taps) for s in system.stages])
    cap['stage_ext'] = np.array([s.ext for s in system.stages])
    taps = [t for s in system.stages for t in s.taps]
    cap['tap_field'] = np.array([t.field for t in taps])
    cap['tap_tshift'] = np.array([t.tshift for t in taps])
    cap['tap_off'] = np.array([t.off for t in taps])
    cap['tap_coef'] = np.array([t.coef for t in taps], dtype=np.float64)
    cap['tap_cfield'] = np.array([t.cfield for t in taps])
    sparse = []

    def sid(sf):
        for i, s in enumerate(sparse):
            if s is sf:
                return i
        sparse.append(sf)
        i = len(sparse) - 1
        cap[f'sp{i}_data'] = _arr(sf.data, 2)
        cap[f'sp{i}_gp'] = _arr(sf.gp, 2, ctypes.c_int)
        for d, w in enumerate(sf.ws):
            cap[f'sp{i}_w{d}'] = _arr(w, 2)
        cap[f'sp{i}_r'], cap[f'sp{i}_pm'], cap[f'sp{i}_pM'] = sf.r, sf.p_m, sf.p_M
        return i
    inj = system.injections
    assert all(p is None for *_, p in inj), "position-dependent injection scales are not captured"
    cap['inj_sparse'] = np.array([sid(q[0]) for q in inj])
    cap['inj_fields'] = np.array([list(q[1]) + [-1] * (3 - len(q[1])) for q in inj])
    cap['inj_nfields'] = np.array([len(q[1]) for q in inj])
    cap['inj_tshift'] = np.array([q[2] for q in inj])
    cap['inj_scale'] = np.array([q[3] for q in inj], dtype=np.float64)
    cap['inj_kind'] = np.array([q[4] for q in inj])
    itp = system.interpolations
    cap['itp_sparse'] = np.array([sid(q[0]) for q in itp])
    cap['itp_field'] = np.array([q[1] for q in itp])
    cap['itp_tshift'] = np.array([q[2] for q in itp])
    cap['itp_name'] = np.array([q[0].name for q in itp])
    cap['nsparse'] = len(sparse)
    from devito_b200._lib import Profiler
    return Profiler(), 0.0


def system_case(name, solver_name, preset, shape, spacing, so, nbl, tn, **kw):
    from examples.seismic import demo_model, setup_geometry
    import devito_b200.refplugin as rp
    from devito_b200.system import LinearSystem
    rp.activate()
    if solver_name == 'elastic':
        from examples.seismic.elastic import ElasticWaveSolver as Solver
    else:
        from examples.seismic.viscoelastic import ViscoelasticWaveSolver as Solver
    model = demo_model(preset, shape=shape, spacing=spacing, nbl=nbl, space_order=so, dtype=np.float32, **kw)
    geometry = setup_geometry(model, tn)
    # the last receiver sits 0.4 cells outside the top face, 2 cells beside the source: base cell -1 along depth
    edge = np.array(geometry.src_positions[0], dtype=np.float64)
    edge[0] += 2 * spacing[0]
    edge[-1] = float(model.grid.origin[-1]) - 0.4 * spacing[-1]
    geometry.rec_positions[-1] = edge
    solver = Solver(model, geometry, space_order=so)
    cap = {}
    orig_apply, orig_sys, orig_res = LinearSystem.apply, rp.B200CudaOperator._apply_system, rp._coef_resident
    plan_names = []

    def run(self, plan, **kwargs):
        orig_sys(self, plan, **kwargs)                       # the plugin's inputs (LinearSystem.apply captures them)
        with rp.reference_cpu():
            summary = self.apply(**kwargs)                   # the reference's own CPU run on the same arguments
        nsub = 2 if plan.grid.dim == 3 else 1
        sl = (slice(None, None, nsub),) * plan.grid.dim
        last = (int(cap['time_M']) + 1) % 2
        cap['ref_fields'] = np.stack([np.array(kwargs[f.name].data[last][sl]) for f in plan.fields])
        cap['ref_sub'] = nsub
        for i, n in enumerate(cap['itp_name']):
            cap[f'ref_trace{i}'] = np.array(kwargs[str(n)].data)
        plan_names.extend(f.name for f in plan.fields)
        return summary
    LinearSystem.apply = lambda self, f, c, lo, hi, tm, tM, deviceid=0: _capture(self, f, c, lo, hi, tm, tM, cap)
    rp.B200CudaOperator._apply_system = run
    rp._coef_resident = lambda arr: arr                      # keep the tabulated arrays on the host
    try:
        solver.forward()
    finally:
        LinearSystem.apply, rp.B200CudaOperator._apply_system, rp._coef_resident = orig_apply, orig_sys, orig_res
    cap['field_names'] = np.array(plan_names)
    cap['dt'] = np.float32(solver.dt)
    cap['spacing'] = np.array(spacing)
    save(name, **cap)


if __name__ == '__main__':
    os.makedirs(OUT, exist_ok=True)
    system_case('sys_el2d_so4', 'elastic', 'layers-elastic', (31, 27), (10., 12.5), 4, 8, 150.0, nlayers=3)
    system_case('sys_el2d_so8', 'elastic', 'layers-elastic', (31, 27), (10., 12.5), 8, 8, 150.0, nlayers=3)
    system_case('sys_ve2d_so4', 'viscoelastic', 'layers-viscoelastic', (29, 33), (10., 12.5), 4, 8, 150.0)
    system_case('sys_el3d_so4', 'elastic', 'layers-elastic', (15, 13, 17), (10., 12.5, 8.), 4, 6, 90.0, nlayers=3)
