#!/usr/bin/env python
"""Whole-gradient times of the acoustic gradient with and without binomial checkpointing on one GPU.

At so=8, 512^3 allocated points (432^3 + 40 absorbing cells per side; 528^3 slots of 0.59 GB), constant vp, NT = 48
time levels (l = NT - 2 = 46 adjoint steps; s = l checkpoints take 2 * 46 * 0.59 = 54 GB, the saved path 48 slots):
- the saved path: `forward(save=True)` (NT slots of u) then `jacobian_adjoint(rec, u)`;
- the checkpointed path `jacobian_adjoint(rec, checkpointing=True, n_checkpoints=s)` for s in {l, 32, 8}, with the
  forward steps its schedule runs next to the optimum r*l - beta(s+1, r-1) (they are equal by construction: the
  schedule's advances are counted);
- the mean device time per launch of the forward sweep and of the adjoint sweep (CUDA events around every stencil
  launch, b2_kernel_timing_*), over one forward and one adjoint apply of the same l steps.
Then one checkpointed gradient at 1024^3 allocated points (944^3 + 40 per side), NT = 256, with the default number
of checkpoints; the saved path would need 256 slots of 4.5 GB there. Every timed call runs once to warm up first
(except the 1024^3 one). Times are host clock around calls that end in a device synchronise. The card's name and
power limit are read in the same run. Prints and writes one JSON document.

    python profiles/gradient_checkpoint_probe.py [--out FILE] [--nt NT] [--skip-large]
"""
import argparse
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from bench import gpu_identity  # noqa: E402

SO, NBL = 8, 40


def _solver(n_alloc, nt):
    from devito_b200.seismic import demo_model, setup_geometry, AcousticWaveSolver
    n = n_alloc - 2 * NBL
    model = demo_model('constant-isotropic', spacing=(10., 10., 10.), shape=(n, n, n), nbl=NBL, space_order=SO)
    dt = float(model.critical_dt)
    geometry = setup_geometry(model, dt * (nt - 1))
    return geometry, AcousticWaveSolver(model, geometry, space_order=SO)


def _clock(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def _forward_steps(sched):
    return sum(a[2] - a[1] for a in sched if a[0] == 'advance')


def _kernel_ms(fn, L):
    import ctypes
    L.b2_kernel_timing_reset()
    L.b2_kernel_timing_enable(1)
    try:
        fn()
    finally:
        L.b2_kernel_timing_enable(0)
    n = ctypes.c_int(0)
    ms = L.b2_kernel_timing_ms(ctypes.byref(n))
    return {'mean_ms_per_launch': ms, 'launches': n.value, 'kernel': L.b2_last_sweep_kernel().decode()}


def probe_512(nt):
    import numpy as np
    from devito_b200 import _lib
    from devito_b200.revolve import optimal_forward_steps, schedule
    L = _lib.lib()
    geometry, solver = _solver(512, nt)
    rec, _, _ = solver.forward()
    nsteps = rec.data.shape[0] - 2
    out = {'alloc_points': 512 ** 3, 'slot_bytes': 528 ** 3 * 4, 'nt': int(rec.data.shape[0]), 'l': nsteps}

    def saved():
        r, u, _ = solver.forward(save=True)
        g, _ = solver.jacobian_adjoint(rec, u)
        del u
        return g
    saved()
    t, g_saved = _clock(saved)
    g_saved = np.array(g_saved.data)
    out['saved'] = {'whole_gradient_s': t, 'forward_steps': nsteps}     # forward(save=True) runs time 1 .. nt - 2
    import torch
    torch.cuda.empty_cache()
    runs = []
    for s in (nsteps, 32, 8):
        steps = _forward_steps(schedule(nsteps, s))
        solver.jacobian_adjoint(rec, checkpointing=True, n_checkpoints=s)
        t, (g, _) = _clock(lambda: solver.jacobian_adjoint(rec, checkpointing=True, n_checkpoints=s))
        runs.append({'n_checkpoints': s, 'whole_gradient_s': t, 'forward_steps': steps,
                     'forward_steps_optimum': optimal_forward_steps(nsteps, s), 'adjoint_steps': nsteps,
                     'sweeps': L.b2_last_sweep_kernel().decode(),
                     'bitwise_equal_to_saved': bool(np.array_equal(np.asarray(g.data), g_saved))})
    out['checkpointed'] = runs
    out['forward_sweep'] = _kernel_ms(lambda: solver.forward(), L)
    out['adjoint_sweep'] = _kernel_ms(lambda: solver.adjoint(rec), L)
    return out


def probe_1024(nt):
    from devito_b200 import _lib
    from devito_b200.revolve import optimal_forward_steps
    L = _lib.lib()
    geometry, solver = _solver(1024, nt)
    rec = geometry.rec
    rec.data[:] = 0.
    rec.data[nt // 2:, :] = 1e-3                # adjoint source: something to propagate
    nsteps = rec.data.shape[0] - 2
    c = solver._revolve_setup(rec)              # the default number of checkpoints, once u, v and grad are resident
    s = c.n_checkpoints
    steps = _forward_steps(c.schedule)
    t, (g, summary) = _clock(lambda: solver._revolve_run(c))
    import numpy as np
    ok = bool(np.isfinite(np.asarray(g.data)).all()) and bool(np.abs(np.asarray(g.data)).max() > 0)
    return {'alloc_points': 1024 ** 3, 'slot_bytes': 1040 ** 3 * 4, 'nt': int(rec.data.shape[0]), 'l': nsteps,
            'completed': ok, 'n_checkpoints_default': s, 'whole_gradient_s': t,
            'loop_s': summary['section0'].time, 'forward_steps': steps,
            'forward_steps_optimum': optimal_forward_steps(nsteps, s), 'sweeps': L.b2_last_sweep_kernel().decode(),
            'saved_path': 'not run: %d slots of %.1f GB' % (nt, 1040 ** 3 * 4 / 1e9)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=os.path.join(HERE, 'h100_gradient_checkpoint_probe.json'))
    ap.add_argument('--nt', type=int, default=48)
    ap.add_argument('--skip-large', action='store_true')
    a = ap.parse_args()
    doc = {'gpu': gpu_identity(0), 'so': SO}
    doc['512'] = probe_512(a.nt)
    doc['1024'] = 'not measured' if a.skip_large else probe_1024(256)
    doc['gpu_after'] = gpu_identity(0)
    s = json.dumps(doc, indent=1)
    print(s)
    with open(a.out, 'w') as f:
        f.write(s + '\n')


if __name__ == '__main__':
    main()
