#!/usr/bin/env python
"""Step and kernel times of the second-order SLS viscoacoustic update on one GPU (DESIGN §3.3k).

At so=8 on 1024^3 (absorbing layers included) with array vp, b, qp and the mask damping, it calls `b2_visco_forward`
on device-resident arrays (p, r: three levels each; vp, b, qp, damp: 4.5 GB per level or field), forward and
adjoint, with the TMA sweep (`visco_tma<4>`, kernel=0) and the one-thread-per-point kernel (`k_visco_generic`,
kernel=1) alternated in the same run, STEPS steps each after a warm-up call. The library adds five tables and, on
the adjoint, s: 72 GB in all with the arrays above, within the 80 GB of an H100. It prints one JSON line with, per
kernel and direction:
- the per-step time (host clock around the blocking call / the number of steps);
- the mean device time per launch of the stencil kernels (CUDA events around every launch, `b2_kernel_timing_ms`;
  on the adjoint the mix `k_visco_adj_mix` and the sweep are both timed launches) and the variant that ran
  (`b2_last_sweep_kernel`);
- GB/s per step at the algorithmic 44 B per point forward and 64 B per point adjoint, and GPts/s;
- the card's name, power limit and the SM clock sampled while it ran.

    python profiles/visco_probe.py [--out FILE] [--steps STEPS] [--n N]
"""
import argparse
import ctypes
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from bench import ClockSampler, gpu_identity  # noqa: E402

SO = 8
BYTES = {0: 44.0, 1: 64.0}         # forward, adjoint (DESIGN §3.3k)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--n', type=int, default=1024, help="grid points per axis, absorbing layers included")
    a = ap.parse_args()
    import torch
    from devito_b200 import _lib as L_
    from devito_b200.operator import sa_weights
    from devito_b200.seismic import damp_profile
    L = L_.lib()
    n, so, R = a.n, SO, SO // 2
    alloc = (n + 2 * so,) * 3
    dev = torch.device('cuda', 0)
    g = torch.Generator(device=dev).manual_seed(0)
    p = torch.zeros((3,) + alloc, dtype=torch.float32, device=dev)
    r = torch.zeros((3,) + alloc, dtype=torch.float32, device=dev)
    b = torch.rand(alloc, generator=g, device=dev) * 0.5 + 0.5
    vp = torch.rand(alloc, generator=g, device=dev) * 1.5 + 1.5
    qp = torch.rand(alloc, generator=g, device=dev) * 90.0 + 10.0
    damp = torch.ones(alloc, dtype=torch.float32, device=dev)
    nbl = 40
    damp[so:-so, so:-so, so:-so] = torch.from_numpy(damp_profile((n,) * 3, [(nbl, nbl)] * 3, (10.0,) * 3,
                                                                 'mask')).to(dev)
    p[1, so + n // 2, so + n // 2, so + n // 2] = 1.0
    torch.cuda.empty_cache()      # the staging copy of damp goes back to the device before the library's scratch
    hold = []
    obj = lambda t: hold.append(L_.make_dataobj(dev_ptr=t.data_ptr(), shape=tuple(t.shape))) or hold[-1].ptr
    args = L_.ViscoArgs()
    args.ndim, args.space_order, args.radius = 3, so, R
    cw = (ctypes.c_float * R)(*sa_weights(R, 10.0))
    for d in range(3):
        args.c[d] = ctypes.cast(cw, ctypes.POINTER(ctypes.c_float))
    args.u, args.r, args.b, args.vp, args.qp, args.damp = obj(p), obj(r), obj(b), obj(vp), obj(qp), obj(damp)
    args.b_value = args.vp_value = args.qp_value = 1.0
    args.f0 = 0.010
    args.dt = 0.5
    args.x_m = args.y_m = args.z_m = 0
    args.x_M = args.y_M = args.z_M = n - 1
    args.deviceid = 0
    out = {'n': n, 'so': so, 'steps': a.steps, 'bytes_per_point': {'forward': BYTES[0], 'adjoint': BYTES[1]},
           'gpu': gpu_identity(0)}
    pts = float(n) ** 3
    with ClockSampler(0) as clk:
        for name, adj, kernel in (('tma_forward', 0, 0), ('generic_forward', 0, 1), ('tma_adjoint', 1, 0),
                                  ('generic_adjoint', 1, 1)):
            args.adjoint = adj
            args.kernel = kernel
            args.time_m, args.time_M = 1, 3
            assert L.b2_visco_forward(ctypes.byref(args)) == 0, L.b2_last_error().decode()
            args.time_m, args.time_M = 1, a.steps
            L.b2_kernel_timing_enable(1)
            L.b2_kernel_timing_reset()
            t0 = time.perf_counter()
            rc = L.b2_visco_forward(ctypes.byref(args))
            wall = time.perf_counter() - t0
            nl = ctypes.c_int(0)
            ms = L.b2_kernel_timing_ms(ctypes.byref(nl))
            L.b2_kernel_timing_enable(0)
            assert rc == 0, L.b2_last_error().decode()
            # b2_kernel_timing_ms gives the mean over the timed launches (one sweep per step forward, the mix and
            # the sweep per step on the adjoint)
            per_step = ms * nl.value / a.steps
            out[name] = {'step_ms': wall / a.steps * 1e3, 'kernel_ms_per_step': per_step, 'launches': nl.value,
                         'kernel_ms_per_launch': ms,
                         'kernel': L.b2_last_sweep_kernel().decode(),
                         'gbs': BYTES[adj] * pts / (per_step * 1e-3) / 1e9, 'gpts': pts / (per_step * 1e-3) / 1e9}
    out['tma_over_generic_forward'] = out['generic_forward']['kernel_ms_per_step'] / \
        out['tma_forward']['kernel_ms_per_step']
    out['tma_over_generic_adjoint'] = out['generic_adjoint']['kernel_ms_per_step'] / \
        out['tma_adjoint']['kernel_ms_per_step']
    out['clock'] = clk.summary()
    out['hbm_datasheet_tbs'] = 3.35
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
