#!/usr/bin/env python
"""Step and kernel times of the self-adjoint variable-density visco-acoustic update on one GPU (DESIGN §3.3h).

At so=8 on 1024^3 (944^3 + 40 absorbing cells per side) with array b, vp and w/Q, it calls `b2_sa_forward` on
device-resident arrays (u, b, vp, w/Q: 4.3 GB per level or field), forward and adjoint, with the TMA sweep
(`sa_tma<4>`, kernel=0) and the one-thread-per-point kernel (`k_sa_generic`, kernel=1) alternated in the same run,
STEPS steps each after a warm-up call. It prints one JSON line with, per kernel and direction:
- the per-step time of each direction (host clock around the blocking call / the number of steps);
- the mean device time per sweep launch (CUDA events around every launch, `b2_kernel_timing_ms`) and the variant that
  ran (`b2_last_sweep_kernel`);
- GB/s at 24 B per point (u[t], u[t-dir], b, C, w read, one level written) and GPts/s of the sweep;
- the card's name, power limit and the SM clock sampled while it ran.

    python profiles/sa_probe.py [--out FILE] [--steps STEPS] [--n N]
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
BYTES = 24.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--n', type=int, default=1024, help="grid points per axis, absorbing layers included")
    a = ap.parse_args()
    import torch
    from devito_b200 import _lib as L_
    from devito_b200.operator import sa_weights
    L = L_.lib()
    n, so, R = a.n, SO, SO // 2
    alloc = (n + 2 * so,) * 3
    dev = torch.device('cuda', 0)
    g = torch.Generator(device=dev).manual_seed(0)
    u = torch.zeros((3,) + alloc, dtype=torch.float32, device=dev)
    b = torch.rand(alloc, generator=g, device=dev) * 0.5 + 0.5
    vp = torch.rand(alloc, generator=g, device=dev) * 1.5 + 1.5
    w = torch.rand(alloc, generator=g, device=dev) * 0.05
    u[1, so + n // 2, so + n // 2, so + n // 2] = 1.0
    hold = []
    obj = lambda t: hold.append(L_.make_dataobj(dev_ptr=t.data_ptr(), shape=tuple(t.shape))) or hold[-1].ptr
    args = L_.SaArgs()
    args.ndim, args.space_order, args.radius = 3, so, R
    cw = (ctypes.c_float * R)(*sa_weights(R, 10.0))
    for d in range(3):
        args.c[d] = ctypes.cast(cw, ctypes.POINTER(ctypes.c_float))
    args.u, args.b, args.vp, args.damp = obj(u), obj(b), obj(vp), obj(w)
    args.b_value = args.vp_value = 1.0
    args.dt = 0.5
    args.x_m = args.y_m = args.z_m = 0
    args.x_M = args.y_M = args.z_M = n - 1
    args.deviceid = 0
    out = {'n': n, 'so': so, 'steps': a.steps, 'bytes_per_point': BYTES, 'gpu': gpu_identity(0)}
    pts = float(n) ** 3
    with ClockSampler(0) as clk:
        for name, adj, kernel in (('tma_forward', 0, 0), ('generic_forward', 0, 1), ('tma_adjoint', 1, 0),
                                  ('generic_adjoint', 1, 1)):
            args.adjoint = adj
            args.kernel = kernel
            args.time_m, args.time_M = 1, 3
            assert L.b2_sa_forward(ctypes.byref(args)) == 0, L.b2_last_error().decode()
            args.time_m, args.time_M = 1, a.steps
            L.b2_kernel_timing_enable(1)
            L.b2_kernel_timing_reset()
            t0 = time.perf_counter()
            rc = L.b2_sa_forward(ctypes.byref(args))
            wall = time.perf_counter() - t0
            nl = ctypes.c_int(0)
            ms = L.b2_kernel_timing_ms(ctypes.byref(nl))
            L.b2_kernel_timing_enable(0)
            assert rc == 0, L.b2_last_error().decode()
            out[name] = {'step_ms': wall / a.steps * 1e3, 'sweep_ms': ms, 'launches': nl.value,
                         'kernel': L.b2_last_sweep_kernel().decode(),
                         'sweep_gbs': BYTES * pts / (ms * 1e-3) / 1e9, 'sweep_gpts': pts / (ms * 1e-3) / 1e9}
    out['tma_over_generic'] = out['generic_forward']['sweep_ms'] / out['tma_forward']['sweep_ms']
    out['clock'] = clk.summary()
    out['hbm_datasheet_tbs'] = 3.35
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
