#!/usr/bin/env python
"""Kernel and per-step times of the centred-TTI forward, adjoint and gradient on one GPU (DESIGN §3.3g).

For so=8 at 512^3 (480^3 + 16 absorbing cells per side), with scalar Thomsen parameters (`constant-tti`) and with
array-valued ones (`layers-tti`, 3 layers), it runs `AnisotropicWaveSolver.forward`, `adjoint` and, from
`forward(save=True)`, `jacobian_adjoint`, each once to warm up and once timed. It prints one JSON line with:
- the per-step time of each operator (CUDA events around the apply / the number of steps);
- the mean device time per launch of the mix (`k_tti_adj_mix`), the sweep (`k_tti_*` update kernels) and the
  imaging condition (`k_imaging`), from torch.profiler's CUDA activity over the timed apply, and the GB/s they
  achieve at the byte counts of DESIGN §3.3g (mix 16 / 24 B per allocated point, sweep 28 / 36 / 52 B and imaging
  40 B per point of the box);
- the card's name, power limit and the SM clock sampled while it ran.

The gradient needs u0 and v0 saved at every step: one time level at 512^3 with the so=8 halo is 528^3 * 4 B =
0.59 GB, so NT = 24 time levels of the two fields take 2 * 24 * 0.59 = 28 GB next to the ~15 GB of wavefields,
parameters, tables and scratch. Every operator runs the same NT - 2 = 22 steps.

    python profiles/tti_adjoint_probe.py [--out FILE] [--nt NT]
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from bench import ClockSampler, gpu_identity  # noqa: E402

N, NBL, SO = 480, 16, 8
SWEEP_BYTES = {'forward': {False: 28.0, True: 52.0}, 'adjoint': {False: 36.0, True: 52.0}}
MIX_BYTES = {False: 16.0, True: 24.0}
IMG_BYTES = 40.0


def _kernel_stats(prof):
    out = {}
    for ev in prof.key_averages():
        name = ev.key
        t = getattr(ev, 'device_time_total', None)
        if t is None:
            t = getattr(ev, 'cuda_time_total', 0.0)
        if not t or not ev.count:
            continue
        for tag, pat in (('mix', 'k_tti_adj_mix'), ('imaging', 'k_imaging'), ('sweep', 'k_tti_fused'),
                         ('sweep', 'k_tti_ws'), ('sweep', 'k_tti_update'), ('sweep_gz', 'k_tti_gz')):
            if pat in name:
                d = out.setdefault(tag, {'launches': 0, 'us_total': 0.0, 'kernels': []})
                d['launches'] += ev.count
                d['us_total'] += t
                d['kernels'].append(name[:90])
    for d in out.values():
        d['mean_ms'] = d['us_total'] / d['launches'] / 1e3
    return out


def _timed(fn, steps):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()                                           # warm-up: tables, scratch, tensor maps
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {'ms_per_step': ms / steps, 'kernels': _kernel_stats(prof)}


def run(preset, nt):
    import numpy as np
    from devito_b200.seismic import demo_model, setup_geometry
    from devito_b200.seismic.tti import AnisotropicWaveSolver
    kw = {'nlayers': 3} if preset == 'layers-tti' else {}
    arrays = preset == 'layers-tti'
    model = demo_model(preset, shape=(N,) * 3, spacing=(10.,) * 3, nbl=NBL, space_order=SO, **kw)
    dt = float(model.critical_dt)
    geometry = setup_geometry(model, dt * (nt - 1))
    solver = AnisotropicWaveSolver(model, geometry, space_order=SO)
    steps = geometry.nt - 2
    box = float((N + 2 * NBL) ** 3)
    alloc = float((N + 2 * NBL + 2 * SO) ** 3)
    res = {'preset': preset, 'nt': geometry.nt, 'steps': steps, 'points': box}
    rec = solver.forward()[0]
    rec_data = np.array(rec.data)
    res['forward'] = _timed(lambda: solver.forward(), steps)

    def adjoint():
        r = geometry.rec
        r.data[:] = rec_data
        solver.adjoint(r)
    res['adjoint'] = _timed(adjoint, steps)
    _, u0, v0, _ = solver.forward(save=True)

    def gradient():
        r = geometry.rec
        r.data[:] = rec_data
        solver.jacobian_adjoint(r, u0, v0)
    res['gradient'] = _timed(gradient, steps)
    for op in ('forward', 'adjoint', 'gradient'):
        ks = res[op]['kernels']
        sb = SWEEP_BYTES['forward' if op == 'forward' else 'adjoint'][arrays]
        for tag, nbytes, pts in (('sweep', sb, box), ('mix', MIX_BYTES[arrays], alloc), ('imaging', IMG_BYTES, box)):
            if tag in ks and 'sweep_gz' not in ks:
                ks[tag]['bytes_per_point'] = nbytes
                ks[tag]['gbs'] = nbytes * pts / (ks[tag]['mean_ms'] * 1e-3) / 1e9
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    ap.add_argument('--nt', type=int, default=24, help='time levels (the gradient saves this many of u0 and v0)')
    a = ap.parse_args()
    with ClockSampler() as clk:
        out = {'probe': 'tti_adjoint', 'so': SO, 'grid': f'{N + 2 * NBL}^3 (nbl={NBL} included)',
               'runs': [run(p, a.nt) for p in ('constant-tti', 'layers-tti')]}
    out['gpu'] = gpu_identity()
    out['clocks'] = clk.summary()
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
