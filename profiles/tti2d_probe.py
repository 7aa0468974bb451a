#!/usr/bin/env python
"""Kernel and per-step times of the 2-D centred-TTI operators on one GPU (DESIGN §3.3i).

For so=8 on 16384 x 8192 points (16320 x 8128 + 32 absorbing cells per side; 0.54 GB per field level, well beyond
the 50 MB L2), with scalar Thomsen parameters (`constant-tti`) and with array-valued ones (`layers-tti`, 3 layers),
it runs `AnisotropicWaveSolver.forward` and `adjoint` with the single-pass sweep (kernel=2) and the two-pass sweep
(kernel=1) alternated in one run, then `jacobian` and, from `forward(save=True)`, `jacobian_adjoint` with the
single-pass sweep on wavefields and dm created once. Each apply runs once to warm up, once timed with CUDA events and once under torch.profiler. It
prints one JSON line with:
- the per-step time of each apply;
- the mean device time per launch of the sweep kernels (`k_tti2d`, `k_tti_gz` + `k_tti_update`) and the GB/s the
  single-pass sweep achieves at the byte counts of DESIGN §3.3i (forward 28 / 48 B per point, adjoint 36 / 48);
- the card's name, power limit and the SM clock sampled while it ran.

    python profiles/tti2d_probe.py [--out FILE] [--nt NT]
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from bench import ClockSampler, gpu_identity  # noqa: E402

SHAPE, NBL, SO = (16320, 8128), 32, 8
SWEEP_BYTES = {'forward': {False: 28.0, True: 48.0}, 'adjoint': {False: 36.0, True: 48.0}}


def _kernel_stats(prof):
    out = {}
    for ev in prof.key_averages():
        name = ev.key
        t = getattr(ev, 'device_time_total', None)
        if t is None:
            t = getattr(ev, 'cuda_time_total', 0.0)
        if not t or not ev.count:
            continue
        for tag, pat in (('sweep', 'k_tti2d'), ('sweep', 'k_tti_update'), ('sweep_gz', 'k_tti_gz'),
                         ('mix', 'k_tti_adj_mix'), ('born', 'k_tti_born_src'), ('imaging', 'k_imaging')):
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
    fn()
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
    from devito_b200 import Function, TimeFunction, _lib
    from devito_b200.seismic import demo_model, setup_geometry
    from devito_b200.seismic.tti import AnisotropicWaveSolver
    kw = {'nlayers': 3} if preset == 'layers-tti' else {}
    arrays = preset == 'layers-tti'
    model = demo_model(preset, shape=SHAPE, spacing=(10., 10.), nbl=NBL, space_order=SO, **kw)
    dt = float(model.critical_dt)
    geometry = setup_geometry(model, dt * (nt - 1))
    solver = AnisotropicWaveSolver(model, geometry, space_order=SO)
    steps = geometry.nt - 2
    box = float(np.prod([n + 2 * NBL for n in SHAPE]))
    res = {'preset': preset, 'nt': geometry.nt, 'steps': steps, 'points': box}
    rec_data = np.array(solver.forward(kernel=2)[0].data)
    name = lambda: _lib.lib().b2_last_sweep_kernel().decode()

    def adjoint(kernel):
        r = geometry.rec
        r.data[:] = rec_data
        solver.adjoint(r, kernel=kernel)
    for rnd in range(2):                     # the two sweeps alternated
        for kernel, tag in ((2, 'single_pass'), (1, 'two_pass')):
            for op, fn in (('forward', lambda: solver.forward(kernel=kernel)), ('adjoint', lambda: adjoint(kernel))):
                r = _timed(fn, steps)
                r['sweep_kernel'] = name()
                ks = r['kernels']
                if tag == 'single_pass' and 'sweep' in ks:
                    nb = SWEEP_BYTES[op][arrays]
                    ks['sweep']['bytes_per_point'] = nb
                    ks['sweep']['gbs'] = nb * box / (ks['sweep']['mean_ms'] * 1e-3) / 1e9
                res.setdefault(f'{op}_{tag}', []).append(r)
    # Born and gradient on fields created once (device-resident after the warm-up apply), so that the per-step times
    # hold no allocation or host-to-device copy of the four wavefields and dm
    mk = lambda n: TimeFunction(name=n, grid=model.grid, time_order=2, space_order=SO)
    b0, c0, bd, cd = mk('u0'), mk('v0'), mk('du'), mk('dv')
    dm = Function(name='dm', grid=model.grid, space_order=0)
    dm.data[:] = 1e-3
    res['born'] = _timed(lambda: solver.jacobian(dm, u0=b0, v0=c0, du=bd, dv=cd, kernel=2), steps)
    res['born']['sweep_kernel'] = name()
    _, u0, v0, _ = solver.forward(save=True, kernel=2)
    grad = Function(name='dm', grid=model.grid)

    def gradient():
        r = geometry.rec
        r.data[:] = rec_data
        solver.jacobian_adjoint(r, u0, v0, du=bd, dv=cd, dm=grad, kernel=2)
    res['gradient'] = _timed(gradient, steps)
    res['gradient']['sweep_kernel'] = name()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    ap.add_argument('--nt', type=int, default=12, help='time levels (the gradient saves this many of u0 and v0)')
    a = ap.parse_args()
    with ClockSampler() as clk:
        out = {'probe': 'tti2d', 'so': SO, 'grid': f'{SHAPE[0] + 2 * NBL} x {SHAPE[1] + 2 * NBL} (nbl={NBL} included)',
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
