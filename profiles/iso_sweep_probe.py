#!/usr/bin/env python
"""Bandwidth ceiling of the isotropic so=8 TMA sweep's stream mix on one GPU (see iso_sweep_probe.cu).

Compiles iso_sweep_probe.cu with nvcc for sm_90a in a private temporary directory, runs it on GPU 0 and prints
one JSON line: the TMA copy (the sweep's producer/mbarrier structure, no arithmetic) for the sweep's boxes at
producer leads 1..8, the same copy without the u[t] halo and with 512-byte rows, the 16 x 128 sweep's boxes with and
without the A tile (`tiles_in` 2 / 1: the mix of the planes whose A the sweep pins), the two-level pass's boxes
(`two_level_16x64*`: k_iso_tma2's mix of one u[t] read, the level-1 tiles and two stores), and a plain read/write stream;
with the card's name, power limit and the SM clock sampled while it ran. The stream's rate is also written to
MEASURED_PEAKS.json (`hbm_gbs`) at the repository root, the peak `bench.py` states its roofline against.

    python profiles/iso_sweep_probe.py [--out FILE] [--no-peaks]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from bench import ClockSampler, gpu_identity  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    ap.add_argument('--no-peaks', action='store_true', help='do not write MEASURED_PEAKS.json')
    a = ap.parse_args()
    nvcc = os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'nvcc')
    if not os.path.exists(nvcc):
        nvcc = 'nvcc'
    with tempfile.TemporaryDirectory(prefix='iso_probe_') as tmp:
        exe = os.path.join(tmp, 'iso_sweep_probe')
        subprocess.run([nvcc, '-O3', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a',
                        '-I', os.path.join(ROOT, 'devito_b200', 'csrc'), os.path.join(HERE, 'iso_sweep_probe.cu'),
                        '-o', exe], check=True)
        with ClockSampler() as clk:
            out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout
    res = json.loads(out.strip().splitlines()[-1])
    res['gpu'] = gpu_identity()
    res['clocks'] = clk.summary()
    res['grid'] = '1024^3 interior points in 1040^3 arrays; u[t], u[t-1], A and u[t+1] separate arrays; 64 output ' \
                  'planes per CTA (+8 halo planes of u[t])'
    res['bytes_per_point'] = 16.0
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')
    if not a.no_peaks:
        with open(os.path.join(ROOT, 'MEASURED_PEAKS.json'), 'w') as f:
            json.dump({'hbm_gbs': res['stream']['gbs'], 'source': 'profiles/iso_sweep_probe.py plain read/write stream',
                       'gpu': res['gpu'], 'clocks': res['clocks']}, f)
            f.write('\n')


if __name__ == '__main__':
    main()
