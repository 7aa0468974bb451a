"""Inputs of the system-executor tests (tests/test_system_ref.py on the CPU, tests/test_system_matrix.py on the GPU):
synthetic tap-table systems on the anisotropic, non-cubic grid of tests/kernel_cases.py, and the fixtures of
oracle/make_golden_system.py.

A synthetic system starts from white noise in every time slot of every field, halo included, and white-noise
coefficient arrays. Its stages mix two-slot fields (updates, out_tshift 1) with one-slot scratch fields (out_tshift 0),
read every field at both time levels, reach +-halo along every axis, and include a stage of 1 tap, one of about 100
and one of B2_SYS_MAX_TAPS; one scratch stage is widened into the halo (ext). Injections go into 1, 2 and 3 fields
with the scalar, VP and M scales; interpolations use linear (r = 1) and sinc (r = 4) tables at tshift 0 and 1 and
sample a scratch field. The sparse points sit next to every face, outside it (their supports cross the guard), far
outside (no support cell at all) and twice in one cell (their deposits meet), and one table starts at p_m > 0.
"""
import numpy as np

import kernel_cases as KC
from oracle import oracle as O

FIXTURES = ['sys_el2d_so4', 'sys_el2d_so8', 'sys_ve2d_so4', 'sys_el3d_so4']
K = 4                                  # time steps per synthetic run
HALO = 4
MAX_FIELDS, MAX_COEFS, MAX_TAPS = 24, 48, 160      # B2_SYS_MAX_* of include/b200stencil.h

# name: (ndim, interior box, time_m, fields, coefficient arrays)
SYNTHETIC = {
    's3_full': (3, False, 1, 7, 5),
    's3_interior_t3': (3, True, 3, 7, 5),
    's2_full': (2, False, 1, 7, 5),
    's2_interior_t3': (2, True, 3, 7, 5),
    's3_max': (3, False, 1, MAX_FIELDS, MAX_COEFS),
}


def shape_of(nd):
    return KC.SHAPE[3 - nd:]


def spacing_of(nd):
    return KC.SPACING[3 - nd:]


def _coords(nd, rng):
    """Grid-unit positions: next to every face, just outside it, far outside, and a pair in one cell."""
    n = np.array(shape_of(nd))
    pts = []
    for d in range(nd):
        for where in (0.4, n[d] - 1 - 0.3, -0.6, n[d] - 1 + 0.45, -2.7, n[d] + 1.6):
            p = rng.uniform(5.0, n - 6.0)
            p[d] = where
            pts.append(p)
    far = rng.uniform(5.0, n - 6.0)
    far[0] = -14.0
    pts.append(far)
    c = np.floor(rng.uniform(5.0, n - 6.0))
    pts.append(c + 0.27)
    pts.append(c + 0.27)                                   # the same point twice
    pts.append(c + 0.81)                                   # and a third in the same cell
    return np.array(pts)


def sparse(nd, r, nt, rng, p_m=0):
    coords = _coords(nd, rng) * np.array(spacing_of(nd))
    gp, ws = O.tabulate(coords, (0.0,) * nd, spacing_of(nd), r, 'linear' if r == 1 else 'sinc', dtype=np.float32)
    data = rng.standard_normal((nt, len(coords))).astype(np.float32)
    return dict(data=data, gp=np.ascontiguousarray(gp, dtype=np.int32), w=[np.ascontiguousarray(w) for w in ws], r=r,
                p_m=p_m, p_M=len(coords) - 1)


def _taps(rng, nd, nf, T, ncoef, out, ots, n, ext=0, coefs=True):
    """n taps; the first 2 nd reach -+(halo - ext) along each axis; none reads shifted points of the written level."""
    taps = []
    reach = HALO - ext
    for i in range(n):
        if i < 2 * nd:
            off = [0] * nd
            off[i // 2] = reach if i % 2 else -reach
        else:
            off = list(rng.integers(-reach, reach + 1, nd))
        f = int(rng.integers(0, nf))
        ts = int(rng.integers(0, 2))
        if f == out and (ts - ots) % T[f] == 0:
            off = [0] * nd
        cf = int(rng.integers(-1, ncoef)) if coefs and ncoef else -1
        taps.append((f, ts, tuple(int(o) for o in off), float(rng.standard_normal() / np.sqrt(n)), cf))
    return taps


def synthetic(name):
    """(system, fields, coefs, lo, hi, time_m, time_M) of a synthetic case; fields and coefs are float32."""
    nd, interior, time_m, nf, nc = SYNTHETIC[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    shape = shape_of(nd)
    alloc = tuple(s + 2 * HALO for s in shape)
    T = [1 if i % 3 == 2 else 2 for i in range(nf)]         # fields 2, 5, 8 ... are one-slot scratch fields
    fields = [rng.standard_normal((t,) + alloc).astype(np.float32) for t in T]
    coefs = [rng.uniform(0.5, 1.5, shape).astype(np.float32) for _ in range(nc)]
    if interior:                                              # KC.SUBBOX, restricted to the last nd axes in 2-D
        lo, hi = KC.SUBBOX[0][3 - nd:], KC.SUBBOX[1][3 - nd:]
    else:
        lo, hi = (0,) * nd, tuple(s - 1 for s in shape)
    ntaps = [1, 100, MAX_TAPS, 13, 9]
    outs = [0, 2, 1, 3, 5]                                    # updates of 0, 1, 3 and the scratch fields 2, 5
    stages = []
    for out, n in zip(outs, ntaps):
        ots = 1 if T[out] == 2 else 0
        stages.append((out, ots, _taps(rng, nd, nf, T, nc, out, ots, n)))
    if name == 's3_max':
        # every coefficient array and every field in one stage of B2_SYS_MAX_TAPS taps
        taps = _taps(rng, nd, nf, T, nc, 4, 1, MAX_TAPS)
        taps = [(i % nf, ts, off, c, (i % (nc + 1)) - 1) if not (i % nf == 4 and (ts - 1) % 2 == 0)
                else (i % nf, ts, (0,) * nd, c, (i % (nc + 1)) - 1) for i, (f, ts, off, c, cf) in enumerate(taps)]
        stages.append((4, 1, taps))
    # a scratch stage widened by 2 into the halo (no coefficient arrays), sampled by a linear interpolation below
    stages.append((5, 0, _taps(rng, nd, nf, T, nc, 5, 0, 11, ext=2, coefs=False), 2))
    nt = time_m + K + 1
    lin, snc, lin2 = sparse(nd, 1, nt, rng), sparse(nd, 4, nt, rng), sparse(nd, 1, nt, rng, p_m=3)
    vp = rng.uniform(1.5, 2.5, alloc).astype(np.float32)
    m = (1.0 / (vp * vp)).astype(np.float32)
    inj = [dict(sp=lin, fields=[1], tshift=1, scale=0.7, kind=0, param=None),
           dict(sp=snc, fields=[0, 3], tshift=1, scale=0.3, kind=1, param=vp),
           dict(sp=lin2, fields=[0, 1, 3], tshift=0, scale=0.2, kind=2, param=m)]
    itp = [dict(sp=sparse(nd, 1, nt, rng), field=1, tshift=0),
           dict(sp=sparse(nd, 4, nt, rng, p_m=2), field=3, tshift=1),
           dict(sp=sparse(nd, 1, nt, rng), field=5, tshift=0),
           dict(sp=sparse(nd, 4, nt, rng), field=2, tshift=0)]
    system = dict(nd=nd, halo=HALO, T=T, stages=stages, injections=inj, interpolations=itp)
    return system, fields, coefs, lo, hi, time_m, time_m + K - 1


def outputs(system, F, traces):
    """Every field (all slots, halo included) and every sparse data array, in a fixed order."""
    sps = []
    for q in list(system['injections']) + list(system['interpolations']):
        if all(q['sp'] is not s for s in sps):
            sps.append(q['sp'])
    return [np.asarray(f) for f in F], [np.asarray(traces[id(s)]) for s in sps]
