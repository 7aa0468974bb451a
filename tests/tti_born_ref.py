"""Centred-TTI Born (linearised) modelling references for the tests -- TEST INFRASTRUCTURE ONLY.

- `oracle_tti_born_forward`: ctypes wrapper of tests/support/oracle_tti_born.c, the float32 C oracle of the
  reference's `BornTTI` operator (examples/seismic/tti/operators.py:532-586) in its generated operation order. The
  library is compiled on first use into a private per-user temporary directory (never into the tree).
- `tti_born_forward`: a float64 NumPy restatement on the update box, with separate weights per axis and the halo
  read as stored, built on the helpers of tests/ref64.py: (u, v) is stepped and driven by the sources, then (du, dv)
  gets the same centred-TTI update plus -dm u.dt2 / -dm v.dt2 over (m/dt^2 + damp/dt), with u / v after the
  injection; the receivers sample du + dv at time % T. `mut` selects one deliberate mistake: any of
  ref64.MUTATIONS that applies to this scheme, or one of MUTATIONS below.
"""
import ctypes
import os
import subprocess
import tempfile
from ctypes import POINTER, c_float, c_int

import numpy as np

import ref64
from ref64 import _at, _box, _bounds, _halo_zeroed, _lap, _shifted, _store, _Support, _transpose_xy, _unit, _weights
from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, 'support', 'oracle_tti_born.c')

MUTATIONS = {
    'born_before_inject': ref64.MUTATIONS['born_before_inject'],
    'born_dm_shift': ref64.MUTATIONS['born_dm_shift'],
    'tti_born_swap': "TTI Born: du driven by v.dt2 and dv by u.dt2",
}

_lib = None


def _build():
    d = os.path.join(tempfile.gettempdir(), f'devito-b200-tti-born-uid{os.getuid()}')
    os.makedirs(d, mode=0o700, exist_ok=True)
    st = os.stat(d)
    if st.st_uid != os.getuid() or st.st_mode & 0o077:
        raise RuntimeError(f"{d} is not a private directory of this user")
    path = os.path.join(d, 'liboracle_tti_born.so')
    deps = [SRC, os.path.join(os.path.dirname(HERE), 'oracle', 'oracle.c')]
    if not os.path.exists(path) or os.path.getmtime(path) < max(os.path.getmtime(p) for p in deps):
        env = dict(os.environ)
        env.pop('CC', None)
        tmp = path + f'.{os.getpid()}'
        # the flags of oracle/Makefile (strict IEEE, -O2)
        subprocess.run(['gcc', '-O2', '-std=c99', '-fPIC', '-shared', '-fopenmp', '-Wno-comment', '-o', tmp, SRC,
                        '-lm'], check=True, capture_output=True, env=env)
        os.replace(tmp, path)
    return path


def _load():
    global _lib
    if _lib is None:
        L = ctypes.CDLL(_build())
        fp, ip = POINTER(c_float), POINTER(c_int)
        L.oracle_tti_born_forward.argtypes = [fp, fp, fp, fp, c_int, ip, c_int, c_int, fp, fp, fp, fp, fp, fp, fp,
                                              c_float, c_float, c_float, c_float, c_float, c_float, ip, ip,
                                              c_int, c_int, POINTER(O.OSparse), POINTER(O.OSparse),
                                              fp, fp, fp, fp, fp, fp, ip, c_int]
        L.oracle_tti_born_forward.restype = c_int
        _lib = L
    return _lib


def oracle_tti_born_forward(u, v, du, dv, dm, so, w2, w1, dt, time_m, time_M, damp, vp, epsilon, delta, theta, phi,
                            src=None, rec=None, dmhalo=0, lo=None, hi=None, arrays=None):
    """float32 C oracle; u, v, du, dv and rec['data'] are updated in place. `arrays`: optional dict name ->
    allocated-layout float32 array for vp / epsilon / delta / theta / phi (else the scalars)."""
    L = _load()
    arrays = arrays or {}
    R = len(w2[0]) - 1
    alloc = np.array(u.shape[1:], dtype=np.int32)
    lo = np.array(lo if lo is not None else [0] * 3, dtype=np.int32)
    hi = np.array(hi if hi is not None else [s - 2 * so - 1 for s in u.shape[1:]], dtype=np.int32)
    w2a = [np.ascontiguousarray(x, dtype=np.float32) for x in w2]
    w1a = [np.ascontiguousarray(x, dtype=np.float32) for x in w1]
    keep = []
    s = O._sparse(src['data'], src['gp'], src['w'], src['r'], keep) if src else None
    r = O._sparse(rec['data'], rec['gp'], rec['w'], rec['r'], keep) if rec else None
    dm = np.ascontiguousarray(dm, dtype=np.float32)
    dmalloc = np.array(dm.shape, dtype=np.int32)
    arr = {n: np.ascontiguousarray(a, dtype=np.float32) for n, a in arrays.items()}
    fp = O._fp
    rc = L.oracle_tti_born_forward(fp(u), fp(v), fp(du), fp(dv), u.shape[0], O._ip(alloc), so, R, fp(w2a[0]),
                                   fp(w2a[1]), fp(w2a[2]), fp(w1a[0]), fp(w1a[1]), fp(w1a[2]), fp(damp), vp,
                                   epsilon, delta, theta, phi, dt, O._ip(lo), O._ip(hi), time_m, time_M,
                                   ctypes.byref(s) if s else None, ctypes.byref(r) if r else None,
                                   fp(arr.get('vp')), fp(arr.get('epsilon')), fp(arr.get('delta')),
                                   fp(arr.get('theta')), fp(arr.get('phi')), fp(dm), O._ip(dmalloc), dmhalo)
    assert rc == 0
    return u, v, du, dv


class _Tti:
    """The centred-TTI update of one field pair on the box: coefficients and the new box values."""

    def __init__(self, so, w2, w1, dt, damp, params, lo, hi, mut):
        self.so, self.dt, self.lo, self.hi, self.mut = so, dt, lo, hi, mut
        R = self.R = so // 2
        h = self.h = R // 2
        self.w2 = _weights(w2, mut)
        self.w1 = _weights(w1, mut)
        P = {k: _shifted(np.asarray(x, dtype=np.float64), mut) for k, x in params.items()}
        self.box = box = _box(lo, hi, so)
        # Gz is needed on the box grown by [-h, h-1]: the points q of the outer derivative
        self.elo = [x - h for x in lo]
        self.ehi = [x + h - 1 for x in hi]
        ebox = _box(self.elo, self.ehi, so)
        self.nb = [b - a + 1 for a, b in zip(lo, hi)]
        st, ct = np.sin(P['theta']), np.cos(P['theta'])
        sp, cp = np.sin(P['phi']), np.cos(P['phi'])
        Call = [st * cp, st * sp, ct * np.ones_like(sp)]
        self.CE = [_at(x, ebox) for x in Call]                       # C at the points of the grown box
        self.CB = [_at(x, box) for x in Call]                        # ... and at the output points
        self.e2 = 1 + 2 * _at(P['epsilon'], box)
        self.sd = np.sqrt(1 + 2 * _at(P['delta'], box))
        self.vp_all = P['vp']
        self.m = 1.0 / _at(self.vp_all * self.vp_all, box)
        self.d = _at(np.asarray(damp, dtype=np.float64), box) if damp is not None else 0.0
        self.den = self.m / dt ** 2 + self.d / dt

    def gzz(self, f):
        R, h, w1, so, mut = self.R, self.h, self.w1, self.so, self.mut
        elo, ehi, nb = self.elo, self.ehi, self.nb
        gz = 0.0
        for e in range(3):
            de = sum(w1[e][j] * f[_box(elo, ehi, so, _unit(e, j - h + 1))] for j in range(R))
            gz = gz + self.CE[e] * de
        out = 0.0
        for dd in range(3):
            cg = gz if mut == 'c_at_output' else self.CE[dd] * gz
            acc = 0.0
            for j in range(R):
                s = _unit(dd, j - h)
                sl = tuple(slice(h + s[a], h + s[a] + nb[a]) for a in range(3))   # box shifted, in grown-box indices
                acc = acc + w1[dd][j] * cg[sl]
            out = out + (self.CB[dd] * acc if mut == 'c_at_output' else acc)
        return out

    def new(self, u0, um, v0, vm):
        box, m, d, dt = self.box, self.m, self.d, self.dt
        lap = _lap(u0, self.w2, self.lo, self.hi, self.so)
        gu, gv = self.gzz(u0), self.gzz(v0)
        den = m / dt ** 2 + d / dt
        un = (self.e2 * (lap - gu) + self.sd * gv + m / dt ** 2 * (2 * u0[box] - um[box]) + d / dt * u0[box]) / den
        vn = (self.sd * (lap - gu) + gv + m / dt ** 2 * (2 * v0[box] - vm[box]) + d / dt * v0[box]) / den
        return un, vn


def tti_born_forward(u, v, du, dv, dm, dmh, so, w2, w1, dt, time_m, time_M, damp, params, lo=None, hi=None,
                     src=None, rec=None, mut=None):
    """Centred-TTI Born (linearised) modelling, time_m .. time_M (the reference's `BornTTI`): (u, v) is stepped and
    driven by `src`; (du, dv) gets the same update plus -dm u.dt2 / -dm v.dt2 over (m/dt^2 + damp/dt), with the
    u / v levels after the injection; `rec` samples du + dv at time % T. `dm` has halo `dmh`.
    Returns (u, v, du, dv, traces) in float64; the inputs are not modified."""
    u, v = np.array(u, dtype=np.float64), np.array(v, dtype=np.float64)
    du, dv = np.array(du, dtype=np.float64), np.array(dv, dtype=np.float64)
    T = u.shape[0]
    lo, hi = _bounds(u.shape[1:], so, lo, hi)
    S_ = _Tti(so, w2, w1, dt, damp, params, lo, hi, mut)
    box = S_.box
    dm = np.asarray(dm, dtype=np.float64)
    if mut == 'born_dm_shift':
        dm = np.roll(dm, 1, axis=0)
    dmb = dm[_box(lo, hi, dmh)]
    if mut == 'transpose_xy':
        for f in (u, v, du, dv):
            _transpose_xy(f)
    S = _Support(src, lo, hi, so) if src is not None else None
    R_ = _Support(rec, lo, hi, so) if rec is not None else None
    traces = np.array(rec['data'], dtype=np.float64) if rec is not None else None
    inj_scale = dt * dt * S_.vp_all * S_.vp_all
    for time in range(time_m, time_M + 1):
        t0, t1, t2 = time % T, (time + 1) % T, (time - 1) % T
        if mut == 'swap_levels':
            t0, t2 = t2, t0
        hz = (lambda f: _halo_zeroed(f, so)) if mut == 'halo_zero' else (lambda f: f)
        un, vn = S_.new(hz(u[t0]), u[t2], hz(v[t0]), v[t2])
        _store(u[t1], un, lo, hi, so, mut)
        _store(v[t1], vn, lo, hi, so, mut)
        before = (u[t1][box].copy(), v[t1][box].copy())
        if S is not None:
            S.inject([u[t1], v[t1]], time, inj_scale)
        u1, v1 = before if mut == 'born_before_inject' else (u[t1][box], v[t1][box])
        qu = -dmb * (u1 - 2 * u[t0][box] + u[t2][box]) / dt ** 2
        qv = -dmb * (v1 - 2 * v[t0][box] + v[t2][box]) / dt ** 2
        if mut == 'tti_born_swap':
            qu, qv = qv, qu
        dun, dvn = S_.new(hz(du[t0]), du[t2], hz(dv[t0]), dv[t2])
        _store(du[t1], dun + qu / S_.den, lo, hi, so, mut)
        _store(dv[t1], dvn + qv / S_.den, lo, hi, so, mut)
        if R_ is not None:
            R_.interpolate(traces, [du[time % T], dv[time % T]], time)
    return u, v, du, dv, traces
