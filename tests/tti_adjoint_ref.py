"""float64 restatement of the centred-TTI adjoint (`AdjointTTI`) and of its imaging condition (`GradientTTI`),
built on the helpers of tests/ref64.py (reference: examples/seismic/tti/operators.py `kernel_centered(...,
forward=False)`, `AdjointOperator`, `JacobianAdjOperator`):

  a = e2 p + sd r,  b = sd p + r           e2 = 1+2 eps, sd = sqrt(1+2 delta) at every point (halo included)
  H0 = lap(a) - Gzz(a),  Hz = Gzz(b)
  p[t-1] = (m/dt^2 (2 p[t] - p[t+1]) + damp/dt p[t] + H0) / (m/dt^2 + damp/dt),  r[t-1] likewise with Hz
  p[t-1], r[t-1] += rec[time] dt^2 / m;   srca[time] = p[t] + r[t]
  grad -= usave[time] (p[t+1] - 2 p[t] + p[t-1]) / dt^2 + vsave[time] (r[t+1] - 2 r[t] + r[t-1]) / dt^2

The mutations are the kernel bugs this path could hide. They live here rather than in ref64.MUTATIONS so that the
parametrisations over that table stay as they are.
"""
import numpy as np

import ref64 as R64
from ref64 import _at, _box, _bounds, _lap, _store, _Support, _unit, _weights

MUTATIONS = {
    'fwd_mix': "the forward combination run backward: H0 = e2 Gh(p) + sd Gzz(r), Hz = sd Gh(p) + Gzz(r)",
    'mix_at_output': "e2 and sd of the mixes taken at the output point instead of at every tap point",
    'mix_swap': "the two mixes exchanged between the equations",
    'inject_level': "the receivers injected into level t instead of the level just written",
    'img_swap': "imaging condition: usave and vsave exchanged",
    'img_before_inject': "imaging condition: p.dt2 / r.dt2 taken before the injection",
}


def _gzz_factory(so, w1, params, lo, hi):
    """Gzz on the box (ref64.tti_forward's restatement): rotation factors at the Gz points of the grown box."""
    R = so // 2
    h = R // 2
    elo = [x - h for x in lo]
    ehi = [x + h - 1 for x in hi]
    ebox = _box(elo, ehi, so)
    nb = [b - a + 1 for a, b in zip(lo, hi)]
    th, ph = np.asarray(params['theta'], np.float64), np.asarray(params['phi'], np.float64)
    st, ct, sp, cp = np.sin(th), np.cos(th), np.sin(ph), np.cos(ph)
    CE = [_at(x, ebox) for x in (st * cp, st * sp, ct * np.ones_like(sp))]

    def gzz(f):
        gz = 0.0
        for e in range(3):
            gz = gz + CE[e] * sum(w1[e][j] * f[_box(elo, ehi, so, _unit(e, j - h + 1))] for j in range(R))
        out = 0.0
        for d in range(3):
            cg = CE[d] * gz
            for j in range(R):
                s = _unit(d, j - h)
                out = out + w1[d][j] * cg[tuple(slice(h + s[a], h + s[a] + nb[a]) for a in range(3))]
        return out
    return gzz


def tti_adjoint(p, r, so, w2, w1, dt, time_m, time_M, damp, params, lo=None, hi=None, src=None, rec=None,
                grad=None, gh=0, usave=None, vsave=None, mut=None):
    """Adjoint steps time_M .. time_m. `src` (the receivers of the reference) is injected, `rec` (the reference's
    srca) sampled from p + r at level time. `grad` (halo `gh`, float64, updated in place) needs usave and vsave.
    Returns (p, r, traces) in float64; the inputs are not modified."""
    p = np.array(p, dtype=np.float64)
    r = np.array(r, dtype=np.float64)
    T = p.shape[0]
    lo, hi = _bounds(p.shape[1:], so, lo, hi)
    w2 = _weights(w2, None)
    w1 = _weights(w1, None)
    P = {k: np.asarray(x, dtype=np.float64) for k, x in params.items()}
    box = _box(lo, hi, so)
    gzz = _gzz_factory(so, w1, P, lo, hi)
    e2_all = 1 + 2 * P['epsilon']
    sd_all = np.sqrt(1 + 2 * P['delta'])
    e2b, sdb = _at(e2_all, box), _at(sd_all, box)
    vp_all = P['vp']
    m = 1.0 / _at(vp_all * vp_all, box)
    d = _at(np.asarray(damp, dtype=np.float64), box) if damp is not None else 0.0
    den = m / dt ** 2 + d / dt
    S = _Support(src, lo, hi, so) if src is not None else None
    R_ = _Support(rec, lo, hi, so) if rec is not None else None
    traces = np.array(rec['data'], dtype=np.float64) if rec is not None else None
    inj_scale = dt * dt * vp_all * vp_all
    gh_ = lambda f: _lap(f, w2, lo, hi, so) - gzz(f)
    for time in range(time_M, time_m - 1, -1):
        t0, t1, t2 = time % T, (time - 1) % T, (time + 1) % T
        p0, r0 = p[t0], r[t0]
        if mut == 'fwd_mix':
            H0 = e2b * gh_(p0) + sdb * gzz(r0)
            Hz = sdb * gh_(p0) + gzz(r0)
        elif mut == 'mix_at_output':
            H0 = e2b * gh_(p0) + sdb * gh_(r0)
            Hz = sdb * gzz(p0) + gzz(r0)
        else:
            a = e2_all * p0 + sd_all * r0
            b = sd_all * p0 + r0
            if mut == 'mix_swap':
                a, b = b, a
            H0, Hz = gh_(a), gzz(b)
        pn = (m / dt ** 2 * (2 * p0[box] - p[t2][box]) + d / dt * p0[box] + H0) / den
        rn = (m / dt ** 2 * (2 * r0[box] - r[t2][box]) + d / dt * r0[box] + Hz) / den
        _store(p[t1], pn, lo, hi, so, None)
        _store(r[t1], rn, lo, hi, so, None)
        before = (p[t1][box].copy(), r[t1][box].copy())
        if S is not None:
            S.inject([p[t0], r[t0]] if mut == 'inject_level' else [p[t1], r[t1]], time, inj_scale)
        if R_ is not None:
            R_.interpolate(traces, [p[t0], r[t0]], time)
        if grad is not None:
            us, vs = np.asarray(usave[time], np.float64), np.asarray(vsave[time], np.float64)
            if mut == 'img_swap':
                us, vs = vs, us
            p1, r1 = before if mut == 'img_before_inject' else (p[t1][box], r[t1][box])
            term = us[box] * (p1 - 2 * p0[box] + p[t2][box]) / dt ** 2 + \
                vs[box] * (r1 - 2 * r0[box] + r[t2][box]) / dt ** 2
            grad[_box(lo, hi, gh)] -= term
    return p, r, traces


def tti_forward(*args, **kw):
    """ref64.tti_forward, re-exported for the dot test."""
    return R64.tti_forward(*args, **kw)
