"""float64 restatement of the 2-D centred-TTI operators (reference: examples/seismic/tti/operators.py
`Gzz_centered_2d`, `Gh_centered`, `kernel_centered`, `ForwardOperator`, `AdjointOperator`, `JacobianOperator`,
`JacobianAdjOperator`) on arrays laid out like the wavefields, (x + 2 so, z + 2 so) per time slot:

  D+_d f (p) = sum_j w1_d[j] f(p + (j - R/2 + 1) e_d),   D-_d g (p) = sum_j w1_d[j] g(p + (j - R/2) e_d)
  Gz(f)  = sin(th) D+_x f + cos(th) D+_z f                     (th at the Gz point)
  Gzz(f) = D-_x(sin(th) Gz f) + D-_z(cos(th) Gz f)             (th at the shifted points)
  forward:  H0 = e2 (lap u - Gzz u) + sd Gzz v,  Hz = sd (lap u - Gzz u) + Gzz v
  adjoint:  H0 = lap a - Gzz a, Hz = Gzz b with a = e2 p + sd r, b = sd p + r  (e2 = 1+2 eps, sd = sqrt(1+2 delta))
  f[t+-1] = (m/dt^2 (2 f[t] - f[t-+1]) + damp/dt f[t] + H) / (m/dt^2 + damp/dt)

Born adds -dm (u0[t+1] - 2 u0[t] + u0[t-1]) / dt^2 / (m/dt^2 + damp/dt) to du[t+1] (dv likewise, u0.dt2 taken after
the injection); the gradient subtracts usave[time] p.dt2 + vsave[time] r.dt2 after each adjoint step and its injection.
Sources are injected with dt^2 vp^2 into the level written, receivers sample f + g at level t (tests/ref64._Support).

MUTATIONS are the kernel bugs the restatement must tell apart from the reference.
"""
import numpy as np

from ref64 import _Support, _at, _box, _lap

MUTATIONS = {
    'sincos_swap': "sin and cos of theta exchanged",
    'theta_at_output': "theta of the outer derivative taken at the output point instead of the shifted points",
    'inner_full_order': "the inner derivative D+ at full order (space_order) instead of space_order / 2",
    'fwd_mix': "the adjoint run with the forward combination",
    'mix_at_output': "adjoint: e2 and sd of the mixes taken at the output point instead of at every tap point",
    'mix_swap': "adjoint: the two mixes exchanged between the equations",
    'inject_level': "adjoint: the receivers injected into level t instead of the level just written",
    'born_sign': "Born: the linearised pair driven by +dm u0.dt2 instead of -dm u0.dt2",
    'born_before_inject': "Born: u0.dt2 / v0.dt2 taken before the injection into u0[t+1] / v0[t+1]",
    'born_dm_shift': "Born: dm read one point off along x",
    'tti_born_swap': "Born: du driven by v0.dt2 and dv by u0.dt2",
    'img_swap': "gradient: usave and vsave exchanged",
    'img_before_inject': "gradient: p.dt2 / r.dt2 taken before the injection",
}


def half_weights(R, h):
    """The weights of D+ (half-node first derivative) of order R for offsets -R/2+1 .. R/2, divided by h."""
    import sympy
    offs = list(range(-(R // 2) + 1, R // 2 + 1))
    c = sympy.finite_diff_weights(1, offs, sympy.Rational(1, 2))[-1][-1]
    return np.array([float(x) for x in c]) / float(h)


class Scheme:
    """The operator pieces on the box [lo, hi] (grid indices) of a (x + 2 so, z + 2 so) layout."""

    def __init__(self, so, w2, w1, dt, damp, params, lo, hi, mut=None):
        self.so, self.R, self.dt, self.lo, self.hi, self.mut = so, so // 2, dt, list(lo), list(hi), mut
        self.w2 = [np.asarray(w, np.float64) for w in w2]
        self.w1 = [np.asarray(w, np.float64) for w in w1]
        P = {k: np.asarray(v, np.float64) for k, v in params.items()}
        th = P['theta']
        st, ct = np.sin(th), np.cos(th)
        if mut == 'sincos_swap':
            st, ct = ct, st
        self.st, self.ct = st, ct
        self.e2_all = 1 + 2 * P['epsilon']
        self.sd_all = np.sqrt(1 + 2 * P['delta'])
        self.box = _box(lo, hi, so)
        self.e2, self.sd = _at(self.e2_all, self.box), _at(self.sd_all, self.box)
        self.vp2_all = P['vp'] * P['vp']
        self.m = 1.0 / _at(self.vp2_all, self.box)
        self.d = _at(np.asarray(damp, np.float64), self.box) if damp is not None else 0.0
        self.den = self.m / dt ** 2 + self.d / dt

    def _sl(self, lo, hi, shift):
        return _box(lo, hi, self.so, shift)

    def gzz(self, f):
        R, h = self.R, self.R // 2
        lo, hi = self.lo, self.hi
        elo, ehi = [x - h for x in lo], [x + h - 1 for x in hi]
        eb = self._sl(elo, ehi, (0, 0))
        if self.mut == 'inner_full_order':              # D+ over offsets -R+1 .. R with the order-2R weights
            hs = [1.0 / self.w1[d][-1] * (half_weights(R, 1.0)[-1]) for d in range(2)]
            wi = [half_weights(2 * R, hs[d]) for d in range(2)]
            offs = list(range(-R + 1, R + 1))
        else:
            wi = self.w1
            offs = list(range(-h + 1, h + 1))
        dx = sum(wi[0][j] * f[self._sl(elo, ehi, (o, 0))] for j, o in enumerate(offs))
        dz = sum(wi[1][j] * f[self._sl(elo, ehi, (0, o))] for j, o in enumerate(offs))
        gz = _at(self.st, eb) * dx + _at(self.ct, eb) * dz
        nb = [b - a + 1 for a, b in zip(lo, hi)]
        cut = lambda a, s: a[h + s[0]:h + s[0] + nb[0], h + s[1]:h + s[1] + nb[1]]
        if self.mut == 'theta_at_output':
            sx, cz = _at(self.st, self.box), _at(self.ct, self.box)
            return sum(self.w1[0][j] * sx * cut(gz, (j - h, 0)) + self.w1[1][j] * cz * cut(gz, (0, j - h))
                       for j in range(R))
        sgz, cgz = _at(self.st, eb) * gz, _at(self.ct, eb) * gz
        return sum(self.w1[0][j] * cut(sgz, (j - h, 0)) + self.w1[1][j] * cut(cgz, (0, j - h)) for j in range(R))

    def lap(self, f):
        return _lap(f, self.w2, self.lo, self.hi, self.so)

    def update(self, fc, fprev, H):
        b = self.box
        return (self.m / self.dt ** 2 * (2 * fc[b] - fprev[b]) + self.d / self.dt * fc[b] + H) / self.den

    def forward_H(self, u, v):
        gxx = self.lap(u) - self.gzz(u)
        gzz = self.gzz(v)
        return self.e2 * gxx + self.sd * gzz, self.sd * gxx + gzz

    def adjoint_H(self, p, r):
        if self.mut == 'fwd_mix':
            return self.forward_H(p, r)
        if self.mut == 'mix_at_output':
            ghp, ghr = self.lap(p) - self.gzz(p), self.lap(r) - self.gzz(r)
            return self.e2 * ghp + self.sd * ghr, self.sd * self.gzz(p) + self.gzz(r)
        a = self.e2_all * p + self.sd_all * r
        b = self.sd_all * p + r
        if self.mut == 'mix_swap':
            a, b = b, a
        return self.lap(a) - self.gzz(a), self.gzz(b)


def _support(sp, lo, hi, so):
    return _Support(sp, lo, hi, so) if sp is not None else None


def forward(u, v, so, w2, w1, dt, time_m, time_M, damp, params, lo=None, hi=None, src=None, rec=None,
            du=None, dv=None, dm=None, dmh=0, mut=None):
    """Forward steps time_m .. time_M (`ForwardTTI`); with du, dv, dm the linearised pair of `BornTTI` too, the
    receivers then sampling du + dv. Returns (u, v, du, dv, traces) in float64; the inputs are not modified."""
    u, v = np.array(u, np.float64), np.array(v, np.float64)
    born = du is not None
    if born:
        du, dv = np.array(du, np.float64), np.array(dv, np.float64)
    T = u.shape[0]
    n = [s - 2 * so for s in u.shape[1:]]
    lo = list(lo) if lo is not None else [0, 0]
    hi = list(hi) if hi is not None else [x - 1 for x in n]
    S = Scheme(so, w2, w1, dt, damp, params, lo, hi, mut)
    Src, Rec = _support(src, lo, hi, so), _support(rec, lo, hi, so)
    traces = np.array(rec['data'], np.float64) if rec is not None else None
    scale = dt * dt * S.vp2_all
    b = S.box
    dmb = None
    if born:
        dm = np.asarray(dm, np.float64)
        dmb = (np.roll(dm, -1, axis=0) if mut == 'born_dm_shift' else dm)[_box(lo, hi, dmh)]
    for time in range(time_m, time_M + 1):
        t0, t1, t2 = time % T, (time + 1) % T, (time - 1) % T
        H0, Hz = S.forward_H(u[t0], v[t0])
        un, vn = S.update(u[t0], u[t2], H0), S.update(v[t0], v[t2], Hz)
        u[t1][b], v[t1][b] = un, vn
        if Src is not None:
            Src.inject([u[t1], v[t1]], time, scale)
        if born:
            G0, Gz_ = S.forward_H(du[t0], dv[t0])
            dun, dvn = S.update(du[t0], du[t2], G0), S.update(dv[t0], dv[t2], Gz_)
            u1, v1 = (un, vn) if mut == 'born_before_inject' else (u[t1][b], v[t1][b])
            if mut == 'born_sign' and time == time_m:
                dmb = -dmb
            qu = (u1 - 2 * u[t0][b] + u[t2][b]) / dt ** 2
            qv = (v1 - 2 * v[t0][b] + v[t2][b]) / dt ** 2
            if mut == 'tti_born_swap':
                qu, qv = qv, qu
            dun = dun - dmb * qu / S.den
            dvn = dvn - dmb * qv / S.den
            du[t1][b], dv[t1][b] = dun, dvn
        if Rec is not None:
            Rec.interpolate(traces, [du[t0], dv[t0]] if born else [u[t0], v[t0]], time)
    return u, v, du, dv, traces


def adjoint(p, r, so, w2, w1, dt, time_m, time_M, damp, params, lo=None, hi=None, src=None, rec=None,
            grad=None, gh=0, usave=None, vsave=None, mut=None):
    """Adjoint steps time_M .. time_m (`AdjointTTI`); with grad (float64, halo gh, updated in place), usave and
    vsave the imaging condition of `GradientTTI`. Returns (p, r, traces) in float64."""
    p, r = np.array(p, np.float64), np.array(r, np.float64)
    T = p.shape[0]
    n = [s - 2 * so for s in p.shape[1:]]
    lo = list(lo) if lo is not None else [0, 0]
    hi = list(hi) if hi is not None else [x - 1 for x in n]
    S = Scheme(so, w2, w1, dt, damp, params, lo, hi, mut)
    Src, Rec = _support(src, lo, hi, so), _support(rec, lo, hi, so)
    traces = np.array(rec['data'], np.float64) if rec is not None else None
    scale = dt * dt * S.vp2_all
    b = S.box
    for time in range(time_M, time_m - 1, -1):
        t0, t1, t2 = time % T, (time - 1) % T, (time + 1) % T
        H0, Hz = S.adjoint_H(p[t0], r[t0])
        p[t1][b], r[t1][b] = S.update(p[t0], p[t2], H0), S.update(r[t0], r[t2], Hz)
        before = (p[t1][b].copy(), r[t1][b].copy())
        if Src is not None:
            Src.inject([p[t0], r[t0]] if mut == 'inject_level' else [p[t1], r[t1]], time, scale)
        if Rec is not None:
            Rec.interpolate(traces, [p[t0], r[t0]], time)
        if grad is not None:
            us, vs = np.asarray(usave[time], np.float64), np.asarray(vsave[time], np.float64)
            if mut == 'img_swap':
                us, vs = vs, us
            p1, r1 = before if mut == 'img_before_inject' else (p[t1][b], r[t1][b])
            grad[_box(lo, hi, gh)] -= (us[b] * (p1 - 2 * p[t0][b] + p[t2][b]) +
                                       vs[b] * (r1 - 2 * r[t0][b] + r[t2][b])) / dt ** 2
    return p, r, traces
