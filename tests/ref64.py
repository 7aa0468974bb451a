"""Float64 NumPy restatement of the explicit time steps the sweep kernels implement.

This is the yardstick of tests/test_kernel_matrix.py (GPU) and tests/test_ref64.py (CPU). It is independent of the
product package and of the C oracle: whole-array slicing, no loops over points, second- and first-derivative weights
computed from sympy's exact rationals, every array widened to float64.

Conventions (those of `data_with_halo` and of the C ABI):
  - wavefields are (T, X, Y, Z) with a halo of `so` points on every space axis; parameter arrays (damp, vp, m and
    the TTI parameters) have the same space layout;
  - `lo` / `hi` are the inclusive update box in domain indices (the operator's x_m .. z_M). Cells outside the box
    keep what their time slot holds; the stencil reads the halo as stored (it is not assumed to be zero);
  - time step `time` reads slots time % T and (time - 1) % T and writes (time + 1) % T, then injects the sources
    into the written slot, then samples the receivers at time level time + rec_toff.

Iso acoustic (the reference's damped update, examples/seismic/acoustic/operators.py):
    (m/dt^2 + damp/dt) u+ = 2m/dt^2 u - m/dt^2 u- + damp/dt u + sum_d sum_k w_d[k] (u[+k e_d] + u[-k e_d])
TTI, centred scheme (examples/seismic/tti/operators.py), C = (sin th cos ph, sin th sin ph, cos th):
    Gz(f)(q)  = sum_e C_e(q) D+_e f(q),      D+_e f(q) = sum_j w1_e[j] f(q + (j - R/2 + 1) e_e)
    Gzz(f)(p) = sum_d sum_j w1_d[j] C_d(q) Gz(f)(q),   q = p + (j - R/2) e_d
    (m/dt^2 + damp/dt) u+ = e2 (lap u - Gzz u) + sd Gzz v + m/dt^2 (2u - u-) + damp/dt u
    (m/dt^2 + damp/dt) v+ = sd (lap u - Gzz u) + Gzz v + m/dt^2 (2v - v-) + damp/dt v
    with e2 = 1 + 2 epsilon, sd = sqrt(1 + 2 delta) and m = 1/vp^2 taken at p.
Sparse points (devito/operations/interpolators.py): base cell and per-axis weights from the host-side tabulation;
a support cell c counts when lo - r <= c <= hi + r on every axis. Injection adds w * src[time] * dt^2 / m(c) to
the written slot (of u and v for TTI), interpolation sums w * f(c) (u + v for TTI).

`mut` selects one deliberate mistake from MUTATIONS. The sensitivity tests run the reference with each of them to
show that the inputs make that kind of kernel bug visible far above the tolerance.
"""
import numpy as np
import sympy

MUTATIONS = {
    'w_xy': "per-axis weights of x and y exchanged",
    'w_yz': "per-axis weights of y and z exchanged",
    'transpose_xy': "x and y of the input wavefields exchanged (on the leading square of the x-y plane)",
    'halo_zero': "the stencil reads the halo as zero",
    'shift_x': "array parameters read one point off along x",
    'shift_y': "array parameters read one point off along y",
    'shift_z': "array parameters read one point off along z",
    'c_at_output': "TTI: the outer derivative takes C_d at the output point instead of the shifted point",
    'tail_y': "the last row of the box in y is not updated",
    'tail_z': "the last four points of the box in z (one float4 group) are not updated",
    'swap_levels': "u and u- exchanged in the update",
}


def fd2_weights(space_order, h):
    """Second-derivative weights / h^2 for offsets 0..so/2 (symmetric), exact rationals rounded once."""
    R = space_order // 2
    c = sympy.finite_diff_weights(2, list(range(-R, R + 1)), 0)[-1][-1]
    return np.array([float(c[R + k]) for k in range(R + 1)]) / float(h) ** 2


def fd1_half_weights(space_order, h):
    """First-derivative weights / h about x + h/2 for offsets -R/2+1 .. R/2, R = so/2 (the TTI D+ operator)."""
    R = space_order // 2
    offs = list(range(-(R // 2) + 1, R // 2 + 1))
    c = sympy.finite_diff_weights(1, offs, sympy.Rational(1, 2))[-1][-1]
    return np.array([float(x) for x in c]) / float(h)


def _box(lo, hi, so, shift=(0, 0, 0)):
    return tuple(slice(l + so + s, h + so + 1 + s) for l, h, s in zip(lo, hi, shift))


def _unit(d, k):
    e = [0, 0, 0]
    e[d] = k
    return tuple(e)


def _bounds(shape, so, lo, hi):
    n = [s - 2 * so for s in shape]
    lo = list(lo) if lo is not None else [0, 0, 0]
    hi = list(hi) if hi is not None else [x - 1 for x in n]
    return lo, hi


def _halo_zeroed(f, so):
    g = np.zeros_like(f)
    dom = tuple(slice(so, s - so) for s in f.shape)
    g[dom] = f[dom]
    return g


def _shifted(a, mut):
    """An array parameter as the mutated kernel would read it."""
    if a is None or np.ndim(a) == 0 or mut not in ('shift_x', 'shift_y', 'shift_z'):
        return a
    return np.roll(a, 1, axis='xyz'.index(mut[-1]))


def _at(a, sl):
    return a[sl] if np.ndim(a) else a


def _weights(w, mut):
    w = [np.asarray(x, dtype=np.float64) for x in w]
    if mut == 'w_xy':
        w[0], w[1] = w[1], w[0]
    elif mut == 'w_yz':
        w[1], w[2] = w[2], w[1]
    return w


def _transpose_xy(f):
    k = min(f.shape[1], f.shape[2])
    f[:, :k, :k, :] = f[:, :k, :k, :].transpose(0, 2, 1, 3).copy()


def _lap(f, w, lo, hi, so):
    R = len(w[0]) - 1
    out = (w[0][0] + w[1][0] + w[2][0]) * f[_box(lo, hi, so)]
    for d in range(3):
        for k in range(1, R + 1):
            out = out + w[d][k] * (f[_box(lo, hi, so, _unit(d, k))] + f[_box(lo, hi, so, _unit(d, -k))])
    return out


def _store(f1, new, lo, hi, so, mut):
    """Write the updated box, minus the part a mutated kernel leaves alone."""
    box = _box(lo, hi, so)
    if mut == 'tail_y':
        new[:, -1, :] = f1[box][:, -1, :]
    elif mut == 'tail_z':
        new[:, :, -4:] = f1[box][:, :, -4:]
    f1[box] = new


class _Support:
    """The valid support cells of every sparse point: flat (point, cell) lists with the product weight."""

    def __init__(self, sp, lo, hi, so):
        gp = np.asarray(sp['gp'], dtype=np.int64)
        r = int(sp['r'])
        n = 2 * r
        off = np.arange(n) - r + 1
        c = [gp[:, d, None] + off[None, :] for d in range(3)]                 # (npoint, 2r) per axis
        ws = [np.asarray(x, dtype=np.float64) for x in sp['w']]
        C = np.broadcast_arrays(c[0][:, :, None, None], c[1][:, None, :, None], c[2][:, None, None, :])
        W = ws[0][:, :, None, None] * ws[1][:, None, :, None] * ws[2][:, None, None, :]
        P = np.broadcast_to(np.arange(gp.shape[0])[:, None, None, None], W.shape)
        ok = np.ones(W.shape, dtype=bool)
        for d in range(3):
            ok &= (C[d] >= lo[d] - r) & (C[d] <= hi[d] + r)
        self.idx = tuple(C[d][ok] + so for d in range(3))
        self.w = W[ok]
        self.p = P[ok]
        self.npoint = gp.shape[0]
        self.data = np.asarray(sp['data'], dtype=np.float64)

    def inject(self, fields, time, scale):
        """fields[cell] += w * src[time] * scale(cell); several points may share a cell."""
        if not 0 <= time < self.data.shape[0]:
            return
        val = self.w * self.data[time, self.p] * (scale[self.idx] if np.ndim(scale) else scale)
        for f in fields:
            np.add.at(f, self.idx, val)

    def interpolate(self, out, fields, time):
        if not 0 <= time < out.shape[0]:
            return
        v = sum(f[self.idx] for f in fields)
        out[time] = np.bincount(self.p, weights=self.w * v, minlength=self.npoint)


def iso_forward(u, so, w, dt, time_m, time_M, damp=None, param=('vp', 1.5), lo=None, hi=None, src=None, rec=None,
                rec_toff=0, mut=None):
    """Isotropic acoustic time steps time_m .. time_M. `param` = ('vp', scalar or array) or ('m', array).
    Returns (u, traces) in float64; the inputs are not modified."""
    u = np.array(u, dtype=np.float64)
    T = u.shape[0]
    lo, hi = _bounds(u.shape[1:], so, lo, hi)
    w = _weights(w, mut)
    box = _box(lo, hi, so)
    kind, pv = param
    pv = _shifted(np.asarray(pv, dtype=np.float64), mut)
    m_all = 1.0 / (pv * pv) if kind == 'vp' else pv                   # squared slowness, where it is sampled
    m = _at(m_all, box)
    d = _at(np.asarray(damp, dtype=np.float64), box) if damp is not None else 0.0
    if mut == 'transpose_xy':
        _transpose_xy(u)
    S = _Support(src, lo, hi, so) if src is not None else None
    R_ = _Support(rec, lo, hi, so) if rec is not None else None
    traces = np.array(rec['data'], dtype=np.float64) if rec is not None else None
    inj_scale = dt * dt / m_all
    for time in range(time_m, time_M + 1):
        t0, t1, t2 = time % T, (time + 1) % T, (time - 1) % T
        if mut == 'swap_levels':
            t0, t2 = t2, t0
        u0 = _halo_zeroed(u[t0], so) if mut == 'halo_zero' else u[t0]
        lap = _lap(u0, w, lo, hi, so)
        c = u0[box]
        new = (2 * m / dt ** 2 * c - m / dt ** 2 * u[t2][box] + d / dt * c + lap) / (m / dt ** 2 + d / dt)
        _store(u[t1], new, lo, hi, so, mut)
        if S is not None:
            S.inject([u[t1]], time, inj_scale)
        if R_ is not None:
            R_.interpolate(traces, [u[t1] if rec_toff else u[time % T]], time)
    return u, traces


def tti_forward(u, v, so, w2, w1, dt, time_m, time_M, damp, params, lo=None, hi=None, src=None, rec=None,
                rec_toff=0, mut=None):
    """TTI (centred) time steps time_m .. time_M. `params`: vp, epsilon, delta, theta, phi -> scalar or array.
    Returns (u, v, traces) in float64; the inputs are not modified."""
    u = np.array(u, dtype=np.float64)
    v = np.array(v, dtype=np.float64)
    T = u.shape[0]
    R = so // 2
    h = R // 2
    lo, hi = _bounds(u.shape[1:], so, lo, hi)
    w2 = _weights(w2, mut)
    w1 = _weights(w1, mut)
    P = {k: _shifted(np.asarray(x, dtype=np.float64), mut) for k, x in params.items()}
    box = _box(lo, hi, so)
    # Gz is needed on the box grown by [-h, h-1]: the points q of the outer derivative
    elo = [x - h for x in lo]
    ehi = [x + h - 1 for x in hi]
    ebox = _box(elo, ehi, so)
    nb = [b - a + 1 for a, b in zip(lo, hi)]
    st, ct = np.sin(P['theta']), np.cos(P['theta'])
    sp, cp = np.sin(P['phi']), np.cos(P['phi'])
    Call = [st * cp, st * sp, ct * np.ones_like(sp)]
    CE = [_at(x, ebox) for x in Call]                                # C at the points of the grown box
    CB = [_at(x, box) for x in Call]                                 # ... and at the output points
    e2 = 1 + 2 * _at(P['epsilon'], box)
    sd = np.sqrt(1 + 2 * _at(P['delta'], box))
    vp_all = P['vp']
    m = 1.0 / _at(vp_all * vp_all, box)
    d = _at(np.asarray(damp, dtype=np.float64), box) if damp is not None else 0.0
    if mut == 'transpose_xy':
        _transpose_xy(u)
        _transpose_xy(v)

    def gzz(f):
        gz = 0.0
        for e in range(3):
            de = sum(w1[e][j] * f[_box(elo, ehi, so, _unit(e, j - h + 1))] for j in range(R))
            gz = gz + CE[e] * de
        out = 0.0
        for dd in range(3):
            cg = gz if mut == 'c_at_output' else CE[dd] * gz
            acc = 0.0
            for j in range(R):
                s = _unit(dd, j - h)
                sl = tuple(slice(h + s[a], h + s[a] + nb[a]) for a in range(3))   # box shifted, in grown-box indices
                acc = acc + w1[dd][j] * cg[sl]
            out = out + (CB[dd] * acc if mut == 'c_at_output' else acc)
        return out

    S = _Support(src, lo, hi, so) if src is not None else None
    R_ = _Support(rec, lo, hi, so) if rec is not None else None
    traces = np.array(rec['data'], dtype=np.float64) if rec is not None else None
    inj_scale = dt * dt * vp_all * vp_all
    for time in range(time_m, time_M + 1):
        t0, t1, t2 = time % T, (time + 1) % T, (time - 1) % T
        if mut == 'swap_levels':
            t0, t2 = t2, t0
        u0 = _halo_zeroed(u[t0], so) if mut == 'halo_zero' else u[t0]
        v0 = _halo_zeroed(v[t0], so) if mut == 'halo_zero' else v[t0]
        lap = _lap(u0, w2, lo, hi, so)
        gu, gv = gzz(u0), gzz(v0)
        den = m / dt ** 2 + d / dt
        un = (e2 * (lap - gu) + sd * gv + m / dt ** 2 * (2 * u0[box] - u[t2][box]) + d / dt * u0[box]) / den
        vn = (sd * (lap - gu) + gv + m / dt ** 2 * (2 * v0[box] - v[t2][box]) + d / dt * v0[box]) / den
        _store(u[t1], un, lo, hi, so, mut)
        _store(v[t1], vn, lo, hi, so, mut)
        if S is not None:
            S.inject([u[t1], v[t1]], time, inj_scale)
        if R_ is not None:
            lvl = t1 if rec_toff else time % T
            R_.interpolate(traces, [u[lvl], v[lvl]], time)
    return u, v, traces
