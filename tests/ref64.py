"""Float64 NumPy restatement of the explicit time steps the sweep kernels implement.

This is the yardstick of tests/test_kernel_matrix.py and tests/test_scheme_matrix.py (GPU) and tests/test_ref64.py
(CPU). It is independent of the product package and of the C oracle: whole-array slicing, no loops over points,
second- and first-derivative weights computed from sympy's exact rationals, every array widened to float64.

Conventions (those of `data_with_halo` and of the C ABI):
  - wavefields are (T, X, Y, Z) (2-D: (T, X, Y)) with a halo of `so` points on every space axis; parameter arrays
    (damp, vp, m and the TTI parameters) have the same space layout;
  - `lo` / `hi` are the inclusive update box in domain indices (the operator's x_m .. z_M). Cells outside the box
    keep what their time slot holds; the stencil reads the halo as stored (it is not assumed to be zero);
  - time step `time` reads slots time % T and (time - 1) % T and writes (time + 1) % T, then injects the sources
    into the written slot, then samples the receivers at time level time + rec_toff.

Iso acoustic (the reference's damped update, examples/seismic/acoustic/operators.py):
    (m/dt^2 + damp/dt) u+ = 2m/dt^2 u - m/dt^2 u- + damp/dt u + H,   H = sum_d sum_k w_d[k] (u[+k e_d] + u[-k e_d])
and the schemes built on it (`iso_forward` / `born_forward` keywords):
  - adjoint: time runs from time_M down to time_m; step `time` writes (time - 1) % T from time % T and
    (time + 1) % T, injects into the slot just written, samples receivers at time % T (the written slot with
    rec_toff);
  - free surface (lo[-1] == 0): after the plain update, rows z <= R of the box are recomputed with every vertical
    tap that reaches z - k < 0 reading -u[k - z] and a tap landing on z - k == 0 contributing 0; then row z = 0 of
    the written slot is cleared, then the sources are injected. The halo above the surface is neither read by the
    mirror nor written by it;
  - OT4: H = lap(u) + dt^2/12 lap(W), W = lap(u) / m on the box grown by R with 1/m at the grown-box point;
  - Born: u is stepped and the sources injected into it first; then U gets the plain update plus
    -dm (u+ - 2u + u-)/dt^2 / (m/dt^2 + damp/dt), with the u levels after the injection; `dm` has its own halo
    `dmh`; receivers sample U;
  - imaging condition: after each (adjoint) step and its injection,
    grad[box + gh] -= usave[time][box] (v+ - 2v + v-)/dt^2, `grad` with its own halo `gh`;
  - snapshots: when time % factor == 0, the box of u[t + snap_toff] (after the injection) is copied into
    snap[time // factor] at box + snap_h; every other cell of `snap` keeps its value.
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
    'tail_z_over': "the 1-3 points past z_M in the last float4 group of a row are updated too",
    'tail_z_short': "the last n2 % 4 points of the box in z (a partial float4 group) are not updated",
    'swap_levels': "u and u- exchanged in the update",
    'adj_inject_level': "adjoint: the sources are injected into u[t] instead of the level just written",
    'fs_surface_tap': "free surface: the vertical tap landing on z = 0 reads u[0] instead of contributing 0",
    'fs_mirror_sign': "free surface: taps above the surface read +u[k - z] instead of -u[k - z]",
    'fs_keep_row0': "free surface: row z = 0 of the written level is not cleared",
    'fs_rows_lt_R': "free surface: only rows z < R are recomputed (row z = R keeps the plain update)",
    'ot4_m_at_output': "OT4: 1/m of the inner Laplacian taken at the output point instead of the shifted point",
    'ot4_factor': "OT4: dt^2/6 instead of dt^2/12",
    'born_before_inject': "Born: u.dt2 taken before the sources were injected into u+",
    'born_dm_shift': "Born: dm read one point off along x",
    'grad_usave_time': "imaging condition: usave[time + 1] instead of usave[time]",
    'grad_assign': "imaging condition: grad = -u v.dt2 instead of grad -= u v.dt2",
    'grad_halo': "imaging condition: the halo width of grad ignored",
    'snap_level': "snapshots: taken from the other time level (u[t] <-> u[t+1])",
    'snap_index': "snapshots: written to index time // factor + 1",
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


def _unit(d, k, nd=3):
    e = [0] * nd
    e[d] = k
    return tuple(e)


def _bounds(shape, so, lo, hi):
    n = [s - 2 * so for s in shape]
    lo = list(lo) if lo is not None else [0] * len(n)
    hi = list(hi) if hi is not None else [x - 1 for x in n]
    return lo, hi


def _update_hi(lo, hi, mut):
    """The upper corner of the points a kernel updates: with 'tail_z_over', the z extent rounded up to whole float4
    groups (the sparse points still see the box as given)."""
    if mut != 'tail_z_over':
        return hi
    return list(hi[:-1]) + [lo[-1] + (hi[-1] - lo[-1] + 4) // 4 * 4 - 1]


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
    elif mut == 'w_yz' and len(w) == 3:
        w[1], w[2] = w[2], w[1]
    return w


def _transpose_xy(f):
    k = min(f.shape[1], f.shape[2])
    f[:, :k, :k, :] = f[:, :k, :k, :].transpose(0, 2, 1, 3).copy()


def _lap(f, w, lo, hi, so):
    nd = len(w)
    R = len(w[0]) - 1
    out = sum(x[0] for x in w) * f[_box(lo, hi, so)]
    for d in range(nd):
        for k in range(1, R + 1):
            out = out + w[d][k] * (f[_box(lo, hi, so, _unit(d, k, nd))] + f[_box(lo, hi, so, _unit(d, -k, nd))])
    return out


def _fs_correction(f, w, lo, hi, so, mut):
    """Free surface: what the mirrored vertical taps add to the plain Laplacian on rows z = 0 .. R of the box.
    Tap z - k reads E[z - k] instead of f[z - k]: E = f below the surface, 0 on it, -f[k - z] above it."""
    nd = len(w)
    R = len(w[0]) - 1
    rows = min(R, hi[-1]) + 1                                          # the box starts at z = 0
    flo, fhi = list(lo), list(hi)
    fhi[-1] = rows - 1
    lead = _box(flo[:-1], fhi[:-1], so)
    corr = 0.0
    for k in range(1, R + 1):
        z = np.arange(rows)
        src = z - k                                                    # domain index of the tap
        mirrored = np.where(src < 0, -src, src) + so
        sign = np.where(src < 0, 1.0 if mut == 'fs_mirror_sign' else -1.0, 1.0)
        if mut != 'fs_surface_tap':
            sign = np.where(src == 0, 0.0, sign)
        tap = f[lead + (src + so,)]
        corr = corr + w[-1][k] * (sign * f[lead + (mirrored,)] - tap)
    if mut == 'fs_rows_lt_R' and rows == R + 1:
        corr[..., R] = 0.0
    return corr, rows


class _Support:
    """The valid support cells of every sparse point: flat (point, cell) lists with the product weight."""

    def __init__(self, sp, lo, hi, so):
        gp = np.asarray(sp['gp'], dtype=np.int64)
        nd = gp.shape[1]
        r = int(sp['r'])
        n = 2 * r
        off = np.arange(n) - r + 1
        ws = [np.asarray(x, dtype=np.float64) for x in sp['w']]

        def axis(a, d):                                                # (npoint, 2r) -> broadcast along axis d
            return a[(slice(None),) + tuple(slice(None) if e == d else None for e in range(nd))]
        C = np.broadcast_arrays(*[axis(gp[:, d, None] + off[None, :], d) for d in range(nd)])
        W = axis(ws[0], 0)
        for d in range(1, nd):
            W = W * axis(ws[d], d)
        P = np.broadcast_to(np.arange(gp.shape[0]).reshape((-1,) + (1,) * nd), W.shape)
        ok = np.ones(W.shape, dtype=bool)
        for d in range(nd):
            ok &= (C[d] >= lo[d] - r) & (C[d] <= hi[d] + r)
        self.idx = tuple(C[d][ok] + so for d in range(nd))
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


class _Iso:
    """The damped iso update of one field on the box: coefficients and the new box values."""

    def __init__(self, so, w, dt, damp, param, lo, hi, mut):
        self.so, self.w, self.dt, self.lo, self.hi, self.mut = so, w, dt, lo, hi, mut
        self.box = _box(lo, hi, so)
        kind, pv = param
        pv = _shifted(np.asarray(pv, dtype=np.float64), mut)
        self.m_all = 1.0 / (pv * pv) if kind == 'vp' else pv           # squared slowness, where it is sampled
        self.m = _at(self.m_all, self.box)
        self.d = _at(np.asarray(damp, dtype=np.float64), self.box) if damp is not None else 0.0
        self.den = self.m / dt ** 2 + self.d / dt

    def new(self, u0, um, H):
        c = u0[self.box]
        return (2 * self.m / self.dt ** 2 * c - self.m / self.dt ** 2 * um[self.box] + self.d / self.dt * c + H) \
            / self.den

    def H(self, u0, ot4=False):
        so, w, lo, hi, mut = self.so, self.w, self.lo, self.hi, self.mut
        lap = _lap(u0, w, lo, hi, so)
        if not ot4:
            return lap
        R = len(w[0]) - 1
        glo, ghi = [x - R for x in lo], [x + R for x in hi]
        gbox = _box(glo, ghi, so)
        W = np.zeros_like(u0)
        minv = 1.0 / self.m_all
        W[gbox] = _lap(u0, w, glo, ghi, so) * (1.0 if mut == 'ot4_m_at_output' else _at(minv, gbox))
        bl = _lap(W, w, lo, hi, so)
        if mut == 'ot4_m_at_output':
            bl = bl * _at(minv, self.box)
        return lap + self.dt ** 2 / (6.0 if mut == 'ot4_factor' else 12.0) * bl


def iso_forward(u, so, w, dt, time_m, time_M, damp=None, param=('vp', 1.5), lo=None, hi=None, src=None, rec=None,
                rec_toff=0, mut=None, adjoint=False, free_surface=False, ot4=False, grad=None, gh=0, usave=None,
                snap=None, snap_h=0, snap_factor=1, snap_toff=0):
    """Isotropic acoustic time steps time_m .. time_M (3-D or 2-D). `param` = ('vp', scalar or array) or
    ('m', array). Returns (u, traces) in float64; u, damp and the parameters are not modified. `grad` (with halo
    `gh`, needs `usave`) and `snap` (nsnaps, ...) with halo `snap_h` are outputs: float64 arrays updated in place."""
    u = np.array(u, dtype=np.float64)
    T = u.shape[0]
    nd = u.ndim - 1
    lo, hi = _bounds(u.shape[1:], so, lo, hi)
    w = _weights(w, mut)
    if free_surface:
        assert lo[-1] == 0, "a free surface needs the box to start at z = 0"
    uhi = _update_hi(lo, hi, mut)
    S_ = _Iso(so, w, dt, damp, param, lo, uhi, mut)
    box = S_.box
    if mut == 'transpose_xy':
        _transpose_xy(u)
    S = _Support(src, lo, hi, so) if src is not None else None
    R_ = _Support(rec, lo, hi, so) if rec is not None else None
    traces = np.array(rec['data'], dtype=np.float64) if rec is not None else None
    inj_scale = dt * dt / S_.m_all
    dirn = -1 if adjoint else 1
    times = range(time_M, time_m - 1, -1) if adjoint else range(time_m, time_M + 1)
    for time in times:
        t0, t1, t2 = time % T, (time + dirn) % T, (time - dirn) % T
        if mut == 'swap_levels':
            t0, t2 = t2, t0
        u0 = _halo_zeroed(u[t0], so) if mut == 'halo_zero' else u[t0]
        H = S_.H(u0, ot4)
        new = S_.new(u0, u[t2], H)
        if free_surface:
            corr, rows = _fs_correction(u0, w, lo, uhi, so, mut)
            new[..., :rows] += corr / (S_.den[..., :rows] if np.ndim(S_.den) else S_.den)
            if mut != 'fs_keep_row0':
                new[..., 0] = 0.0
        _store(u[t1], new, lo, uhi, so, mut)
        if S is not None:
            S.inject([u[t0] if mut == 'adj_inject_level' else u[t1]], time, inj_scale)
        if snap is not None and time % snap_factor == 0:
            lvl = t1 if (snap_toff != 0) != (mut == 'snap_level') else t0
            idx = time // snap_factor + (1 if mut == 'snap_index' else 0)
            snap[(idx,) + _box(lo, hi, snap_h)] = u[lvl][box]
        if R_ is not None:
            R_.interpolate(traces, [u[t1] if rec_toff else u[t0]], time)
        if grad is not None:
            us = np.asarray(usave[time + 1 if mut == 'grad_usave_time' else time], dtype=np.float64)
            term = us[box] * (u[t1][box] - 2 * u[t0][box] + u[t2][box]) / dt ** 2
            gbox = _box(lo, hi, 0 if mut == 'grad_halo' else gh)
            grad[gbox] = -term if mut == 'grad_assign' else grad[gbox] - term
    return u, traces


def born_forward(u, U, dm, dmh, so, w, dt, time_m, time_M, damp=None, param=('vp', 1.5), lo=None, hi=None,
                 src=None, rec=None, mut=None):
    """Born (linearised) modelling, time_m .. time_M, 3-D: u driven by `src`, U by -dm u.dt2, `rec` sampled from
    U at time % T. `dm` has halo `dmh`. Returns (u, U, traces) in float64; the inputs are not modified."""
    u = np.array(u, dtype=np.float64)
    U = np.array(U, dtype=np.float64)
    T = u.shape[0]
    lo, hi = _bounds(u.shape[1:], so, lo, hi)
    w = _weights(w, mut)
    S_ = _Iso(so, w, dt, damp, param, lo, hi, mut)
    box = S_.box
    dm = np.asarray(dm, dtype=np.float64)
    if mut == 'born_dm_shift':
        dm = np.roll(dm, 1, axis=0)
    dmb = dm[_box(lo, hi, dmh)]
    if mut == 'transpose_xy':
        _transpose_xy(u)
        _transpose_xy(U)
    S = _Support(src, lo, hi, so) if src is not None else None
    R_ = _Support(rec, lo, hi, so) if rec is not None else None
    traces = np.array(rec['data'], dtype=np.float64) if rec is not None else None
    inj_scale = dt * dt / S_.m_all
    for time in range(time_m, time_M + 1):
        t0, t1, t2 = time % T, (time + 1) % T, (time - 1) % T
        if mut == 'swap_levels':
            t0, t2 = t2, t0
        u0 = _halo_zeroed(u[t0], so) if mut == 'halo_zero' else u[t0]
        U0 = _halo_zeroed(U[t0], so) if mut == 'halo_zero' else U[t0]
        _store(u[t1], S_.new(u0, u[t2], S_.H(u0)), lo, hi, so, mut)
        before = u[t1][box].copy()
        if S is not None:
            S.inject([u[t1]], time, inj_scale)
        u1 = before if mut == 'born_before_inject' else u[t1][box]
        q = -dmb * (u1 - 2 * u[t0][box] + u[t2][box]) / dt ** 2
        _store(U[t1], S_.new(U0, U[t2], S_.H(U0)) + q / S_.den, lo, hi, so, mut)
        if R_ is not None:
            R_.interpolate(traces, [U[time % T]], time)
    return u, U, traces


def _store(f1, new, lo, hi, so, mut):
    """Write the updated box, minus the part a mutated kernel leaves alone."""
    box = _box(lo, hi, so)
    if mut == 'tail_y':
        new[:, -1, :] = f1[box][:, -1, :]
    elif mut == 'tail_z':
        new[:, :, -4:] = f1[box][:, :, -4:]
    elif mut == 'tail_z_short' and new.shape[-1] % 4:
        k = new.shape[-1] % 4
        new[:, :, -k:] = f1[box][:, :, -k:]
    f1[box] = new


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
    uhi = _update_hi(lo, hi, mut)
    w2 = _weights(w2, mut)
    w1 = _weights(w1, mut)
    P = {k: _shifted(np.asarray(x, dtype=np.float64), mut) for k, x in params.items()}
    box = _box(lo, uhi, so)
    # Gz is needed on the box grown by [-h, h-1]: the points q of the outer derivative
    elo = [x - h for x in lo]
    ehi = [x + h - 1 for x in uhi]
    ebox = _box(elo, ehi, so)
    nb = [b - a + 1 for a, b in zip(lo, uhi)]
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
        lap = _lap(u0, w2, lo, uhi, so)
        gu, gv = gzz(u0), gzz(v0)
        den = m / dt ** 2 + d / dt
        un = (e2 * (lap - gu) + sd * gv + m / dt ** 2 * (2 * u0[box] - u[t2][box]) + d / dt * u0[box]) / den
        vn = (sd * (lap - gu) + gv + m / dt ** 2 * (2 * v0[box] - v[t2][box]) + d / dt * v0[box]) / den
        _store(u[t1], un, lo, uhi, so, mut)
        _store(v[t1], vn, lo, uhi, so, mut)
        if S is not None:
            S.inject([u[t1], v[t1]], time, inj_scale)
        if R_ is not None:
            lvl = t1 if rec_toff else time % T
            R_.interpolate(traces, [u[lvl], v[lvl]], time)
    return u, v, traces
