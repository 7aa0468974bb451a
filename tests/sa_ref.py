"""float64 restatement of the self-adjoint variable-density visco-acoustic update (reference: examples/seismic/
self_adjoint/operators.py `iso_stencil`, `IsoFwdOperator`, `IsoAdjOperator`), in the conventions of tests/ref64.py
(allocated layout with a halo of `so`, inclusive box `lo` .. `hi` in domain indices, the halo read as stored):

  c_k = sympy weights of d/dx at x + h/2 on offsets -R+1 .. R, at offset +k, over h (offset -k+1 carries -c_k)
  F_d(q)   = b(q) sum_k c_k (u(q + k e_d) - u(q - (k-1) e_d))         q = p - R .. p + R - 1
  u_new(p) = C(p) sum_d sum_k c_k (F_d(p + (k-1) e_d) - F_d(p - k e_d)) + (2 - dt w) u(p) + (dt w - 1) u_old(p)
  C = dt^2 vp^2 / b

Forward: step `time` writes (time + 1) % T from time % T and (time - 1) % T, injects `src` into the written slot with
the scale C at the cell, samples `rec` at time % T (the written slot with rec_toff). Adjoint: time runs from time_M
down to time_m, step `time` writes (time - 1) % T from time % T and (time + 1) % T, the rest alike.

`mut` selects one deliberate mistake from MUTATIONS; the sensitivity tests show each moves the answer far above the
tolerance.
"""
import numpy as np
import sympy

from ref64 import _Support, _at, _bounds, _box, _unit

MUTATIONS = {
    'b_at_output': "b taken at the output point instead of at the flux nodes",
    'b_half_node': "b averaged to the half node (b(q) + b(q+1))/2 instead of sampled at the node q",
    'order_mismatch': "the outer derivative at order 2R-2 while the inner one is at order 2R",
    'w_swap': "the two w/Q factors exchanged: (dt w - 1) u + (2 - dt w) u_old",
    'c_yz': "the per-axis weights of the last two axes exchanged",
    'last_z_group': "the last four points of the box along z (one float4 group) not updated",
}


def sa_weights(R, h):
    """c_k / h, k = 1..R, from sympy's exact rationals."""
    c = sympy.finite_diff_weights(1, list(range(-R + 1, R + 1)), sympy.Rational(1, 2))[-1][-1]
    return np.array([float(c[R - 1 + k]) for k in range(1, R + 1)]) / float(h)


def _div(u0, b, c, co, lo, hi, so, mut):
    """sum_d (D- F_d) on the box; `co` are the outer weights."""
    nd = len(c)
    R = len(c[0])
    box = _box(lo, hi, so)
    acc = 0.0
    for d in range(nd):
        glo, ghi = list(lo), list(hi)
        glo[d] -= R
        ghi[d] += R - 1
        gb = _box(glo, ghi, so)
        inner = sum(c[d][i - 1] * (u0[_box(glo, ghi, so, _unit(d, i, nd))] -
                                   u0[_box(glo, ghi, so, _unit(d, -(i - 1), nd))]) for i in range(1, R + 1))
        if mut == 'b_at_output':
            F = inner
        elif mut == 'b_half_node':
            F = inner * 0.5 * (_at(b, gb) + _at(b, _box(glo, ghi, so, _unit(d, 1, nd))))
        else:
            F = inner * _at(b, gb)
        n = hi[d] - lo[d] + 1

        def Fs(j):
            return F[tuple(slice(R + j, R + j + n) if e == d else slice(None) for e in range(nd))]
        out = sum(co[d][k - 1] * (Fs(k - 1) - Fs(-k)) for k in range(1, len(co[d]) + 1))
        if mut == 'b_at_output':
            out = out * _at(b, box)
        acc = acc + out
    return acc


def sa_forward(u, so, c, dt, time_m, time_M, b, vp, w=None, lo=None, hi=None, src=None, rec=None, rec_toff=0,
               adjoint=False, mut=None):
    """Time steps of the self-adjoint update (3-D or 2-D). `b`, `vp`: scalars or arrays in u's space layout; `w`: an
    array or None. Returns (u, traces) in float64; the inputs are not modified."""
    u = np.array(u, dtype=np.float64)
    T = u.shape[0]
    lo, hi = _bounds(u.shape[1:], so, lo, hi)
    c = [np.asarray(x, dtype=np.float64) for x in c]
    if mut == 'c_yz':
        c[-2], c[-1] = c[-1], c[-2]
    co = c
    if mut == 'order_mismatch':
        R = len(c[0])
        co = [sa_weights(R - 1, 1.0) * (x[0] / sa_weights(R, 1.0)[0]) for x in c]
    b = np.asarray(b, dtype=np.float64)
    vp = np.asarray(vp, dtype=np.float64)
    Call = dt * dt * vp * vp / b
    box = _box(lo, hi, so)
    C = _at(Call, box)
    dw = dt * _at(np.asarray(w, dtype=np.float64), box) if w is not None else 0.0
    k0, km = (2.0 - dw, dw - 1.0) if mut != 'w_swap' else (dw - 1.0, 2.0 - dw)
    S = _Support(src, lo, hi, so) if src is not None else None
    R_ = _Support(rec, lo, hi, so) if rec is not None else None
    traces = np.array(rec['data'], dtype=np.float64) if rec is not None else None
    dirn = -1 if adjoint else 1
    times = range(time_M, time_m - 1, -1) if adjoint else range(time_m, time_M + 1)
    for time in times:
        t0, t1, t2 = time % T, (time + dirn) % T, (time - dirn) % T
        new = C * _div(u[t0], b, c, co, lo, hi, so, mut) + k0 * u[t0][box] + km * u[t2][box]
        if mut == 'last_z_group':
            new[..., -4:] = u[t1][box][..., -4:]
        u[t1][box] = new
        if S is not None:
            S.inject([u[t1]], time, Call)
        if R_ is not None:
            R_.interpolate(traces, [u[t1] if rec_toff else u[t0]], time)
    return u, traces


def smooth_vp_b(shape):
    """vp and b = 1/rho of the reference goldens (oracle/make_golden_sa.py builds them with the same formula)."""
    axes = [np.linspace(0.0, 1.0, n) for n in shape]
    grids = np.meshgrid(*axes, indexing='ij')
    vp = 1.5 + 0.6 * grids[-1] + 0.2 * np.sin(2.5 * grids[0])
    rho = 1.0 + 0.8 * grids[-1] ** 2 + 0.3 * np.cos(3.0 * grids[0])
    if len(shape) == 3:
        vp = vp + 0.15 * np.cos(2.0 * grids[1])
        rho = rho + 0.25 * np.sin(3.5 * grids[1])
    return vp.astype(np.float32), (1.0 / rho).astype(np.float32)
