"""float64 restatement of the second-order SLS viscoacoustic update (reference: examples/seismic/viscoacoustic/
operators.py `sls_2nd_order`, `ForwardOperator`, `AdjointOperator` at kernel='sls', time_order=2), in the conventions
of tests/ref64.py (allocated layout with a halo of `so`, inclusive box `lo` .. `hi` in domain indices, the halo read
as stored). It is written from the equations, not from the kernels' tables:

  t_s = (sqrt(1 + 1/qp^2) - 1/qp) / f0,  t_ep = 1 / (f0^2 t_s),  tt = t_ep / t_s - 1,  m = 1/vp^2,  rho = 1/b
  L(f) = sum_d D-_d (b D+_d f)            the nested operator of tests/sa_ref.py (b at the nodes)
  e    = (1 - damp) / dt

`r.dt` and `p.dt` are the reference's first-order forward differences (f[t+1] - f[t]) / dt, whose transposes `.dt.T`
are (f[t-1] - f[t]) / dt, whatever the time order of the field; solved for the level written:

  forward  r[t+1] = damp (r[t] + dt ((tt/t_s) rho L(p[t]) - r[t]/t_s))
           p[t+1] = damp (rho (1+tt) L(p[t]) - r[t+1] + m (2 p[t] - p[t-1]) / dt^2 + e p[t]) / (m/dt^2 + e)
  adjoint  r[t-1] = damp (r[t] - dt ((tt/t_s) p[t] + r[t]/t_s))                       on the box
           p[t-1] = damp (L(rho (1+tt) p[t]) + L(rho r[t-1]) + m (2 p[t] - p[t+1]) / dt^2 + e p[t]) / (m/dt^2 + e)

The source is injected into the level written with the scale dt^2 / m at the cell; the receivers sample p[t] (the
written level with rec_toff).

`mut` selects one deliberate mistake from MUTATIONS; the sensitivity tests show each moves the answer far above the
tolerance.
"""
import numpy as np

from ref64 import _Support, _at, _bounds, _box
from sa_ref import _div, sa_weights  # noqa: F401  (sa_weights: the same half-node weights)

MUTATIONS = {
    'b_at_output': "b taken at the output point instead of at the flux nodes",
    'b_half_node': "b averaged to the half node instead of sampled at the node",
    'no_rho': "the factor rho = 1/b in front of L(p) left out",
    'tt_ts_swap': "tt and 1/t_s exchanged in the memory-variable update",
    'r_at_t': "the pressure update reads r[t] instead of the level r[t+1] just written",
    'damp_added': "damp added to the solved update (x + damp - 1) instead of multiplying it",
    'last_z_group': "the last four points of the box along z (one float4 group) not updated",
}


def relaxation(qp, f0):
    """(t_s, tt) of the reference's sls kernels."""
    qp = np.asarray(qp, dtype=np.float64)
    t_s = (np.sqrt(1.0 + 1.0 / qp ** 2) - 1.0 / qp) / f0
    t_ep = 1.0 / (f0 ** 2 * t_s)
    return t_s, t_ep / t_s - 1.0


def visco_forward(p, r, so, c, dt, f0, time_m, time_M, b, vp, qp, damp=None, lo=None, hi=None, src=None, rec=None,
                  rec_toff=0, adjoint=False, mut=None):
    """Time steps of the SLS update (3-D or 2-D). `b`, `vp`, `qp`: scalars or arrays in p's space layout; `damp`: an
    array or None (1). Returns (p, r, traces) in float64; the inputs are not modified."""
    p = np.array(p, dtype=np.float64)
    r = np.array(r, dtype=np.float64)
    T = p.shape[0]
    lo, hi = _bounds(p.shape[1:], so, lo, hi)
    c = [np.asarray(x, dtype=np.float64) for x in c]
    shape = p.shape[1:]
    full = lambda x: np.broadcast_to(np.asarray(x, dtype=np.float64), shape)
    b, vp, qp = full(b), full(vp), full(qp)
    dm = full(1.0 if damp is None else damp)
    t_s, tt = relaxation(qp, f0)
    if mut == 'tt_ts_swap':
        t_s, tt = 1.0 / tt, 1.0 / t_s
    m = 1.0 / vp ** 2
    rho = 1.0 / b
    box = _box(lo, hi, so)
    at = lambda x: _at(x, box)
    e = (1.0 - dm) / dt
    den = at(m / dt ** 2 + e)
    dmask = (lambda x: x + at(dm) - 1.0) if mut == 'damp_added' else (lambda x: at(dm) * x)
    lmut = mut if mut in ('b_at_output', 'b_half_node') else None
    L = lambda f: _div(f, b, c, c, lo, hi, so, lmut)
    S = _Support(src, lo, hi, so) if src is not None else None
    R_ = _Support(rec, lo, hi, so) if rec is not None else None
    traces = np.array(rec['data'], dtype=np.float64) if rec is not None else None
    dirn = -1 if adjoint else 1
    times = range(time_M, time_m - 1, -1) if adjoint else range(time_m, time_M + 1)
    for time in times:
        t0, t1, t2 = time % T, (time + dirn) % T, (time - dirn) % T
        old_p1, old_r1 = p[t1][box].copy(), r[t1][box].copy()
        if not adjoint:
            Lp = L(p[t0])
            rho_ = 1.0 if mut == 'no_rho' else at(rho)
            r[t1][box] = dmask(at(r[t0]) + dt * (at(tt / t_s) * rho_ * Lp - at(r[t0]) / at(t_s)))
            rr = r[t0][box] if mut == 'r_at_t' else r[t1][box]
            rhs = rho_ * at(1.0 + tt) * Lp - rr
        else:
            r[t1][box] = dmask(at(r[t0]) - dt * (at(tt / t_s) * at(p[t0]) + at(r[t0]) / at(t_s)))
            rr = r[t0] if mut == 'r_at_t' else r[t1]
            rho_ = 1.0 if mut == 'no_rho' else rho
            rhs = L(rho_ * (1.0 + tt) * p[t0]) + L(rho_ * rr)
        p[t1][box] = dmask((rhs + at(m) * (2.0 * at(p[t0]) - at(p[t2])) / dt ** 2 + at(e) * at(p[t0])) / den)
        if mut == 'last_z_group':
            p[t1][box][..., -4:] = old_p1[..., -4:]
            r[t1][box][..., -4:] = old_r1[..., -4:]
        if S is not None:
            S.inject([p[t1]], time, dt * dt * vp * vp)
        if R_ is not None:
            R_.interpolate(traces, [p[t1] if rec_toff else p[t0]], time)
    return p, r, traces


def smooth_vp_b_qp(shape):
    """vp, b = 1/rho and qp of the reference goldens (oracle/make_golden_visco.py builds them with the same
    formula)."""
    from sa_ref import smooth_vp_b
    vp, b = smooth_vp_b(shape)
    axes = [np.linspace(0.0, 1.0, n) for n in shape]
    grids = np.meshgrid(*axes, indexing='ij')
    qp = 30.0 + 40.0 * grids[-1] + 10.0 * np.sin(2.0 * grids[0])
    if len(shape) == 3:
        qp = qp + 8.0 * np.cos(3.0 * grids[1])
    return vp, b, qp.astype(np.float32)
