"""float64 restatement of `b2_system_forward` (include/b200stencil.h), written from the C ABI's documented semantics and
independent of both the CUDA executor (devito_b200/csrc/b2_api_system.cu) and the plugin that builds its tables
(devito_b200/refplugin.py).

A system is a dict:

    nd, halo            2 or 3 space dimensions; every field has `halo` cells on each side of every axis
    T                   time slots per field (1 = scratch field)
    stages              [(out_field, out_tshift, [(field, tshift, off, coef, cfield), ...][, ext]), ...]
    injections          [dict(sp=sparse, fields=[...], tshift, scale, kind, param), ...]
    interpolations      [dict(sp=sparse, field, tshift), ...]

and a sparse function is dict(data=(nt, npoint), gp=(npoint, nd), w=[(npoint, 2r)] * nd, r, p_m, p_M).

Per time step `time` in [time_m, time_M]:

1. every stage, in order: for each point p of the box [lo, hi] (domain indices; array index p + halo)
       F[out][(time + out_tshift) mod T[out]][p] =
           sum_k coef_k * C[cfield_k][p] * F[field_k][(time + tshift_k) mod T[field_k]][p + off_k]
   where C is an unhaloed coefficient array read at the OUTPUT point (cfield -1 = 1); a stage with `ext` > 0 covers
   [lo - ext, hi + ext] instead (and has no coefficient arrays);
2. every injection: for p in [p_m, p_M], every support cell c of p inside the guard lo - r <= c <= hi + r,
       F[f][(time + tshift) mod T[f]][c] += w(p, c) * data[time][p] * s(c)   for each of its 1..3 fields f,
   s = scale (kind 0), scale * param[c]^2 (kind 1, B2_PARAM_VP) or scale / param[c] (kind 2, B2_PARAM_M), param with
   the fields' allocated layout; only when 0 <= time < nt;
3. every interpolation: data[time][p] = sum over the guarded support of w(p, c) * F[f][(time + tshift) mod T[f]][c]
   (overwritten, for p in [p_m, p_M] only).

`mut` names one deliberate defect, each a kernel bug the tests must be able to see:

    coef_shifted     coefficient read at the tap's shifted point instead of the output point
    coef_no_origin   the box origin dropped from the coefficient index
    tap_slot_out_T   a tap's slot taken modulo the OUTPUT field's slot count
    inject_first     injections run before the stages
    inject_two       only the first two of three injection fields deposited into
    vp_m_swap        the VP and M injection scales exchanged
    interp_tshift1   interpolation reads level time + 1
    swap_xy_2d       x and y tap offsets exchanged on 2-D grids
    guard_narrow     the sparse guard narrowed to lo - (r - 1) .. hi + (r - 1)
"""
import numpy as np

MUTATIONS = ('coef_shifted', 'coef_no_origin', 'tap_slot_out_T', 'inject_first', 'inject_two', 'vp_m_swap',
             'interp_tshift1', 'swap_xy_2d', 'guard_narrow')


class Support:
    """Valid support cells (array indices) of the points p_m..p_M, their weights and point ids."""

    def __init__(self, sp, lo, hi, halo, guard=None):
        gp = np.asarray(sp['gp'], dtype=np.int64)
        nd = gp.shape[1]
        r = int(sp['r'])
        g = r if guard is None else guard
        pts = np.arange(int(sp['p_m']), int(sp['p_M']) + 1)
        k = np.arange(2 * r) - r + 1
        shape = (len(pts),) + (2 * r,) * nd

        def axis(a, d):
            return a[(slice(None),) + tuple(slice(None) if e == d else None for e in range(nd))]
        C = [np.broadcast_to(axis(gp[pts, d, None] + k[None, :], d), shape) for d in range(nd)]
        W = np.ones(shape)
        for d in range(nd):
            W = W * axis(np.asarray(sp['w'][d], dtype=np.float64)[pts], d)
        ok = np.ones(shape, dtype=bool)
        for d in range(nd):
            ok &= (C[d] >= lo[d] - g) & (C[d] <= hi[d] + g)
        self.idx = tuple(C[d][ok] + halo for d in range(nd))
        self.w = W[ok]
        self.p = np.broadcast_to(pts.reshape((-1,) + (1,) * nd), shape)[ok]
        self.pts = pts


def run(system, fields, coefs, lo, hi, time_m, time_M, traces=None, mut=None):
    """fields: list of (T_f,) + alloc arrays (copied to float64); coefs: list of unhaloed arrays; traces: the data
    arrays of the sparse functions, by id (default: their `data`, copied). Returns (fields, traces)."""
    assert mut is None or mut in MUTATIONS, mut
    nd, h = system['nd'], system['halo']
    T = [int(t) for t in system['T']]
    F = [np.array(f, dtype=np.float64) for f in fields]
    C = [np.asarray(c, dtype=np.float64) for c in coefs]
    box = tuple(slice(l + h, u + h + 1) for l, u in zip(lo, hi))
    cbox = tuple(slice(l, u + 1) for l, u in zip(lo, hi))
    if mut == 'coef_no_origin':
        cbox = tuple(slice(0, u - l + 1) for l, u in zip(lo, hi))
    Cpad = [np.pad(c, h) for c in C] if mut == 'coef_shifted' else None
    sparse = {}
    for q in list(system['injections']) + list(system['interpolations']):
        sparse.setdefault(id(q['sp']), q['sp'])
    out_tr = {k: np.array(s['data'], dtype=np.float64) for k, s in sparse.items()}
    if traces is not None:
        out_tr.update({k: np.array(v, dtype=np.float64) for k, v in traces.items()})
    sup = {k: Support(s, lo, hi, h, guard=(int(s['r']) - 1 if mut == 'guard_narrow' else None))
           for k, s in sparse.items()}

    def stages(time):
        for out, ots, taps, *ext in system['stages']:
            e = ext[0] if ext else 0
            sbox = tuple(slice(b.start - e, b.stop + e) for b in box)
            acc = 0.0
            for f, ts, off, coef, cf in taps:
                assert e == 0 or cf < 0, "a widened stage has no coefficient arrays"
                off = tuple(int(o) for o in off)
                if mut == 'swap_xy_2d' and nd == 2:
                    off = (off[1], off[0])
                slot = (time + ts) % (T[out] if mut == 'tap_slot_out_T' else T[f]) % T[f]
                src = F[f][slot][tuple(slice(b.start + o, b.stop + o) for b, o in zip(sbox, off))]
                if cf < 0:
                    c = 1.0
                elif mut == 'coef_shifted':
                    c = Cpad[cf][tuple(slice(b.start + o, b.stop + o) for b, o in zip(box, off))]
                else:
                    c = C[cf][cbox]
                acc = acc + coef * c * src
            F[out][(time + ots) % T[out]][sbox] = acc

    def injections(time):
        for q in system['injections']:
            s, sp = sup[id(q['sp'])], q['sp']
            data = out_tr[id(sp)]
            if not 0 <= time < data.shape[0]:
                continue
            kind = int(q['kind'])
            if mut == 'vp_m_swap' and kind in (1, 2):
                kind = 3 - kind
            if kind == 0:
                sc = float(q['scale'])
            elif kind == 1:
                sc = float(q['scale']) * np.asarray(q['param'], dtype=np.float64)[s.idx] ** 2
            else:
                sc = float(q['scale']) / np.asarray(q['param'], dtype=np.float64)[s.idx]
            val = s.w * data[time, s.p] * sc
            flds = list(q['fields'])
            if mut == 'inject_two' and len(flds) == 3:
                flds = flds[:2]
            for f in flds:
                np.add.at(F[f][(time + int(q['tshift'])) % T[f]], s.idx, val)

    def interpolations(time):
        for q in system['interpolations']:
            s, sp = sup[id(q['sp'])], q['sp']
            data = out_tr[id(sp)]
            if not 0 <= time < data.shape[0]:
                continue
            ts = 1 if mut == 'interp_tshift1' else int(q['tshift'])
            f = q['field']
            v = F[f][(time + ts) % T[f]][s.idx]
            data[time, s.pts] = np.bincount(s.p - s.pts[0], weights=s.w * v, minlength=len(s.pts)) \
                if len(s.pts) else 0.0
    for time in range(time_m, time_M + 1):
        if mut == 'inject_first':
            injections(time)
        stages(time)
        if mut != 'inject_first':
            injections(time)
        interpolations(time)
    return F, out_tr


# ---------------------------------------------------------------------------------------------------------------
# the fixtures of oracle/make_golden_system.py
# ---------------------------------------------------------------------------------------------------------------
def from_fixture(g):
    """(system, zero fields, coefficient arrays, lo, hi, time_m, time_M) of a `sys_*` fixture."""
    nd = int(g['nd'])
    sps = []
    for i in range(int(g['nsparse'])):
        sps.append(dict(data=g[f'sp{i}_data'], gp=g[f'sp{i}_gp'], w=[g[f'sp{i}_w{d}'] for d in range(nd)],
                        r=int(g[f'sp{i}_r']), p_m=int(g[f'sp{i}_pm']), p_M=int(g[f'sp{i}_pM'])))
    stages, k = [], 0
    for out, ts, n, ext in zip(g['stage_out'], g['stage_tshift'], g['stage_ntaps'], g['stage_ext']):
        taps = [(int(g['tap_field'][j]), int(g['tap_tshift'][j]), tuple(int(o) for o in g['tap_off'][j]),
                 float(g['tap_coef'][j]), int(g['tap_cfield'][j])) for j in range(k, k + int(n))]
        stages.append((int(out), int(ts), taps, int(ext)))
        k += int(n)
    inj = [dict(sp=sps[int(s)], fields=[int(f) for f in fl[:int(nf)]], tshift=int(ts), scale=float(sc), kind=int(kd),
                param=None)
           for s, fl, nf, ts, sc, kd in zip(g['inj_sparse'], g['inj_fields'], g['inj_nfields'], g['inj_tshift'],
                                            g['inj_scale'], g['inj_kind'])]
    itp = [dict(sp=sps[int(s)], field=int(f), tshift=int(ts))
           for s, f, ts in zip(g['itp_sparse'], g['itp_field'], g['itp_tshift'])]
    T = [int(t) for t in g['T']]
    system = dict(nd=nd, halo=int(g['halo']), T=T, stages=stages, injections=inj, interpolations=itp)
    alloc = tuple(int(a) for a in g['alloc'])
    fields = [np.zeros((t,) + alloc, dtype=np.float32) for t in T]
    coefs = list(g['coefs'])
    return system, fields, coefs, tuple(int(x) for x in g['lo']), tuple(int(x) for x in g['hi']), \
        int(g['time_m']), int(g['time_M'])


def fixture_outputs(g, system, F, traces):
    """(last level written of every reference field, domain only and subsampled like the fixture, traces in
    interpolation order) of an interpreter or executor run on a fixture."""
    nd, h, sub = system['nd'], system['halo'], int(g['ref_sub'])
    last = (int(g['time_M']) + 1) % 2
    sl = tuple(slice(h, -h, sub) for _ in range(nd))
    nref = len(g['field_names'])
    fl = np.stack([np.asarray(F[i])[last % system['T'][i]][sl] for i in range(nref)])
    tr = [np.asarray(traces[id(q['sp'])]) for q in system['interpolations']]
    return fl, tr
