"""The float64 reference (tests/ref64.py) against the float32 C oracle, and proof that the kernel-matrix inputs
can fail a wrong kernel. CPU only.

1. Pin: for every case of the GPU kernel matrix, ref64 and `oracle.iso_forward` / `oracle.tti_forward` (two
   independent restatements, per-axis weights, update box) agree to rel L-inf 1e-5 (iso) / 1e-4 (TTI). TTI at
   so=12 and so=16 has no golden fixture: this agreement is its pin.
2. Sensitivity: every mutation of ref64.MUTATIONS that applies to a case moves the result by at least 100x the GPU
   tolerance of that case. A kernel with that kind of bug therefore fails tests/test_kernel_matrix.py whatever
   else it does. What float32 cannot resolve is not claimed: a mistake confined to the outermost tap at so=16
   (w8/w0 ~ 1e-6) is below float32 resolution, and no mutation here is of that kind.
"""
import numpy as np
import pytest

from oracle import oracle as O
from helpers import rel_linf
import kernel_cases as KC
import ref64

ISO = [(so, p) for so in (4, 8, 12, 16) for p in ('scalar', 'vp', 'm')]
TTI = [(so, arrays) for so in (4, 8, 12, 16) for arrays in (False, True)]


def _iso_oracle(c, src=None, rec=None):
    _, w32 = KC.weights('iso', c['so'])
    kind, pv = c['param']
    pk = 0 if np.ndim(pv) == 0 else (1 if kind == 'vp' else 2)
    u = c['u'].copy()
    O.iso_forward(u, c['so'], w32, c['dt'], 1, KC.K, damp=c['damp'], vp=float(pv) if pk == 0 else 1.0,
                  param=pv if pk else None, param_kind=pk, lo=c['lo'], hi=c['hi'], src=src, rec=rec)
    return (u,)


def _tti_oracle(c):
    _, (w2, w1) = KC.weights('tti', c['so'])
    P = c['params']
    arrays = {n: x for n, x in P.items() if np.ndim(x)}
    sc = {n: (1.0 if n == 'vp' else 0.0) if np.ndim(x) else float(x) for n, x in P.items()}
    u, v = c['u'].copy(), c['v'].copy()
    O.tti_forward(u, v, c['so'], w2, w1, c['dt'], 1, KC.K, c['damp'], sc['vp'], sc['epsilon'], sc['delta'],
                  sc['theta'], sc['phi'], lo=c['lo'], hi=c['hi'], arrays=arrays)
    return (u, v)


def _case_mutations(c):
    arrays = (c['kind'] == 'iso' and np.ndim(c['param'][1]) > 0) or \
             (c['kind'] == 'tti' and any(np.ndim(x) for x in c['params'].values()))
    out = ['w_xy', 'w_yz', 'transpose_xy', 'halo_zero', 'tail_y', 'tail_z', 'swap_levels']
    # a partial last float4 group exists where the TMA sweeps take the layout (z extent of the allocation and z_m
    # multiples of 4) and the box's z extent is not a multiple of 4
    if c['shape'][2] % 4 == 0 and c['lo'][2] % 4 == 0 and (c['hi'][2] - c['lo'][2] + 1) % 4:
        out += ['tail_z_over', 'tail_z_short']
    if arrays:
        out += ['shift_x', 'shift_y', 'shift_z']
        if c['kind'] == 'tti':
            out.append('c_at_output')
    return out


def _distance(a, b):
    return max(rel_linf(x, y) for x, y in zip(a, b))


def _check(c, oracle_fields, unclaimed=()):
    tol = KC.TOL[c['kind']]
    ref, _ = KC.reference(c)
    assert np.abs(ref[0]).max() > 0.5
    err = _distance(oracle_fields, ref)
    assert err < tol, f"oracle vs float64: {err:.2e}"
    for mut in [m for m in _case_mutations(c) if m not in unclaimed]:
        moved = _distance(KC.reference(c, mut=mut)[0], ref)
        assert moved >= 100 * tol, f"mutation {mut!r} moves the result by only {moved:.2e}"


@pytest.mark.parametrize('so,param', ISO)
def test_iso_reference_matches_oracle_and_mutations_show(so, param):
    c = KC.iso_case(so, param)
    _check(c, _iso_oracle(c))


def _outside_the_box_nothing_moves(c):
    lo, hi, so = c['lo'], c['hi'], c['so']
    ref, _ = KC.reference(c)
    keep = np.ones(ref[0].shape[1:], dtype=bool)
    keep[tuple(slice(l + so, h + so + 1) for l, h in zip(lo, hi))] = False
    for got, name in zip(ref, ('u', 'v')):
        assert np.array_equal(got[:, keep], c[name][:, keep].astype(np.float64))


@pytest.mark.parametrize('name', ['subbox', 'nz67', 'zm3'] + list(KC.ZTAIL))
def test_iso_reference_boxes_and_fallback_shapes(name):
    """The boxes of the sub-box and fallback GPU cases: an interior box (z_m % 4 == 0), nz % 4 != 0, z_m = 3; and the
    z-tail boxes (z extent 1, 2 or 3 past a multiple of 4), whose mutations include the partial float4 group."""
    if name == 'subbox':
        c = KC.iso_case(8, 'vp', box=KC.SUBBOX)
    elif name == 'nz67':
        c = KC.iso_case(8, 'vp', shape=(37, 45, 67))
    elif name == 'zm3':
        c = KC.iso_case(8, 'vp', box=((0, 0, 3), (36, 44, 67)))
    else:
        c = KC.iso_case(8, 'vp', box=KC.ZTAIL[name])
        assert {'tail_z_over', 'tail_z_short'} <= set(_case_mutations(c))
    _check(c, _iso_oracle(c))
    _outside_the_box_nothing_moves(c)


@pytest.mark.parametrize('so,arrays', TTI)
def test_tti_reference_matches_oracle_and_mutations_show(so, arrays):
    c = KC.tti_case(so, arrays)
    _check(c, _tti_oracle(c))


@pytest.mark.parametrize('arrays', [False, True], ids=['scalar', 'arrays'])
@pytest.mark.parametrize('name', list(KC.ZTAIL))
def test_tti_reference_z_tail_boxes(name, arrays):
    """TTI on the z-tail boxes: pinned against the oracle, every mutation (the partial float4 group's included) far
    above the tolerance, and nothing outside the box moves."""
    c = KC.tti_case(8, arrays, box=KC.ZTAIL[name])
    assert {'tail_z_over', 'tail_z_short'} <= set(_case_mutations(c))
    # an interior box reads the halo only with the outer taps in x and y: a halo read as zero moves TTI by ~5e-3
    # there, below 100x the tolerance; face3 (and the whole-grid cases) claim it
    _check(c, _tti_oracle(c), unclaimed=('halo_zero',) if name != 'face3' else ())
    _outside_the_box_nothing_moves(c)


@pytest.mark.parametrize('kind', ['iso', 'tti'])
def test_tail_mutations_change_only_the_tail(kind):
    """One step on the z-tail boxes: tail_z_over moves exactly the 4 - n2 % 4 points past z_M of every row of the box,
    tail_z_short exactly its last n2 % 4 points."""
    for lo, hi in KC.ZTAIL.values():
        c = KC.iso_case(4, 'vp', box=(lo, hi)) if kind == 'iso' else KC.tti_case(4, False, box=(lo, hi))
        so, r = c['so'], (hi[2] - lo[2] + 1) % 4
        fields = ('u',) if kind == 'iso' else ('u', 'v')
        out = {}
        for mut in (None, 'tail_z_over', 'tail_z_short'):
            if kind == 'iso':
                f = ref64.iso_forward(c['u'], so, KC.weights('iso', so)[0], c['dt'], 1, 1, damp=c['damp'],
                                      param=c['param'], lo=lo, hi=hi, mut=mut)[:1]
            else:
                (w2, w1), _ = KC.weights('tti', so)
                f = ref64.tti_forward(c['u'], c['v'], so, w2, w1, c['dt'], 1, 1, c['damp'], c['params'], lo=lo,
                                      hi=hi, mut=mut)[:2]
            out[mut] = [x[2] for x in f]                                     # the slot written by time 1
        xy = tuple(slice(l + so, h + so + 1) for l, h in zip(lo[:2], hi[:2]))
        zover = slice(hi[2] + 1 + so, hi[2] + 1 + so + 4 - r)
        zshort = slice(hi[2] + 1 + so - r, hi[2] + 1 + so)
        for i, _ in enumerate(fields):
            base = out[None][i]
            for mut, zs in (('tail_z_over', zover), ('tail_z_short', zshort)):
                moved = out[mut][i] != base
                assert moved[xy + (zs,)].all(), mut
                moved[xy + (zs,)] = False
                assert not moved.any(), mut


def test_kernel_case_tilings():
    """The tilings the kernel_cases comments claim: (y tiles, z tiles), (last y tile, last z tile) per (TY, TZ)."""
    assert set(KC.TILES.values()) == {(32, 64), (16, 128), (16, 64), (8, 64), (28, 64), (24, 64), (30, 64), (20, 64)}
    claims = {
        ('MULTI', (16, 128)): ((3, 3), (12, 44)), ('MULTI', (32, 64)): ((2, 5), (12, 44)),
        ('MULTI', (16, 64)): ((3, 5), (12, 44)), ('MULTI', (8, 64)): ((6, 5), (4, 44)),
        ('MULTI_TAIL', (16, 128)): ((3, 3), (12, 42)),
        ('EXACT', (16, 128)): ((2, 2), (16, 128)), ('EXACT', (32, 64)): ((1, 4), (32, 64)),
        ('EXACT', (16, 64)): ((2, 4), (16, 64)), ('EXACT', (8, 64)): ((4, 4), (8, 64)),
    }
    n = {'MULTI': KC.MULTI, 'MULTI_TAIL': KC.box_extent(KC.MULTI_TAIL), 'EXACT': KC.EXACT}
    for (name, (ty, tz)), want in claims.items():
        (ky, ly), (kz, lz) = KC.tiling(n[name][1], ty), KC.tiling(n[name][2], tz)
        assert ((ky, kz), (ly, lz)) == want, (name, ty, tz)
    # every iso tile: MULTI cuts >= 2 y tiles and >= 3 z tiles, the last of each partial; EXACT only full tiles
    for name, (ty, tz) in KC.TILES.items():
        if name.startswith('iso_tma'):
            (ky, ly), (kz, lz) = KC.tiling(KC.MULTI[1], ty), KC.tiling(KC.MULTI[2], tz)
            assert ky >= 2 and kz >= 3 and ly < ty and lz < tz, name
            assert KC.EXACT[1] % ty == 0 and KC.EXACT[2] % tz == 0, name
    # the z-tail boxes: a partial last float4 group of 1, 2, 3 and 3 points, z_m % 4 == 0
    for name, want in (('tail1', 1), ('tail2', 2), ('tail3', 3), ('face3', 3)):
        lo, hi = KC.ZTAIL[name]
        assert lo[2] % 4 == 0 and KC.box_extent((lo, hi))[2] % 4 == want, name
    assert KC.box_extent(KC.ZTAIL['face3']) == (37, 45, 67) and KC.ZTAIL['face3'][0] == (0, 0, 0)
    lo, hi = KC.XPLANE
    assert lo[0] == hi[0] and lo[2] % 4 == 0 and KC.box_extent(KC.XPLANE)[2] % 4 == 3
    # the size gate (n[1] >= 8 and n[2] >= 16): in, out in y, out in z
    assert [KC.box_extent(KC.GATE[g]) for g in ('gate_in', 'gate_y', 'gate_z')] == [(8, 8, 16), (8, 7, 16), (8, 8, 12)]
    assert [KC.box_extent(b) for b in KC.TINY.values()] == [(1, 1, 1), (1, 1, 4), (2, 5, 7)]
    for lo, hi in KC.BOXES.values():
        assert lo[2] % 4 == 0 and all(0 <= l <= h < n for l, h, n in zip(lo, hi, KC.SHAPE))


@pytest.mark.parametrize('param', ['vp', 'm'])
@pytest.mark.parametrize('interpolation', ['linear', 'sinc'])
def test_sparse_reference_matches_oracle(param, interpolation):
    """Injection and interpolation at the faces, outside the domain and two points in one cell."""
    c = KC.iso_case(8, param)
    coords = KC.sparse_coordinates()
    src = KC.sparse_tables(coords, interpolation, KC.K + 2)
    rec = dict(src, data=np.zeros_like(src['data']))
    ref, tr = KC.reference(c, src=src, rec=rec)
    orec = dict(rec, data=rec['data'].copy())
    fields = _iso_oracle(c, src=src, rec=orec)
    assert _distance(fields, ref) < KC.TOL['iso']
    assert rel_linf(orec['data'], tr) < KC.TOL['iso']
    # the sources matter: without them the wavefield differs far beyond the tolerance (near the faces too)
    bare, _ = KC.reference(c, rec=rec)
    assert _distance(bare, ref) > 100 * KC.TOL['iso']
    # the point far outside has no support cell; every other point samples something
    far = 12
    assert not tr[1:KC.K + 1, far].any()
    assert np.all(np.abs(np.delete(tr[1:KC.K + 1], far, axis=1)).max(axis=0) > 0)
    # the halo was written: sources outside the domain deposit into it
    so = c['so']
    dom = np.zeros(ref[0].shape[1:], dtype=bool)
    dom[so:-so, so:-so, so:-so] = True
    assert np.abs(ref[0][:, ~dom] - bare[0][:, ~dom]).max() > 0


# ---------------------------------------------------------------------------------------------------------------
# The schemes built on the iso update: adjoint, free surface, OT4, imaging condition, Born, snapshots, 2-D.
# Same inputs as the GPU scheme matrix (tests/test_scheme_matrix.py): white noise in every slot and halo, the KC
# sparse points (faces, outside the domain, two in one cell) as sources and receivers.
# ---------------------------------------------------------------------------------------------------------------
OUT_TOL = {'u': 1e-5, 'snap': 1e-5, 'traces': 1e-5, 'U': 1e-4, 'grad': 1e-4}


def _out_tol(c, name):
    return 1e-4 if c['scheme'] == 'born' and name == 'traces' else OUT_TOL[name]


def scheme_sparse(c):
    """sinc points (r = 4) from so = 8 on, linear below; receivers record into zeros."""
    src = KC.sparse_tables(KC.sparse_coordinates(c['shape']), 'sinc' if c['so'] >= 8 else 'linear', KC.K + 2)
    return src, dict(src, data=np.zeros_like(src['data']))


def _scheme_oracle(c, src, rec):
    """float32 C oracle of a scheme case: dict of the outputs it has (no snapshots)."""
    _, w32 = KC.weights('iso', c['so'])
    w32 = w32[3 - len(c['shape']):]
    kind, pv = c['param']
    pk = 0 if np.ndim(pv) == 0 else (1 if kind == 'vp' else 2)
    pkw = dict(damp=c['damp'], vp=float(pv) if pk == 0 else 1.0, param=pv if pk else None, param_kind=pk)
    orec = dict(rec, data=rec['data'].copy()) if rec is not None else None
    u = c['u'].copy()
    s = c['scheme']
    if s == 'born':
        U = c['U'].copy()
        O.born_forward(u, U, c['dm'], c['so'], w32, c['dt'], 1, KC.K, src=src, rec=orec, dmhalo=c['dmh'],
                       lo=c['lo'], hi=c['hi'], **pkw)
        return dict(u=u, U=U, traces=orec['data'])
    out = {}
    kw = {}
    if s == 'grad':
        out['grad'] = c['grad'].copy()
        kw = dict(grad=out['grad'], ghalo=KC.GRAD_HALO, usave=c['usave'])
    O.iso_forward(u, c['so'], w32, c['dt'], 1, KC.K, lo=c['lo'], hi=c['hi'], src=src, rec=orec,
                  adjoint=s in ('adjoint', 'adjoint_fs', 'adjoint_ot4', 'grad'),
                  free_surface=s in ('fs', 'adjoint_fs'), ot4=s in ('ot4', 'adjoint_ot4'), **kw, **pkw)
    out['u'] = u
    if orec is not None:
        out['traces'] = orec['data']
    return out


def scheme_mutations(c):
    """The mutations of ref64.MUTATIONS a kernel of this scheme could have."""
    s = c['scheme']
    arrays = np.ndim(c['param'][1]) > 0
    out = ['w_xy', 'halo_zero', 'swap_levels']
    if len(c['shape']) == 3:
        out += ['w_yz', 'transpose_xy', 'tail_y', 'tail_z']
        if arrays:
            out += ['shift_x', 'shift_y', 'shift_z']
    if s in ('adjoint', 'adjoint_fs', 'adjoint_ot4', 'grad'):
        out.append('adj_inject_level')
    if s in ('fs', 'adjoint_fs'):
        out += ['fs_surface_tap', 'fs_mirror_sign', 'fs_keep_row0']
        # Row z = R differs from the plain update only by its outermost lower tap, w_R u[0], and u[0] is non-zero
        # only in the initial level and where a source deposited into the surface row. At so = 8 that moves u by
        # about 4x the tolerance (w_4 / w_0 = 1/1594), so the mutation is claimed at so = 4 only.
        if c['so'] == 4:
            out.append('fs_rows_lt_R')
    if s in ('ot4', 'adjoint_ot4'):
        out.append('ot4_factor')
        if arrays:
            out.append('ot4_m_at_output')           # with a scalar m the two places hold the same value
    if s == 'born':
        out += ['born_before_inject', 'born_dm_shift']
    if s == 'grad':
        out += ['grad_usave_time', 'grad_assign', 'grad_halo']
    if s in ('snap', 'snap_fwd'):
        out += ['snap_level', 'snap_index']
    return out


def scheme_distance(c, got, want):
    """max over the outputs of rel L-inf / that output's tolerance (1 = at the tolerance)."""
    return max(rel_linf(got[k], want[k]) / _out_tol(c, k) for k in want if want[k] is not None)


def _check_scheme(c, sparse=True, oracle=True):
    src, rec = scheme_sparse(c) if sparse else (None, None)
    ref = KC.scheme_reference(c, src=src, rec=rec)
    assert np.abs(ref['u']).max() > 0.5
    if oracle:
        got = _scheme_oracle(c, src, rec)
        for k, v in got.items():
            err = rel_linf(v, ref[k])
            assert err < _out_tol(c, k), f"oracle vs float64, {k}: {err:.2e}"
    for mut in scheme_mutations(c):
        moved = scheme_distance(c, KC.scheme_reference(c, src=src, rec=rec, mut=mut), ref)
        assert moved >= 100, f"mutation {mut!r} moves the result by only {moved:.0f}x the tolerance"
    return ref


SCHEME_CASES = [(s, so, p, b) for s in ('adjoint', 'ot4', 'grad', 'born')
                for so in (4, 8, 16) for p in ('scalar', 'vp', 'm') for b in ('full', 'sub')] + \
               [(s, so, p, 'full') for s in ('fs', 'adjoint_fs', 'adjoint_ot4') for so in (4, 8, 16)
                for p in ('scalar', 'vp', 'm')]


@pytest.mark.parametrize('scheme,so,param,box', SCHEME_CASES)
def test_scheme_reference_matches_oracle_and_mutations_show(scheme, so, param, box):
    c = KC.scheme_case(scheme, so, param, box=KC.SUBBOX if box == 'sub' else None, dmh=3 if so == 8 else 0)
    _check_scheme(c)


@pytest.mark.parametrize('scheme', ['snap', 'snap_fwd'])
@pytest.mark.parametrize('box', ['full', 'sub'])
def test_snapshot_reference_mutations_show(scheme, box):
    """Snapshots have no oracle counterpart (a plain copy): the mutation distances are their check here, and the
    cells the reference leaves alone keep the sentinel."""
    c = KC.scheme_case(scheme, 8, 'vp', box=KC.SUBBOX if box == 'sub' else None)
    ref = _check_scheme(c, oracle=False)
    snap = ref['snap']
    visited = np.zeros(snap.shape, dtype=bool)
    sh = KC.SNAP_HALO
    for time in range(1, KC.K + 1):
        if time % KC.SNAP_FACTOR == 0:
            visited[(time // KC.SNAP_FACTOR,) + tuple(slice(l + sh, h + sh + 1) for l, h in zip(c['lo'], c['hi']))] = True
    assert np.all(snap[~visited] == KC.SNAP_SENTINEL) and not np.any(snap[visited] == KC.SNAP_SENTINEL)


@pytest.mark.parametrize('scheme', ['plain', 'fs'])
@pytest.mark.parametrize('param', ['scalar', 'vp'])
def test_2d_reference_matches_oracle_and_mutations_show(scheme, param):
    """2-D (45, 68), spacing (12.5, 8): the plain update and the free surface on the last axis."""
    c = KC.scheme_case(scheme, 8, param, shape=KC.SHAPE[1:])
    _check_scheme(c, sparse=False)
