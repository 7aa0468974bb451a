"""The two-level isotropic pass (`iso_tma2<4,scalar>`, b2_iso.cu::k_iso_tma2, DESIGN.md §3.7) against the float64
reference (tests/ref64.py), on the machinery tests/test_iso_two_level.py leaves alone:

1. absorbing-layer damping, so that nearly every x-plane takes A from the pinned tile in both levels, with perturbed
   planes that put every pinned/streamed switch at the offsets level 2's R-plane lag reads;
2. the in-kernel injection table: 64 entries with shared deposits and face-touching supports, one sinc r=2 support
   across a y-tile, z-tile and x-chunk corner, 72 entries (the one-step loop), supports one cell outside each face of
   the box (the one-step loop), no source, and traces that end at time_M;
3. time ranges of one to four passes, time_m = 0, and a run handed between the two loops across calls;
4. the size-gate box, a box one x-plane thick, a grid of whole tiles only, and x-chunks shorter than R and 4R;
5. the scratch slots' "zero outside the box" across calls that change the box, and the extents at one slot size;
6. the automatic selection: either side of the 1 GiB threshold, bit equality with `k_iso_tma` above it, and the
   configurations that must never take the pass.

Every case loads white noise into u inside the update box (zero elsewhere), compares all three time slots, halo
included, and the receiver traces with float64, and asserts which sweep kernel ran. The grid (70, 45, 148) with the
spacing of tests/kernel_cases.py has partial y and z tiles of the pass's 16 x 64 tile (45 = 2*16 + 13,
148 = 2*64 + 20). The CPU twins at the end check, without a GPU, that each case still means what it claims.
"""
import functools
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest

from helpers import rel_linf
import kernel_cases as KC
from oracle import oracle as O
import ref64
from test_iso_coef_reuse import expected_reuse

SO, R = 8, 4
SHAPE = (70, 45, 148)
TSHAPE = (SHAPE[1], SHAPE[0], SHAPE[2])          # transposed in x and y: the same slot size
WHOLE = (40, 32, 128)                            # whole 16 x 64 tiles only
TWO, ONE = 'iso_tma2<4,scalar>', 'iso_tma<4,scalar>'
LX = 32                                          # forced x-chunk length: chunks [0, 32), [32, 64), [64, 70)
NT = 12
DT = float(O.critical_dt(SO, 3, min(KC.SPACING), 2.5))
W64 = [ref64.fd2_weights(SO, h) for h in KC.SPACING]

_CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'devito_b200', 'csrc')


def _constant(path, pattern):
    with open(os.path.join(_CSRC, path)) as f:
        return int(re.search(pattern, f.read()).group(1))


MAX_INJ = _constant('b2_iso.cuh', r'B2_ISO2_MAX_INJ = (\d+);')                 # entries the pass takes
TY = _constant('b2_iso.cu', r'I2TY = (\d+)')                                     # Iso2Cfg's output tile
TZ = 4 * _constant('b2_iso.cu', r'I2TZ4 = (\d+)')


def _full(shape):
    return ((0, 0, 0), tuple(n - 1 for n in shape))


FULL = _full(SHAPE)
SUB = ((2, 3, 4), (SHAPE[0] - 3, SHAPE[1] - 2, SHAPE[2] - 7))   # nz = 138 (a z tail of 2); touches no face of FULL
GATE = ((1, 2, 4), (8, 9, 19))                                     # n = (8, 8, 16): the TMA size gate, one partial tile
XPLANE = ((5, 2, 4), (5, 41, 62))                                  # one x-plane

# Sources, in grid points (the grids' origin is 0). CORNER's support straddles x = 31|32 (an edge of LX = 32
# chunks), y = 15|16 (a y-tile edge) and z = 63|64 (a z-tile edge); SHARED has the same base cell.
CORNER = (31.5, 15.4, 63.6)
SHARED = (31.8, 15.7, 63.2)
# supports touching the lo and hi faces of FULL from inside, one per face: x lo, x hi, y lo, y hi, z lo, z hi
FACES = ((0.3, 20.2, 70.3), (68.6, 25.5, 30.7), (40.2, 0.4, 100.5), (20.7, 43.5, 50.2), (50.5, 30.3, 0.6),
         (10.4, 8.8, 146.3))
POINTS8 = (CORNER, SHARED) + FACES                                 # 64 entries: the most the pass takes
POINTS9 = POINTS8 + ((45.2, 30.6, 100.1),)                         # 72: the one-step loop
SINC = (31.3, 15.6, 63.45)                                         # r = 2: 4^3 = 64 cells, 30..33, 14..17, 62..65
# one support cell one cell outside FULL, per face
OUTSIDE = {'x_lo': (-0.5, 20.2, 70.3), 'x_hi': (69.5, 20.2, 70.3), 'y_lo': (30.2, -0.5, 70.3),
           'y_hi': (30.2, 44.5, 70.3), 'z_lo': (30.2, 20.2, -0.5), 'z_hi': (30.2, 20.2, 147.5)}
# receivers inside both SHAPE and TSHAPE
REC = ((31.5, 15.4, 63.6), (10.2, 40.7, 140.3), (40.9, 3.3, 2.5), (25.0, 30.0, 100.25))
GATE_SRC = (4.3, 5.6, 10.2)                                        # support 4..5, 5..6, 10..11: inside GATE
GATE_REC = (GATE_SRC, (7.5, 8.2, 17.6))
XPLANE_REC = ((5.0, 20.3, 30.6), (5.0, 40.2, 61.5))                # x = 5 exactly: weight 0 on plane 6
WHOLE_SRC = (19.5, 15.5, 63.5)
WHOLE_REC = ((19.5, 15.5, 63.5), (5.2, 28.7, 120.3))

# absorbing-layer damp: x-planes perturbed inside the box's rows, relative to the box's first plane. With LX = 32:
# the first plane of a chunk (32), the last plane of a chunk (63), a run of two (45, 46) and a plane R after
# another perturbed one (50)
LAYER = 4
PERTURBED = (32, 45, 46, 50, 63)

# the u of these grids (3 slots, halo included) lies just below / just above 1 GiB: one x-plane apart
BELOW = (416, 385, 500)
ABOVE = (417, 385, 500)


def _lib():
    from devito_b200 import _lib as L
    return L.lib()


def _kernel():
    return _lib().b2_last_sweep_kernel().decode()


def _coords(pts):
    return (np.array(pts, dtype=np.float64).reshape(-1, 3) * np.array(KC.SPACING)).astype(np.float32)


def _table(pts, interpolation, r, nt, seed):
    """base cells, float64 weights (the oracle's tabulation) and random traces"""
    coords = _coords(pts)
    gp, ws = O.tabulate(coords, (0.0, 0.0, 0.0), KC.SPACING, r, interpolation, dtype=np.float64)
    data = np.random.default_rng(seed).standard_normal((nt, len(coords))).astype(np.float32)
    return dict(data=data, gp=gp, w=ws, r=r)


def _support(pts, r=1, interpolation='linear'):
    """(npoint, (2r)^3, 3) support cells of every point"""
    gp, _ = O.tabulate(_coords(pts), (0.0, 0.0, 0.0), KC.SPACING, r, interpolation)
    off = np.arange(2 * r) - r + 1
    o = np.stack(np.meshgrid(off, off, off, indexing='ij'), axis=-1).reshape(-1, 3)
    return gp.astype(np.int64)[:, None, :] + o[None]


def _inside(cells, box):
    lo, hi = box
    return np.all((cells >= np.array(lo)) & (cells <= np.array(hi)), axis=-1)


def _u_bytes(shape):
    return 3 * 4 * int(np.prod([n + 2 * SO for n in shape]))


@functools.lru_cache(maxsize=None)
def _setup(shape=SHAPE, src=(CORNER,), interpolation='linear', r=1, src_nt=NT, rec=REC, rec_nt=NT, rec_toff=0):
    """u, damp, a Constant vp, `src` injected into u.forward (none if empty) and `rec` interpolated from u (or
    u.forward); one operator per configuration"""
    from devito_b200 import Constant, Eq, Function, Grid, Operator, SparseTimeFunction, TimeFunction, solve
    grid = Grid(shape=shape, extent=tuple((n - 1) * h for n, h in zip(shape, KC.SPACING)))
    u = TimeFunction(name='u', grid=grid, time_order=2, space_order=SO)
    damp = Function(name='damp', grid=grid, space_order=SO)
    m = 1 / Constant(name='vp', value=2.0) ** 2
    dt = grid.stepping_dim.spacing
    eqs = [Eq(u.forward, solve(m * u.dt2 - u.laplace + damp * u.dt, u.forward))]
    stab = None
    if src:
        stab = _table(src, interpolation, r, src_nt, 5)
        s = SparseTimeFunction(name='src', grid=grid, npoint=len(src), nt=src_nt, interpolation=interpolation, r=r,
                               coordinates=_coords(src))
        s.data[:] = stab['data']
        eqs += s.inject(field=u.forward, expr=s * dt ** 2 / m)
    rtab = _table(rec, 'linear', 1, rec_nt, 6)
    rf = SparseTimeFunction(name='rec', grid=grid, npoint=len(rec), nt=rec_nt, interpolation='linear', r=1,
                            coordinates=_coords(rec))
    eqs += rf.interpolate(expr=u.forward if rec_toff else u)
    op = Operator(eqs)
    assert op.backend == 'cuda-sm90a'
    return SimpleNamespace(op=op, u=u, damp=damp, rec=rf, stab=stab, rtab=rtab, shape=shape, rec_toff=rec_toff)


def _noise_u(shape, box, seed):
    """white noise inside the box in all three slots, zero elsewhere"""
    a = tuple(n + 2 * SO for n in shape)
    lo, hi = box
    u = np.zeros((3,) + a, dtype=np.float32)
    sl = tuple(slice(l + SO, h + SO + 1) for l, h in zip(lo, hi))
    u[(slice(None),) + sl] = np.random.default_rng(seed).standard_normal((3,) + KC.box_extent(box))
    return u


def _white_damp(shape, seed):
    a = tuple(n + 2 * SO for n in shape)
    return (0.1 * np.random.default_rng(seed + 1000).uniform(0.0, 1.0, a)).astype(np.float32)


def _profile(n):
    """a ramp over the LAYER points next to each end of the domain, and the halo; zero inside"""
    i = np.arange(n + 2 * SO, dtype=np.float64) - SO
    d = np.maximum(np.maximum(LAYER - i, i - (n - 1 - LAYER)), 0.0) / LAYER
    return (0.08 * d * d).astype(np.float32)


def layered_damp(shape, box, planes=PERTURBED):
    """sum of per-axis profiles (float32, x + y + z), then the box's rows of the x-planes lo[0] + `planes` raised"""
    p = [_profile(n) for n in shape]
    damp = (p[0][:, None, None] + p[1][None, :, None]) + p[2][None, None, :]
    lo, hi = box
    rows = (slice(SO + lo[1], SO + hi[1] + 1), slice(SO + lo[2], SO + hi[2] + 1))
    for x in planes:
        damp[(SO + lo[0] + x,) + rows] += np.float32(1e-3)
    return damp


def _apply(c, box, ranges, monkeypatch, lx=LX, damp=None, seed=1):
    """Load u (white noise in the box) and damp (white noise unless given), then apply each (time_m, time_M[, B2_ISO2])
    range, with B2_ISO2=2 unless the range says otherwise. Returns (u0, damp, the kernel of each apply)."""
    if lx is None:
        monkeypatch.delenv('B2_ISO_LX', raising=False)
    else:
        monkeypatch.setenv('B2_ISO_LX', str(lx))
    u0 = _noise_u(c.shape, box, seed)
    d = _white_damp(c.shape, seed) if damp is None else damp
    c.u.data_with_halo[:] = u0
    c.damp.data_with_halo[:] = d
    c.rec.data[:] = 0.0
    lo, hi = box
    bounds = dict(x_m=lo[0], x_M=hi[0], y_m=lo[1], y_M=hi[1], z_m=lo[2], z_M=hi[2])
    kernels = []
    for rg in ranges:
        monkeypatch.setenv('B2_ISO2', rg[2] if len(rg) > 2 else '2')
        c.op.apply(time_m=rg[0], time_M=rg[1], dt=DT, **bounds)
        kernels.append(_kernel())
    return u0, d, kernels


def _check(c, box, u0, d, time_m, time_M):
    """every slot, halo included, and the traces against one float64 run over time_m .. time_M"""
    lo, hi = box
    rec = dict(c.rtab, data=np.zeros_like(c.rtab['data']))
    want, traces = ref64.iso_forward(u0, SO, W64, DT, time_m, time_M, damp=d, param=('vp', 2.0), lo=lo, hi=hi,
                                     src=c.stab, rec=rec, rec_toff=c.rec_toff)
    got = np.array(c.u.data_ro_with_halo)
    assert np.abs(got).max() > 0.5
    assert rel_linf(got, want) < KC.TOL['iso']
    got_tr = np.array(c.rec.data)
    assert np.abs(traces).max() > 1e-3
    assert rel_linf(got_tr, traces) < KC.TOL['iso']


def _run(c, box, ranges, monkeypatch, **kw):
    u0, d, kernels = _apply(c, box, ranges, monkeypatch, **kw)
    _check(c, box, u0, d, ranges[0][0], ranges[-1][1])
    return kernels


# ---------------------------------------------------------------------------------------------------------------
# 1. Absorbing-layer damping: A from the pinned tile in both levels
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('lx', [None, LX])
@pytest.mark.parametrize('box', ['full', 'sub'])
def test_layered_damp_pins_a_in_both_levels(box, lx, monkeypatch):
    b = {'full': FULL, 'sub': SUB}[box]
    c = _setup()
    d = layered_damp(SHAPE, b)
    assert _run(c, b, [(1, 6)], monkeypatch, lx=lx, damp=d) == [TWO]
    n = expected_reuse(d, SO, *b)
    assert 1 < n < b[1][0] - b[0][0] + 1 - len(PERTURBED)
    assert _lib().b2_last_iso_coef_reuse() == n


# ---------------------------------------------------------------------------------------------------------------
# 2. The injection table
# ---------------------------------------------------------------------------------------------------------------
INJECTION = {
    # name: (setup keywords, time range, kernel)
    'shared_faces_corner_64': (dict(src=POINTS8), (1, 6), TWO),
    'sinc_r2_corner_64': (dict(src=(SINC,), interpolation='sinc', r=2), (1, 6), TWO),
    'linear_72': (dict(src=POINTS9), (1, 6), ONE),
    'no_source': (dict(src=()), (1, 6), TWO),
    # traces as short as `Operator.apply` allows (nt = time_M + 1): the last pass injects and records the last rows
    'tight_traces': (dict(src=POINTS8, src_nt=9, rec_nt=9, rec_toff=1), (1, 8), TWO),
}
INJECTION.update({f'outside_{f}': (dict(src=(p,)), (1, 6), ONE) for f, p in OUTSIDE.items()})


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(INJECTION))
def test_injection_table(case, monkeypatch):
    """Shared deposits are atomics in the one-step loop, in any order: compared with float64 only."""
    kw, rg, expect = INJECTION[case]
    c = _setup(**kw)
    assert _run(c, FULL, [rg], monkeypatch) == [expect]
    if case == 'tight_traces':
        # shorter traces are refused before the call: the entries of a time past the traces are never read
        from devito_b200.exceptions import InvalidArgument
        with pytest.raises(InvalidArgument):
            c.op.apply(time_m=1, time_M=9, dt=DT)


# ---------------------------------------------------------------------------------------------------------------
# 3. Time ranges and the hand-over between the two loops
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('rec_toff', [0, 1])
@pytest.mark.parametrize('rg', [(0, 1), (0, 2), (1, 7), (1, 8)], ids=lambda r: f'{r[0]}-{r[1]}')
def test_time_ranges(rg, rec_toff, monkeypatch):
    """(0, 1): one pass from the wrapped slot -1; (1, 7): one ordinary step, then three passes; (1, 8): four passes,
    the scratch slots turn over twice and both end-of-call copies run."""
    assert _run(_setup(rec_toff=rec_toff), FULL, [rg], monkeypatch) == [TWO]


@pytest.mark.gpu
@pytest.mark.parametrize('rec_toff', [0, 1])
def test_handover_between_loops(rec_toff, monkeypatch):
    """two-level 1..4, one-step 5..6, two-level 7..10 against one float64 run over 1..10: each loop continues from
    the slots the other left"""
    ks = _run(_setup(rec_toff=rec_toff), FULL, [(1, 4), (5, 6, '0'), (7, 10)], monkeypatch)
    assert ks == [TWO, ONE, TWO]


# ---------------------------------------------------------------------------------------------------------------
# 4. Boxes and x-chunks
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize('case', ['gate', 'xplane', 'whole_tiles'])
def test_boxes(case, monkeypatch):
    """gate: one partial tile, smaller than the level-1 region in y and z. xplane: one x-plane (the march primes 4R
    planes for it); no source, since a support spans two x-planes and would reach outside the box. whole_tiles:
    (40, 32, 128), every tile full."""
    c, box = {'gate': (_setup(src=(GATE_SRC,), rec=GATE_REC), GATE),
              'xplane': (_setup(src=(), rec=XPLANE_REC), XPLANE),
              'whole_tiles': (_setup(shape=WHOLE, src=(WHOLE_SRC,), rec=WHOLE_REC), _full(WHOLE))}[case]
    assert _run(c, box, [(1, 6)], monkeypatch) == [TWO]


@pytest.mark.gpu
@pytest.mark.parametrize('lx', [1, 3, 16, 32, None])
def test_x_chunks(lx, monkeypatch):
    """chunks of 1 and 3 planes are shorter than R, 16 is 4R (the march's priming length); None: the chosen one"""
    assert _run(_setup(), FULL, [(1, 6)], monkeypatch, lx=lx) == [TWO]


# ---------------------------------------------------------------------------------------------------------------
# 5. The scratch slots stay zero outside the box across calls
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_scratch_across_box_and_extent_changes(monkeypatch):
    """FULL -> SUB -> FULL on one operator: the scratch slots keep FULL's values where SUB's halo is unless they are
    re-zeroed. Then the transposed grid (same slot size: the allocation is kept, its extents change), then FULL
    again. Four passes per call, so that a later pass reads its u[t] from scratch."""
    c, ct = _setup(), _setup(shape=TSHAPE, src=((20.5, 30.4, 63.6),))
    for seed, (cc, box) in enumerate([(c, FULL), (c, SUB), (ct, _full(TSHAPE)), (c, FULL)]):
        assert _run(cc, box, [(1, 8)], monkeypatch, seed=10 + seed) == [TWO]


# ---------------------------------------------------------------------------------------------------------------
# 6. Automatic selection
# ---------------------------------------------------------------------------------------------------------------
def _big_setup(shape):
    c = _setup.__wrapped__(shape=shape, src=((200.5, 150.4, 255.6),),
                           rec=((200.5, 150.4, 255.6), (30.2, 370.7, 480.3), (400.9, 3.3, 10.5)))
    u0 = np.zeros((3,) + tuple(n + 2 * SO for n in shape), dtype=np.float32)
    u0[(slice(None),) + (slice(SO, -SO),) * 3] = np.random.default_rng(3).standard_normal((3,) + shape,
                                                                                         dtype=np.float32)
    return c, u0, layered_damp(shape, _full(shape), planes=(100, 101, 105))


def _big_apply(c, u0, d, iso2, monkeypatch, time_M=4):
    if iso2 is None:
        monkeypatch.delenv('B2_ISO2', raising=False)
    else:
        monkeypatch.setenv('B2_ISO2', iso2)
    monkeypatch.delenv('B2_ISO_LX', raising=False)
    c.u.data_with_halo[:] = u0
    c.damp.data_with_halo[:] = d
    c.rec.data[:] = 0.0
    c.op.apply(time_m=1, time_M=time_M, dt=DT)
    return _kernel()


@pytest.mark.gpu
def test_auto_selection_below_one_gib(monkeypatch):
    assert _u_bytes(BELOW) < 2 ** 30
    c, u0, d = _big_setup(BELOW)
    assert _big_apply(c, u0, d, None, monkeypatch, time_M=2) == ONE
    assert _big_apply(c, u0, d, '2', monkeypatch, time_M=2) == TWO       # nothing else keeps the pass out


@pytest.mark.gpu
def test_auto_selection_above_one_gib_is_bit_exact(monkeypatch):
    """The chosen chunk length, pinned planes, one source and receivers: the pass gives the one-step kernel's bits
    (DESIGN.md §3.7: the arithmetic and its order are unchanged)."""
    assert _u_bytes(ABOVE) >= 2 ** 30
    c, u0, d = _big_setup(ABOVE)
    assert _big_apply(c, u0, d, None, monkeypatch) == TWO
    assert _lib().b2_last_iso_coef_reuse() == expected_reuse(d, SO, *_full(ABOVE)) > 1
    two = np.array(c.u.data_ro_with_halo)
    two_tr = np.array(c.rec.data)
    assert _big_apply(c, u0, d, '0', monkeypatch) == ONE
    one = np.array(c.u.data_ro_with_halo)
    one_tr = np.array(c.rec.data)
    assert np.abs(one).max() > 0.5 and np.abs(one_tr[:6]).max() > 1e-3
    assert not np.array_equal(one[1], u0[1])                               # the run moved u
    assert np.array_equal(two, one)
    assert np.array_equal(two_tr, one_tr)


EXCLUDED = {
    # configuration: the kernel it takes with B2_ISO2=2 ('plain' is the control)
    'plain': TWO,
    'vp_function': 'iso_tma<4,vp>',
    'so4': 'iso_tma<2,scalar>',
    'so12': 'iso_tma<6,scalar>',
    'adjoint': ONE,
    'ot4': 'iso_generic',
    'free_surface': ONE,
    'born': ONE,
    'snapshots': ONE,
    'gradient': ONE,
}


@functools.lru_cache(maxsize=None)
def _excluded_setup(case):
    """the configuration without sparse points; fields other than u start at zero (halo included)"""
    from devito_b200 import (ConditionalDimension, Constant, Eq, FreeSurface, Function, Inc, Operator, TimeFunction,
                             solve)
    from test_scheme_matrix import _grid
    so = {'so4': 4, 'so12': 12}.get(case, SO)
    grid = _grid(SHAPE, case == 'free_surface', so)
    adjoint = case in ('adjoint', 'gradient')
    u = TimeFunction(name='v' if adjoint else 'u', grid=grid, time_order=2, space_order=so)
    damp = Function(name='damp', grid=grid, space_order=so)
    if case == 'vp_function':
        vp = Function(name='vp', grid=grid, space_order=so)
        vp.data_with_halo[:] = 2.0
    else:
        vp = Constant(name='vp', value=2.0)
    m = 1 / vp ** 2
    s = grid.time_dim.spacing

    def stencil(f, q=0):
        nxt = f.backward if adjoint else f.forward
        lap = f.laplace + (s ** 2 / 12 * f.biharmonic(1 / m) if case == 'ot4' else 0)
        pde = m * f.dt2 - lap - q + damp * (f.dt.T if adjoint else f.dt)
        if case != 'free_surface':
            return [Eq(nxt, solve(pde, nxt))]
        update = Eq(nxt, solve(pde, nxt), subdomain=grid.subdomains['physdomain'])
        return [update, FreeSurface(update, grid.subdomains['fsdomain'])]

    eqs = stencil(u)
    if case == 'born':
        U = TimeFunction(name='U', grid=grid, time_order=2, space_order=so)
        dm = Function(name='dm', grid=grid, space_order=0)
        dm.data_with_halo[:] = 0.01
        eqs += stencil(U, q=-dm * u.dt2)
    elif case == 'gradient':
        usave = TimeFunction(name='u', grid=grid, time_order=2, space_order=so, save=KC.K + 2)
        eqs.append(Inc(Function(name='grad', grid=grid), -usave * u.dt2))
    elif case == 'snapshots':
        t_sub = ConditionalDimension('t_sub', parent=grid.time_dim, factor=2)
        snap = TimeFunction(name='usave', grid=grid, time_order=2, space_order=so, save=KC.K // 2 + 2, time_dim=t_sub)
        eqs.append(Eq(snap, u))
    op = Operator(eqs)
    assert op.backend == 'cuda-sm90a', getattr(op, '_why_not', None)
    return op, u, damp, so


@pytest.mark.gpu
@pytest.mark.parametrize('case', list(EXCLUDED))
def test_excluded_configurations(case, monkeypatch):
    """With B2_ISO2=2, a zero halo and no sparse points, only the configuration itself keeps the pass out. These
    paths have their own float64 matrices (test_kernel_matrix, test_scheme_matrix)."""
    monkeypatch.setenv('B2_ISO2', '2')
    monkeypatch.delenv('B2_ISO_LX', raising=False)
    op, u, damp, so = _excluded_setup(case)
    a = tuple(n + 2 * so for n in SHAPE)
    u0 = np.zeros((3,) + a, dtype=np.float32)
    u0[(slice(None),) + (slice(so, -so),) * 3] = np.random.default_rng(2).standard_normal((3,) + SHAPE)
    u.data_with_halo[:] = u0
    damp.data_with_halo[:] = (0.1 * np.random.default_rng(3).uniform(0.0, 1.0, a)).astype(np.float32)
    op.apply(time_m=1, time_M=KC.K, dt=float(O.critical_dt(so, 3, min(KC.SPACING), 2.5)))
    assert _kernel() == EXCLUDED[case]
    assert np.abs(np.array(u.data_ro_with_halo)).max() > 0.5


# ---------------------------------------------------------------------------------------------------------------
# 7. CPU twins: the cases above still mean what they claim
# ---------------------------------------------------------------------------------------------------------------
def test_entry_counts():
    assert MAX_INJ == 64
    assert _support(POINTS8).size // 3 == MAX_INJ
    assert _support((SINC,), 2, 'sinc').size // 3 == MAX_INJ
    assert _support(POINTS9).size // 3 == MAX_INJ + 8


def test_supports_inside_and_outside_the_box():
    for pts, r, interp in [(POINTS9, 1, 'linear'), ((SINC,), 2, 'sinc'), (REC, 1, 'linear')]:
        assert _inside(_support(pts, r, interp), FULL).all()
    assert _inside(_support(REC), _full(TSHAPE)).all()
    assert _inside(_support(GATE_REC), GATE).all()
    # the x-plane receivers sample plane 5 (weight 1) and plane 6 (weight 0), inside the box's rows and columns
    cells = _support(XPLANE_REC)
    assert set(cells[..., 0].ravel()) == {5, 6} and _inside(cells[..., 1:], (XPLANE[0][1:], XPLANE[1][1:])).all()
    assert _inside(_support((WHOLE_SRC,) + WHOLE_REC), _full(WHOLE)).all()
    assert _inside(_support(((20.5, 30.4, 63.6),)), _full(TSHAPE)).all()
    assert _inside(_support((CORNER,)), SUB).all()
    # SUB touches no face of FULL on any axis: stale scratch values inside FULL would sit in SUB's halo
    assert all(0 < l and h < n - 1 for l, h, n in zip(*SUB, SHAPE)) and (SUB[1][2] - SUB[0][2] + 1) % 4 != 0
    # every face of FULL is touched from inside by one of FACES
    cells = _support(FACES)
    for d in range(3):
        assert cells[2 * d][:, d].min() == 0
        assert cells[2 * d + 1][:, d].max() == SHAPE[d] - 1
    # OUTSIDE: exactly one support plane one cell beyond its face
    for f, p in OUTSIDE.items():
        cells = _support((p,))[0]
        d = 'xyz'.index(f[0])
        beyond = -1 if f.endswith('lo') else SHAPE[d]
        assert np.count_nonzero(~_inside(cells, FULL)) == 4
        assert np.all(cells[~_inside(cells, FULL)][:, d] == beyond)
    # SHARED deposits into CORNER's cells
    g = _support((CORNER, SHARED))
    assert np.array_equal(g[0], g[1])


def test_corner_supports_straddle_tile_and_chunk_edges():
    assert (TY, TZ) == (16, 64)
    assert SHAPE[1] % TY and SHAPE[2] % TZ and WHOLE[1] % TY == 0 and WHOLE[2] % TZ == 0
    for pts, r, interp in [((CORNER,), 1, 'linear'), ((SHARED,), 1, 'linear'), ((SINC,), 2, 'sinc')]:
        cells = _support(pts, r, interp)[0]
        for d, edge in enumerate((LX, TY, TZ)):
            assert cells[:, d].min() == edge - r and cells[:, d].max() == edge + r - 1
    cells = _support((WHOLE_SRC,))[0]
    assert [(cells[:, d].min(), cells[:, d].max()) for d in (1, 2)] == [(TY - 1, TY), (TZ - 1, TZ)]
    # the gate box: one partial tile, smaller than the level-1 region (16 + 2R) x (64 + 2R)
    n = KC.box_extent(GATE)
    assert n == (8, 8, 16) and n[1] < TY + 2 * R and n[2] < TZ + 2 * R
    assert KC.box_extent(XPLANE)[0] == 1


def test_layered_damp_reuse_counts():
    """the pinned planes of the layered damp, and the pinned/streamed switches the perturbed planes put at every
    offset level 2's R-plane lag reads"""
    assert PERTURBED[0] % LX == 0 and PERTURBED[-1] % LX == LX - 1
    assert PERTURBED[2] == PERTURBED[1] + 1 and PERTURBED[3] == PERTURBED[2] + R
    for box, want in [(FULL, 70 - 2 * LAYER - 5), (SUB, 66 - 2 * (LAYER - 2) - 5)]:
        d = layered_damp(SHAPE, box)
        n = expected_reuse(d, SO, *box)
        assert n == want
        assert 1 < n < box[1][0] - box[0][0] + 1
        # the centre plane is not perturbed; perturbing it inside the box's rows does change the count
        lo, hi = box
        assert lo[0] + (hi[0] - lo[0] + 1) // 2 - lo[0] not in PERTURBED
        assert expected_reuse(layered_damp(SHAPE, box, planes=()), SO, *box) == want + 5
    d = layered_damp(ABOVE, _full(ABOVE), planes=(100, 101, 105))
    assert expected_reuse(d, SO, *_full(ABOVE)) == ABOVE[0] - 2 * LAYER - 3


def test_one_gib_threshold_sides():
    assert _u_bytes(BELOW) < 2 ** 30 <= _u_bytes(ABOVE)
    assert ABOVE[0] == BELOW[0] + 1 and ABOVE[1:] == BELOW[1:]
    assert len(set(ABOVE)) == 3 and ABOVE[1] % TY and ABOVE[2] % TZ and ABOVE[2] % 4 == 0
    assert _u_bytes(TSHAPE) == _u_bytes(SHAPE)


def test_sinc_r2_tabulation_matches_the_oracle():
    """the device takes SparseTimeFunction's float32 table; the float64 reference takes the oracle's"""
    from devito_b200 import Grid, SparseTimeFunction
    grid = Grid(shape=SHAPE, extent=tuple((n - 1) * h for n, h in zip(SHAPE, KC.SPACING)))
    s = SparseTimeFunction(name='src', grid=grid, npoint=1, nt=NT, interpolation='sinc', r=2, coordinates=_coords(SINC))
    gp, ws = s.tabulate()
    ogp, ows = O.tabulate(_coords(SINC), (0.0, 0.0, 0.0), KC.SPACING, 2, 'sinc')
    _, w64 = O.tabulate(_coords(SINC), (0.0, 0.0, 0.0), KC.SPACING, 2, 'sinc', dtype=np.float64)
    assert np.array_equal(gp, ogp) and tuple(gp[0]) == (31, 15, 63)
    for w, ow, o64 in zip(ws, ows, w64):
        assert w.dtype == np.float32 and w.shape == (1, 4)
        assert np.array_equal(w, ow)
        assert np.abs(w - o64).max() < 1e-7 and np.abs(w).min() > 1e-3
