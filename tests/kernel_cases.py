"""Inputs of the kernel-variant matrix (tests/test_kernel_matrix.py on the GPU, tests/test_ref64.py on the CPU).

Every case starts from white noise in all three time slots of the wavefields, halo included, a spatially varying
damping field and, for array parameters, white-noise parameter fields. The grid is anisotropic and not a cube:
spacing (10, 12.5, 8), shape (37, 45, 68) -- nx != ny != nz, ny a multiple of none of the sweep kernels' tile
heights, nz a multiple of 4 but not of the 64-point z tiles. So an exchanged axis, stride or weight list, a wrong
parameter sample, a skipped partial tile or a swapped time level changes the answer by far more than the tolerance
(tests/test_ref64.py shows by how much). K = 4 steps: every slot rotation happens once, errors do not pile up.
"""
import numpy as np

from oracle import oracle as O
import ref64

SHAPE = (37, 45, 68)
SPACING = (10.0, 12.5, 8.0)
K = 4                                   # time steps 1 .. K
TOL = {'iso': 1e-5, 'tti': 1e-4}       # rel L-inf against float64 (BASELINE.json north star)
TTI_SCALARS = dict(vp=2.0, epsilon=0.2, delta=0.1, theta=0.6, phi=0.35)
SUBBOX = ((1, 2, 4), (SHAPE[0] - 3, SHAPE[1] - 4, SHAPE[2] - 9))   # reaches the halo in x and y, z_m % 4 == 0

# Boxes on SHAPE whose z extent is not a multiple of 4, z_m % 4 == 0 (so the TMA sweeps still take them): the last
# float4 group of every row holds 1, 2 or 3 points and goes through the sweeps' partial (scalar) loads and stores.
# face3 reaches every face; unlike a grid of nz = 67 (an allocation the TMA sweeps refuse) its allocation is aligned.
ZTAIL = {
    'tail1': ((1, 2, 4), (34, 41, 60)),        # z extent 57
    'tail2': ((1, 2, 4), (34, 41, 61)),        # 58
    'tail3': ((1, 2, 4), (34, 41, 62)),        # 59
    'face3': ((0, 0, 0), (36, 44, 66)),        # 67
}
# The size gate of iso_plan_init / tti_plan_init: boxes with n[1] < 8 or n[2] < 16 run the generic / two-pass kernels.
GATE = {
    'gate_in': ((1, 2, 4), (8, 9, 19)),        # n = (8, 8, 16): the TMA / fused sweep
    'gate_y': ((1, 2, 4), (8, 8, 19)),         # n = (8, 7, 16): falls back
    'gate_z': ((1, 2, 4), (8, 9, 15)),         # n = (8, 8, 12): falls back
}
# One x-plane (the 2.5-D march primes 2R planes for one output plane), z extent 59
XPLANE = ((5, 2, 4), (5, 41, 62))
# Boxes for the sweeps without a size gate (sa_plan_init), z_m % 4 == 0: a corner point, a corner float4 group at the
# far faces, a small interior box with a z tail of 3
TINY = {
    'tiny111': ((0, 0, 0), (0, 0, 0)),
    'tiny114': ((36, 44, 64), (36, 44, 67)),
    'tiny257': ((3, 5, 8), (4, 9, 14)),
}
BOXES = dict(ZTAIL, **GATE, xplane=XPLANE, **TINY, sub=SUBBOX)

# Grids cut into several yz-tiles by every iso tile configuration (TILES):
#   MULTI: >= 2 y tiles and >= 3 z tiles, the last of each partial. 16 x 128: 3 x 3 tiles, the last 12 x 44;
#          32 x 64: 2 x 5, the last 12 x 44; 16 x 64: 3 x 5, the last 12 x 44; 8 x 64: 6 x 5, the last 4 x 44.
#   EXACT: every tile full. 16 x 128: 2 x 2; 32 x 64: 1 x 4; 16 x 64: 2 x 4; 8 x 64: 4 x 4.
MULTI = (13, 44, 300)
MULTI_TAIL = ((0, 0, 0), (12, 43, 297))        # z extent 298: 16 x 128 tiles 3 x 3, the last 12 x 42
EXACT = (9, 32, 256)

# (TY, TZ) of the yz-tile each 3-D sweep marches along x, per `b2_last_sweep_kernel` name
TILES = {
    # b2_iso.cu TileOf<R, ARR>: (TY, 4 TZ4)
    'iso_tma<2,scalar>': (32, 64), 'iso_tma<2,vp>': (32, 64), 'iso_tma<2,m>': (32, 64),
    'iso_tma<4,scalar>': (16, 128), 'iso_tma<4,vp>': (32, 64), 'iso_tma<4,m>': (32, 64),
    'iso_tma<6,scalar>': (16, 64), 'iso_tma<6,vp>': (16, 64), 'iso_tma<6,m>': (16, 64),
    'iso_tma<8,scalar>': (8, 64), 'iso_tma<8,vp>': (8, 64), 'iso_tma<8,m>': (8, 64),
    # b2_tti.cu TtiTile<R>::TY, kTtiWsTY, TtiArrTile<R>::TY; TZ: TtiCfg / TtiWsCfg
    'tti_fused<2>': (32, 64), 'tti_fused<4>': (28, 64), 'tti_ws<pf1>': (24, 64),
    'tti_arr_ct2<2>': (30, 64), 'tti_arr_ct2<4>': (20, 64),
    # b2_nested.cuh NestedCfg<R> (the SA sweep k_nested_tma<R, SaEpi>)
    'sa_tma<2>': (16, 64), 'sa_tma<4>': (16, 64),
}
TTI_SA_TILES = {name: t for name, t in TILES.items() if name.startswith(('tti_', 'sa_'))}

# Grids cut into several yz-tiles by every TTI and SA tile (tests/test_tti_sa_tiling.py checks these claims):
#   TTI_MULTI: y tiles of 32, 28, 24, 30, 20, 16 rows: 3, 3, 3, 3, 4, 5 tiles, the last 7, 15, 23, 11, 11, 7 rows;
#              z: 6 tiles, the last 44 points. nty != ntz everywhere, so a block index decoded with the two counts
#              exchanged (or the tile origins of y and z exchanged) covers other tiles. The z allocation 364 + 2 so
#              keeps the rows 16-byte aligned.
#   TTI_MULTI_TAIL: z extent 362: the last z tile 42 points, every row ends in a partial float4 group of 2.
#   TTI_MULTI_SUB: y extent 65 (a last y tile of one row for TY 32 and 16), z extent 352 (the last z tile 32);
#                  x extent 11: x-chunks of 5, 5, 1 with B2_TTI_LX=5.
#   TTI_EXACT: (9, 3 TY, 256) per sweep: 3 x 4 full tiles.
#   LONGX: nothing forced, choose_chunk_len on 132 SMs cuts the 150 x-planes of every TTI sweep into chunks of
#          LONGX_LX = 38 planes (38, 38, 38, 36).
TTI_MULTI = (13, 71, 364)
TTI_MULTI_TAIL = ((0, 0, 0), (12, 70, 361))
TTI_MULTI_SUB = ((1, 3, 4), (11, 67, 355))
TTI_EXACT = {name: (9, 3 * ty, 256) for name, (ty, _) in TTI_SA_TILES.items()}
LONGX = (150, 30, 64)
LONGX_LX = 38
H100_SMS = 132


def tiling(n, t):
    """(number of tiles, extent of the last one) of an extent n cut into tiles of t"""
    k = -(-n // t)
    return k, n - (k - 1) * t


def chunk_len(sms, tiles, xcount, prime, min_len=32):
    """b2_common.cuh choose_chunk_len: the x-chunk length that minimises wave quantisation x priming overhead"""
    best, best_n = 1e30, 1
    for n in range(1, 65):
        lx = -(-xcount // n)
        if n > 1 and lx < min_len:
            break
        if lx > 256 and (xcount + n) // (n + 1) >= min_len:
            continue
        ctas = tiles * n
        rounds = -(-ctas // sms)
        cost = rounds * sms / ctas * (1.0 + prime / lx)
        if cost < best - 1e-9:
            best, best_n = cost, n
    return -(-xcount // best_n)


def x_chunks(xcount, lx):
    """extents of the x-chunks of length lx (the last may be shorter)"""
    return [min(lx, xcount - s) for s in range(0, xcount, lx)]


def box_extent(box):
    return tuple(h - l + 1 for l, h in zip(*box))


def _alloc(shape, so):
    return tuple(n + 2 * so for n in shape)


def iso_case(so, param, shape=SHAPE, box=None, seed=0):
    """param: 'scalar' (vp = 2), 'vp' (vp array) or 'm' (squared-slowness array)."""
    rng = np.random.default_rng(seed + 100 * so)
    a = _alloc(shape, so)
    u = rng.standard_normal((3,) + a).astype(np.float32)
    damp = (0.1 * rng.uniform(0.0, 1.0, a)).astype(np.float32)
    vp = rng.uniform(1.5, 2.5, a).astype(np.float32)
    p = {'scalar': ('vp', np.float32(2.0)), 'vp': ('vp', vp), 'm': ('m', (1.0 / (vp * vp)).astype(np.float32))}[param]
    lo, hi = box if box is not None else ((0,) * len(shape), tuple(n - 1 for n in shape))
    return dict(kind='iso', so=so, shape=shape, u=u, damp=damp, param=p, lo=tuple(lo), hi=tuple(hi),
                dt=float(O.critical_dt(so, 3, min(SPACING), 2.5)))


def tti_case(so, arrays, shape=SHAPE, box=None, seed=0):
    """arrays: vp, epsilon, delta, theta, phi as white-noise fields (else the scalars TTI_SCALARS, phi != 0)."""
    rng = np.random.default_rng(seed + 100 * so + 7)
    a = _alloc(shape, so)
    u = rng.standard_normal((3,) + a).astype(np.float32)
    v = rng.standard_normal((3,) + a).astype(np.float32)
    damp = (0.1 * rng.uniform(0.0, 1.0, a)).astype(np.float32)
    if arrays:
        rg = dict(vp=(1.5, 2.5), epsilon=(0.05, 0.3), delta=(0.02, 0.15), theta=(0.2, 1.2), phi=(-0.6, 0.9))
        params = {n: rng.uniform(lo, hi, a).astype(np.float32) for n, (lo, hi) in rg.items()}
    else:
        params = {n: np.float32(x) for n, x in TTI_SCALARS.items()}
    lo, hi = box if box is not None else ((0,) * len(shape), tuple(n - 1 for n in shape))
    return dict(kind='tti', so=so, shape=shape, u=u, v=v, damp=damp, params=params, lo=tuple(lo), hi=tuple(hi),
                dt=float(O.critical_dt(so, 3, min(SPACING), 2.5, eps_max=0.3)))


def sparse_coordinates(shape=SHAPE, seed=3, seams=None):
    """Physical coordinates (origin 0) of points within one cell of every face, points outside the domain on both
    sides of every axis (their supports reach into the halo, or miss the grid entirely), and two points in one
    cell (their deposits meet in the same cells).

    seams = (origin, xcuts) appends, after those, points half a cell either side of every seam inside the grid: of the
    TTI and SA yz-tiles counted from the box corner `origin` (y = origin + TY k for every tile height TY, z = origin +
    64 and + 128) and of the x-chunks that begin at the x indices `xcuts`. Their supports straddle the seam."""
    rng = np.random.default_rng(seed)
    n = np.array(shape)
    h = np.array(SPACING)
    pts = []

    def interior():
        return rng.uniform(2.0, n - 3.0)

    for d in range(3):
        for where in (0.4, n[d] - 1 - 0.3, -1.6, n[d] - 1 + 1.3):   # inside near the faces, then just outside
            p = interior()
            p[d] = where
            pts.append(p)
    far = interior()
    far[1] = -12.0                                                  # no support cell inside any halo
    pts.append(far)
    c = np.floor(interior())
    pts.append(c + 0.27)
    pts.append(c + np.array([0.81, 0.62, 0.55]))                    # same base cell as the point above
    if seams is not None:
        origin, xcuts = seams
        tys = sorted({ty for ty, _ in TTI_SA_TILES.values()})
        (tz,) = {tz for _, tz in TTI_SA_TILES.values()}
        cuts = [sorted(xcuts),
                sorted({origin[1] + ty * k for ty in tys for k in range(1, n[1] // ty + 1)}),
                [origin[2] + tz, origin[2] + 2 * tz]]
        for d, cs in enumerate(cuts):
            for cut in cs:
                for where in (cut - 0.5, cut + 0.5):
                    if 0 < where < n[d] - 1:
                        p = interior()
                        p[d] = where
                        pts.append(p)
    return (np.array(pts) * h).astype(np.float32)


def sparse_tables(coords, interpolation, nt):
    """Base cells and float64 weights (the host-side tabulation of the oracle) plus random traces."""
    r = 1 if interpolation == 'linear' else 4
    gp, ws = O.tabulate(coords, (0.0, 0.0, 0.0), SPACING, r, interpolation, dtype=np.float64)
    rng = np.random.default_rng(11)
    data = rng.standard_normal((nt, coords.shape[0])).astype(np.float32)
    return dict(data=data, gp=gp, w=ws, r=r)


def weights(kind, so):
    """(float64 weights for the reference, float32 weights for the oracle) per axis."""
    w64 = [ref64.fd2_weights(so, h) for h in SPACING]
    w32 = [O.fd2_weights(so, h) for h in SPACING]
    if kind == 'iso':
        return w64, w32
    w164 = [ref64.fd1_half_weights(so, h) for h in SPACING]
    w132 = [O.fd1_half_weights(so, h) for h in SPACING]
    return (w64, w164), (w32, w132)


GRAD_HALO = 1                            # grad is a Function with its own (smaller) halo
SNAP_HALO = 3                            # snapshot halo != so
SNAP_FACTOR = 2
SNAP_SENTINEL = -7.25                    # exactly representable: unvisited snapshot cells must keep it bit for bit


def scheme_case(scheme, so, param, box=None, dmh=0, shape=SHAPE, seed=0):
    """An iso case plus what a scheme needs, white noise throughout:
    'plain' | 'adjoint' | 'fs' | 'adjoint_fs' | 'ot4' | 'adjoint_ot4' (nothing more), 'grad' (adjoint + imaging condition:
    usave for times 0 .. K+1 with u's layout, grad with halo GRAD_HALO), 'born' (U, dm with halo `dmh`),
    'snap' / 'snap_fwd' (Eq(usave, u) / Eq(usave, u.forward): a snapshot array of halo SNAP_HALO, filled with
    SNAP_SENTINEL). 2-D cases pass a 2-D `shape` (the time-slot noise and the parameters are drawn the same way)."""
    c = iso_case(so, param, shape=shape, box=box, seed=seed)
    if len(shape) == 2:
        c['dt'] = float(O.critical_dt(so, 2, min(SPACING[1:]), 2.5))
    c['scheme'] = scheme
    rng = np.random.default_rng(seed + 100 * so + 31)
    if scheme == 'grad':
        c['usave'] = rng.standard_normal((K + 2,) + c['u'].shape[1:]).astype(np.float32)
        c['grad'] = rng.standard_normal(tuple(n + 2 * GRAD_HALO for n in shape)).astype(np.float32)
    elif scheme == 'born':
        c['U'] = rng.standard_normal(c['u'].shape).astype(np.float32)
        c['dm'] = (0.05 * rng.standard_normal(tuple(n + 2 * dmh for n in shape))).astype(np.float32)
        c['dmh'] = dmh
    elif scheme in ('snap', 'snap_fwd'):
        c['snap'] = np.full((K // SNAP_FACTOR + 2,) + tuple(n + 2 * SNAP_HALO for n in shape), SNAP_SENTINEL,
                            dtype=np.float32)
    return c


def scheme_reference(c, src=None, rec=None, mut=None):
    """float64 run of a scheme case: dict of every output ('u', 'traces', and 'U', 'grad' or 'snap')."""
    so, s = c['so'], c['scheme']
    w64 = [ref64.fd2_weights(so, h) for h in SPACING[3 - len(c['shape']):]]
    kw = dict(damp=c['damp'], param=c['param'], lo=c['lo'], hi=c['hi'], src=src, rec=rec, mut=mut)
    if s == 'born':
        u, U, tr = ref64.born_forward(c['u'], c['U'], c['dm'], c['dmh'], so, w64, c['dt'], 1, K, **kw)
        return dict(u=u, U=U, traces=tr)
    out = {}
    if s == 'grad':
        out['grad'] = c['grad'].astype(np.float64)
        kw.update(grad=out['grad'], gh=GRAD_HALO, usave=c['usave'])
    if s in ('snap', 'snap_fwd'):
        out['snap'] = c['snap'].astype(np.float64)
        kw.update(snap=out['snap'], snap_h=SNAP_HALO, snap_factor=SNAP_FACTOR, snap_toff=int(s == 'snap_fwd'))
    u, tr = ref64.iso_forward(c['u'], so, w64, c['dt'], 1, K, adjoint=s in ('adjoint', 'adjoint_fs', 'adjoint_ot4',
                                                                              'grad'),
                              free_surface=s in ('fs', 'adjoint_fs'), ot4=s in ('ot4', 'adjoint_ot4'), **kw)
    out.update(u=u, traces=tr)
    return out


def reference(c, src=None, rec=None, mut=None):
    """float64 run of a case: (fields..., traces)."""
    so = c['so']
    if c['kind'] == 'iso':
        w64, _ = weights('iso', so)
        u, tr = ref64.iso_forward(c['u'], so, w64, c['dt'], 1, K, damp=c['damp'], param=c['param'], lo=c['lo'],
                                  hi=c['hi'], src=src, rec=rec, mut=mut)
        return (u,), tr
    (w2, w1), _ = weights('tti', so)
    u, v, tr = ref64.tti_forward(c['u'], c['v'], so, w2, w1, c['dt'], 1, K, c['damp'], c['params'], lo=c['lo'],
                                 hi=c['hi'], src=src, rec=rec, mut=mut)
    return (u, v), tr
