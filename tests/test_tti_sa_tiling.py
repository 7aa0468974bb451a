"""The tilings the TTI / SA grids of tests/kernel_cases.py claim, and that KC.TILES still matches the kernels. CPU only.

tests/test_tti_sa_tiling_matrix.py runs every TTI and SA sweep on these grids on the GPU. What they are for holds
only while the kernels' tiles are the ones KC.TILES lists: the tile sizes are read from the CUDA sources here, so a
retuned tile fails this file instead of quietly leaving a grid with one tile per axis.
"""
import os
import re

import pytest

import kernel_cases as KC

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'devito_b200', 'csrc')


def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _ints(body, *names):
    """the `static constexpr int` members `names` of a struct body (integer expressions of earlier members)"""
    decl = {}
    for line in re.findall(r'static constexpr int ([^;]*);', body):
        for item in line.split(','):
            k, _, v = item.partition('=')
            decl[k.strip()] = v.strip()
    env = {}

    def value(k):
        if k not in env:
            expr = decl[k]
            assert re.fullmatch(r'[\w\s*+/()-]+', expr), (k, expr)
            for dep in set(re.findall(r'[A-Za-z_]\w*', expr)):
                value(dep)
            env[k] = int(eval(expr, {'__builtins__': {}}, dict(env)))
        return env[k]
    return tuple(value(k) for k in names)


def _struct(src, head):
    """the body of the struct whose declaration matches `head` (up to its closing brace)"""
    m = re.search(head + r'\s*\{(.*?)\n?\};', src, re.S)
    assert m, head
    return m.group(1)


def kernel_tiles():
    """(TY, TZ) per sweep name, as the CUDA sources define them"""
    iso, tti, nested = _source('b2_iso.cu'), _source('b2_tti.cu'), _source('b2_nested.cuh')
    out = {}
    for r in (2, 4, 6, 8):
        for param in ('scalar', 'vp', 'm'):
            arr = 'false' if param == 'scalar' else 'true'
            m = re.search(rf'struct TileOf<{r}, {arr}>\s*\{{([^}}]*)\}}', iso) or \
                re.search(rf'struct TileOf<{r}, ARR>\s*\{{([^}}]*)\}}', iso)
            assert m, (r, param)
            ty, tz4 = _ints(m.group(1), 'TY', 'TZ4')
            out[f'iso_tma<{r},{param}>'] = (ty, 4 * tz4)
    (tz,) = _ints(_struct(tti, r'struct TtiCfg'), 'TZ')
    (tz_ws,) = _ints(_struct(tti, r'struct TtiWsCfg'), 'TZ')
    for r in (2, 4):
        (ty,) = _ints(_struct(tti, rf'struct TtiTile<{r}>'), 'TY')
        out[f'tti_fused<{r}>'] = (ty, tz)
        (ty,) = _ints(_struct(tti, rf'struct TtiArrTile<{r}>'), 'TY')
        out[f'tti_arr_ct2<{r}>'] = (ty, tz)
    out['tti_ws<pf1>'] = (int(re.search(r'constexpr int kTtiWsTY = (\d+);', tti).group(1)), tz_ws)
    ty, tz = _ints(_struct(nested, r'template <int R> struct NestedCfg'), 'TY', 'TZ')
    out['sa_tma<2>'] = out['sa_tma<4>'] = (ty, tz)
    return out


def test_tiles_match_the_kernel_sources():
    """the iso and TTI tiles of their sweep files, and the SA tile of the nested-operator sweep (b2_nested.cuh)"""
    assert kernel_tiles() == KC.TILES


# (y tiles, z tiles), (last y tile, last z tile) per sweep and layout: the tables of kernel_cases
CLAIMS = {
    'tti_fused<2>':   {'multi': ((3, 6), (7, 44)), 'multi_tail': ((3, 6), (7, 42)), 'multi_sub': ((3, 6), (1, 32)),
                       'exact': ((3, 4), (32, 64)), 'longx': ((1, 1), (30, 64))},
    'tti_fused<4>':   {'multi': ((3, 6), (15, 44)), 'multi_tail': ((3, 6), (15, 42)), 'multi_sub': ((3, 6), (9, 32)),
                       'exact': ((3, 4), (28, 64)), 'longx': ((2, 1), (2, 64))},
    'tti_ws<pf1>':    {'multi': ((3, 6), (23, 44)), 'multi_tail': ((3, 6), (23, 42)), 'multi_sub': ((3, 6), (17, 32)),
                       'exact': ((3, 4), (24, 64)), 'longx': ((2, 1), (6, 64))},
    'tti_arr_ct2<2>': {'multi': ((3, 6), (11, 44)), 'multi_tail': ((3, 6), (11, 42)), 'multi_sub': ((3, 6), (5, 32)),
                       'exact': ((3, 4), (30, 64)), 'longx': ((1, 1), (30, 64))},
    'tti_arr_ct2<4>': {'multi': ((4, 6), (11, 44)), 'multi_tail': ((4, 6), (11, 42)), 'multi_sub': ((4, 6), (5, 32)),
                       'exact': ((3, 4), (20, 64)), 'longx': ((2, 1), (10, 64))},
    'sa_tma<2>':      {'multi': ((5, 6), (7, 44)), 'multi_tail': ((5, 6), (7, 42)), 'multi_sub': ((5, 6), (1, 32)),
                       'exact': ((3, 4), (16, 64))},
    'sa_tma<4>':      {'multi': ((5, 6), (7, 44)), 'multi_tail': ((5, 6), (7, 42)), 'multi_sub': ((5, 6), (1, 32)),
                       'exact': ((3, 4), (16, 64))},
}
# x-chunks per layout: with B2_TTI_LX=5 (the multi layouts and exact) and with nothing forced
CHUNKS = {
    ('multi', 5): [5, 5, 3], ('multi_tail', 5): [5, 5, 3], ('multi_sub', 5): [5, 5, 1], ('exact', 5): [5, 4],
    ('multi', None): [13], ('multi_tail', None): [13], ('multi_sub', None): [11], ('longx', None): [38, 38, 38, 36],
}
MULTI = ('multi', 'multi_tail', 'multi_sub')


def extent(sweep, layout):
    """the update box's extent of a layout"""
    if layout == 'multi':
        return KC.TTI_MULTI
    if layout == 'multi_tail':
        return KC.box_extent(KC.TTI_MULTI_TAIL)
    if layout == 'multi_sub':
        return KC.box_extent(KC.TTI_MULTI_SUB)
    if layout == 'exact':
        return KC.TTI_EXACT[sweep]
    return KC.LONGX


def _radius(sweep):
    return 4 if sweep == 'tti_ws<pf1>' else int(re.search(r'<(\d)>', sweep).group(1))


def test_claims_cover_every_tti_and_sa_sweep():
    assert set(CLAIMS) == set(KC.TTI_SA_TILES)


@pytest.mark.parametrize('sweep', list(KC.TTI_SA_TILES))
def test_tti_sa_tilings(sweep):
    ty, tz = KC.TTI_SA_TILES[sweep]
    for layout, want in CLAIMS[sweep].items():
        n = extent(sweep, layout)
        (ky, ly), (kz, lz) = KC.tiling(n[1], ty), KC.tiling(n[2], tz)
        assert ((ky, kz), (ly, lz)) == want, (sweep, layout)
    for layout in MULTI:
        n = extent(sweep, layout)
        (ky, ly), (kz, lz) = KC.tiling(n[1], ty), KC.tiling(n[2], tz)
        # several tiles on both axes, the last of each partial, and as many y tiles as z tiles nowhere
        assert ky >= 3 and kz >= 3 and ly < ty and lz < tz and ky != kz, (sweep, layout)
    n = KC.TTI_EXACT[sweep]
    assert n[1] % ty == 0 and n[2] % tz == 0 and (n[1] // ty, n[2] // tz) == (3, 4), sweep


def _tiles_visited(ny, nz, ty, tz, exchange):
    """(y, z) origins of the tiles a grid of ny x nz tiles visits, decoding the block index like the sweeps (iz =
    b % ntz, iy = (b / ntz) % nty). exchange='counts': ntz and nty exchanged; 'origins': y0 from iz, z0 from iy."""
    cz, cy = (ny, nz) if exchange == 'counts' else (nz, ny)
    out = set()
    for b in range(ny * nz):
        iz, iy = b % cz, (b // cz) % cy
        out.add((iz * ty, iy * tz) if exchange == 'origins' else (iy * ty, iz * tz))
    return out


@pytest.mark.parametrize('sweep', list(KC.TTI_SA_TILES))
def test_exchanged_tile_indices_show_on_the_multi_grids(sweep):
    """An exchange of ntz and nty in the block decoding, or of the tiles' y and z origins, visits other tiles on every
    multi layout; on KC.SHAPE it is invisible wherever that grid has as many y tiles as z tiles."""
    ty, tz = KC.TTI_SA_TILES[sweep]
    for layout in MULTI:
        n = extent(sweep, layout)
        ny, nz = KC.tiling(n[1], ty)[0], KC.tiling(n[2], tz)[0]
        right = _tiles_visited(ny, nz, ty, tz, None)
        assert len(right) == ny * nz
        for exchange in ('counts', 'origins'):
            assert _tiles_visited(ny, nz, ty, tz, exchange) != right, (sweep, layout, exchange)
    ny, nz = KC.tiling(KC.SHAPE[1], ty)[0], KC.tiling(KC.SHAPE[2], tz)[0]
    if ny == nz:
        for exchange in ('counts', 'origins'):
            assert _tiles_visited(ny, nz, ty, tz, exchange) == _tiles_visited(ny, nz, ty, tz, None)


def test_x_chunks():
    """B2_TTI_LX=5 on the multi and exact layouts; the default (choose_chunk_len on 132 SMs, priming 2R planes) on
    the multi layouts (one chunk: chunks are at least 32 planes) and on LONGX (>= 3 chunks, the last shorter)."""
    for (layout, lx), want in CHUNKS.items():
        for sweep in [s for s in KC.TTI_SA_TILES if s.startswith('tti_')]:
            n = extent(sweep, layout)
            if lx is None:
                ty, tz = KC.TTI_SA_TILES[sweep]
                tiles = KC.tiling(n[1], ty)[0] * KC.tiling(n[2], tz)[0]
                got = KC.x_chunks(n[0], KC.chunk_len(KC.H100_SMS, tiles, n[0], 2 * _radius(sweep)))
            else:
                got = KC.x_chunks(n[0], lx)
            assert got == want, (sweep, layout, lx)
    assert KC.x_chunks(KC.LONGX[0], KC.LONGX_LX) == CHUNKS[('longx', None)]
    longx = CHUNKS[('longx', None)]
    assert len(longx) >= 3 and longx[-1] < longx[0]


def test_layout_alignment():
    """The TMA sweeps take these layouts: z allocation and box start multiples of 4 (16-byte rows), and the TTI
    array sweeps' R rows and 4 z points of halo either side of the box; the tail box ends rows in a group of 2."""
    for so in (4, 8):
        for shape in (KC.TTI_MULTI, KC.LONGX, *KC.TTI_EXACT.values()):
            assert (shape[2] + 2 * so) % 4 == 0
    for lo, hi in (KC.TTI_MULTI_TAIL, KC.TTI_MULTI_SUB):
        assert lo[2] % 4 == 0 and all(0 <= l <= h < n for l, h, n in zip(lo, hi, KC.TTI_MULTI))
    assert KC.box_extent(KC.TTI_MULTI_TAIL)[2] % 4 == 2
    assert KC.box_extent(KC.TTI_MULTI_SUB) == (11, 65, 352)


def test_seam_points():
    """KC.sparse_coordinates(seams=...) keeps the usual points first, then puts two points around every tile seam
    in y and z and every x-chunk seam, each half a cell away from it"""
    base = KC.sparse_coordinates(KC.TTI_MULTI)
    lo = KC.TTI_MULTI_SUB[0]
    pts = KC.sparse_coordinates(KC.TTI_MULTI, seams=(lo, (6, 11)))
    assert (pts[:len(base)] == base).all()
    idx = pts[len(base):] / KC.SPACING
    ys = {KC.TTI_MULTI_SUB[0][1] + ty * k for ty, _ in KC.TTI_SA_TILES.values() for k in (1, 2)}
    for d, cuts in ((0, (6, 11)), (1, ys), (2, (lo[2] + 64, lo[2] + 128))):
        for cut in cuts:
            for where in (cut - 0.5, cut + 0.5):
                assert abs(idx[:, d] - where).min() < 1e-4, (d, where)
