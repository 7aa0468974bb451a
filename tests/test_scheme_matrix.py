"""The schemes `b2_iso_forward` runs besides the plain forward step, against the float64 reference (tests/ref64.py)
on the anisotropic, non-cubic grid of tests/kernel_cases.py: adjoint, free surface, OT4, the imaging condition, Born,
snapshots (resident and streamed to the host), 2-D, and the streamed time loop of host-staged applies.

Operators are built with the DSL in the formulations of devito_b200/seismic/acoustic.py (`iso_stencil` forward and
backward, `Inc(grad, -u * v.dt2)`, Born's `q = -dm * u.dt2`, `u.biharmonic(1/m)`, `FreeSurface` on the
`physdomain` / `fsdomain` of a `SeismicModel(..., fs=True)`), so that the recogniser sees what the solvers build.
Every time slot (halo included), the traces, grad, U and the whole snapshot array are compared; unvisited snapshot
slots and the snapshot halo must keep their sentinel bit for bit. Each case asserts which sweep kernel ran.
Tolerances: rel L-inf 1e-5 for u and the snapshots, 1e-4 for U, Born traces and grad (tests/test_ref64.py pins
the reference against the C oracle at these bounds and shows what each kind of kernel bug would move).
"""
import ctypes
import functools

import numpy as np
import pytest

from helpers import rel_linf
import kernel_cases as KC
import ref64
from test_ref64 import OUT_TOL

pytestmark = pytest.mark.gpu

ADJOINT = ('adjoint', 'adjoint_fs', 'adjoint_ot4', 'grad')


def _last_kernel():
    from devito_b200 import _lib
    return _lib.lib().b2_last_sweep_kernel().decode()


def _last_call_streamed():
    from devito_b200 import _lib
    prof = (ctypes.c_double * 5)()
    _lib.lib().b2_last_call_profile(prof)
    return prof[4] == 1.0


def _grid(shape, fs, so):
    """The grid; with a free surface that of SeismicModel(fs=True): nbl = 4 around a physical grid 4 points
    shorter on top, origin chosen so that the extended grid starts at 0 like the KC sparse coordinates."""
    from devito_b200 import Grid
    sp = KC.SPACING[3 - len(shape):]
    if not fs:
        return Grid(shape=shape, extent=tuple((n - 1) * h for n, h in zip(shape, sp)))
    from devito_b200.seismic.model import SeismicModel
    nbl = 4
    phys = tuple(n - 2 * nbl for n in shape[:-1]) + (shape[-1] - nbl,)
    model = SeismicModel(origin=tuple(nbl * h for h in sp[:-1]) + (0.0,), spacing=sp, shape=phys, space_order=so,
                         vp=2.0, nbl=nbl, fs=True, bcs='damp')
    assert model.grid.shape == tuple(shape)
    assert all(float(o) == 0.0 for o in model.grid.origin)
    return model.grid


def _function(name, grid, so, values):
    from devito_b200 import Function
    f = Function(name=name, grid=grid, space_order=so)
    f.data_with_halo[:] = values
    return f


def _sparse(name, grid, tables, coords):
    from devito_b200 import SparseTimeFunction
    s = SparseTimeFunction(name=name, grid=grid, npoint=len(coords), nt=KC.K + 2,
                           interpolation='linear' if tables['r'] == 1 else 'sinc', r=tables['r'], coordinates=coords)
    s.data[:] = tables['data']
    return s


@functools.lru_cache(maxsize=None)
def _setup(scheme, so, param, box=None, dmh=0, interpolation='linear', shape=KC.SHAPE, rec_fwd=False):
    """(operator, {role: Function}, case, source tables); one operator per configuration."""
    from devito_b200 import (ConditionalDimension, Constant, Eq, FreeSurface, Function, Inc, Operator,
                             TimeFunction, solve)
    c = KC.scheme_case(scheme, so, param, box=box, dmh=dmh, shape=shape)
    fs = scheme in ('fs', 'adjoint_fs')
    grid = _grid(shape, fs, so)
    u = TimeFunction(name='v' if scheme in ADJOINT else 'u', grid=grid, time_order=2, space_order=so)
    damp = _function('damp', grid, so, c['damp'])
    kind, pv = c['param']
    if param == 'scalar':
        m = 1 / Constant(name='vp', value=float(pv)) ** 2
    elif kind == 'vp':
        m = 1 / _function('vp', grid, so, pv) ** 2
    else:
        m = _function('m', grid, so, pv)
    s = grid.time_dim.spacing
    dt = grid.stepping_dim.spacing

    def stencil(f, q=0):
        """seismic/acoustic.py::iso_stencil"""
        forward = scheme not in ADJOINT
        unext = f.forward if forward else f.backward
        lap = f.laplace + (s ** 2 / 12 * f.biharmonic(1 / m) if scheme in ('ot4', 'adjoint_ot4') else 0)
        pde = m * f.dt2 - lap - q + damp * (f.dt if forward else f.dt.T)
        if not fs:
            return [Eq(unext, solve(pde, unext))]
        update = Eq(unext, solve(pde, unext), subdomain=grid.subdomains['physdomain'])
        return [update, FreeSurface(update, grid.subdomains['fsdomain'])]

    roles = {'u': u}
    tables, src, rec = None, None, None
    if len(shape) == 3:
        coords = KC.sparse_coordinates(shape)
        tables = KC.sparse_tables(coords, interpolation, KC.K + 2)
        src = _sparse('src', grid, tables, coords)
        if scheme != 'grad':
            rec = _sparse('rec', grid, tables, coords)
    eqs = stencil(u) if scheme != 'born' else []
    if scheme in ADJOINT:
        eqs += src.inject(field=u.backward, expr=src * dt ** 2 / m)
        if rec is not None:
            eqs += rec.interpolate(expr=u)
    elif scheme == 'born':
        U = TimeFunction(name='U', grid=grid, time_order=2, space_order=so)
        dm = Function(name='dm', grid=grid, space_order=dmh)
        dm.data_with_halo[:] = c['dm']
        roles.update(U=U)
        eqs = stencil(u) + src.inject(field=u.forward, expr=src * dt ** 2 / m) + stencil(U, q=-dm * u.dt2) + \
            rec.interpolate(expr=U)
    elif src is not None:
        eqs += src.inject(field=u.forward, expr=src * dt ** 2 / m)
    if scheme == 'grad':
        usave = TimeFunction(name='u', grid=grid, time_order=2, space_order=so, save=KC.K + 2)
        usave.data_with_halo[:] = c['usave']
        grad = Function(name='grad', grid=grid)
        roles.update(grad=grad)
        eqs.append(Inc(grad, -usave * u.dt2))
    if scheme in ('snap', 'snap_fwd'):
        t_sub = ConditionalDimension('t_sub', parent=grid.time_dim, factor=KC.SNAP_FACTOR)
        snap = TimeFunction(name='usave', grid=grid, time_order=2, space_order=KC.SNAP_HALO,
                            save=c['snap'].shape[0], time_dim=t_sub)
        roles.update(snap=snap)
        eqs.append(Eq(snap, u.forward if scheme == 'snap_fwd' else u))
    if scheme not in ADJOINT + ('born',) and rec is not None:
        eqs += rec.interpolate(expr=u.forward if rec_fwd else u)
    op = Operator(eqs)
    assert op.backend == 'cuda-sm90a', getattr(op, '_why_not', None)
    if rec is not None:
        roles['rec'] = rec
    if src is not None:
        roles['src'] = src
    return op, roles, c, tables


@functools.lru_cache(maxsize=None)
def _reference(key):
    _, roles, c, tables = _setup(*key)
    rec = dict(tables, data=np.zeros_like(tables['data'])) if 'rec' in roles else None
    return KC.scheme_reference(c, src=tables, rec=rec)


def _apply(key, expect, src_data=None, **kw):
    """Reset every input (the source traces to `src_data` if given), apply for time 1..K, assert the kernel; the
    outputs as float arrays."""
    op, roles, c, tables = _setup(*key)
    roles['u'].data_with_halo[:] = c['u']
    if 'src' in roles:
        roles['src'].data[:] = tables['data'] if src_data is None else src_data
    for r in ('U', 'grad', 'snap'):
        if r in roles:
            roles[r].data_with_halo[:] = c[r]
    if 'rec' in roles:
        roles['rec'].data[:] = 0.0
    nd = len(c['shape'])
    bounds = {f'{a}_m': l for a, l in zip('xyz'[:nd], c['lo'])}
    bounds.update({f'{a}_M': h for a, h in zip('xyz'[:nd], c['hi'])})
    op.apply(time_m=1, time_M=KC.K, dt=c['dt'], **bounds, **kw)
    assert _last_kernel() == expect
    out = {r: np.array(f.data_ro_with_halo if r != 'rec' else f.data) for r, f in roles.items() if r != 'src'}
    out['traces'] = out.pop('rec', None)
    return out


def _check(key, expect, **kw):
    got = _apply(key, expect, **kw)
    want = _reference(key)
    scheme = key[0]
    assert np.abs(got['u']).max() > 0.5
    for r, w in want.items():
        if w is None:
            continue
        tol = 1e-4 if scheme == 'born' and r == 'traces' else OUT_TOL[r]
        err = rel_linf(got[r], w)
        assert err < tol, f"{r}: {err:.2e}"
    if 'snap' in want:
        visited = want['snap'] != KC.SNAP_SENTINEL
        assert np.all(got['snap'][~visited] == np.float32(KC.SNAP_SENTINEL))
    return got


PARAMS = ['scalar', 'vp', 'm']
PK = {'scalar': 'scalar', 'vp': 'vp', 'm': 'm'}
# tail3: a z extent of 59, every row ending in a partial float4 group
BOXES = dict(full=None, sub=KC.SUBBOX, tail3=KC.ZTAIL['tail3'])


def _tma(so, param):
    return f'iso_tma<{so // 2},{PK[param]}>'


@pytest.mark.parametrize('kernel', ['generic', 'tma'])
@pytest.mark.parametrize('param', PARAMS)
@pytest.mark.parametrize('so', [4, 8, 16])
def test_adjoint(so, param, kernel):
    """Time reversed: sources into u[t-1], receivers from u[t]."""
    key = ('adjoint', so, param, None, 0, 'sinc' if so >= 8 else 'linear')
    if kernel == 'generic':
        _check(key, 'iso_generic', kernel=1)
    else:
        _check(key, _tma(so, param))


@pytest.mark.parametrize('scheme,expect', [('adjoint_fs', 'iso_tma<4,vp>'), ('adjoint_ot4', 'iso_generic')])
def test_adjoint_free_surface_and_ot4(scheme, expect):
    _check((scheme, 8, 'vp', None, 0, 'sinc'), expect)


@pytest.mark.parametrize('box', list(BOXES))
@pytest.mark.parametrize('kernel', ['generic', 'tma'])
def test_gradient(kernel, box):
    """Imaging condition into a grad with halo 1, after each adjoint step and its injection."""
    key = ('grad', 8, 'vp', BOXES[box], 0, 'sinc')
    if kernel == 'generic':
        _check(key, 'iso_generic', kernel=1)
    else:
        _check(key, 'iso_tma<4,vp>')


@pytest.mark.parametrize('box', list(BOXES))
@pytest.mark.parametrize('dmh', [0, 3])
@pytest.mark.parametrize('kernel', ['generic', 'tma'])
@pytest.mark.parametrize('param', ['vp', 'm'])
@pytest.mark.parametrize('so', [4, 8])
def test_born(so, param, kernel, dmh, box):
    key = ('born', so, param, BOXES[box], dmh, 'sinc' if so >= 8 else 'linear')
    if kernel == 'generic':
        _check(key, 'iso_generic', kernel=1)
    else:
        _check(key, _tma(so, param))


@pytest.mark.parametrize('interpolation', ['linear', 'sinc'])
@pytest.mark.parametrize('kernel', ['generic', 'tma'])
@pytest.mark.parametrize('param', ['scalar', 'vp'])
@pytest.mark.parametrize('so', [4, 8])
def test_free_surface(so, param, kernel, interpolation):
    """Sources and receivers next to the surface (z = 0.4 cells) and just above it (z = -1.6 cells, supports in
    the halo above the surface)."""
    key = ('fs', so, param, None, 0, interpolation)
    if kernel == 'generic':
        _check(key, 'iso_generic', kernel=1)
    else:
        _check(key, _tma(so, param))


@pytest.mark.parametrize('box', ['full', 'sub'])
@pytest.mark.parametrize('param', PARAMS)
@pytest.mark.parametrize('so', [4, 8, 16])
def test_ot4(so, param, box):
    """Two-pass generic kernels (k_ot4_w on the box grown by R, then the update with lap(W)): its only kernel."""
    _check(('ot4', so, param, KC.SUBBOX if box == 'sub' else None, 0, 'sinc' if so >= 8 else 'linear'),
           'iso_generic')


@pytest.mark.parametrize('box', ['full', 'sub'])
@pytest.mark.parametrize('stream', ['0', '1'])
@pytest.mark.parametrize('scheme', ['snap', 'snap_fwd'])
def test_snapshots(scheme, stream, box, monkeypatch):
    """Eq(usave, u) / Eq(usave, u.forward), factor 2, snapshot halo 3, host-resident snapshots: B2_SNAP_STREAM=1
    drains box by box on a copy stream (cudaMemcpy3DAsync), 0 stages the whole array."""
    monkeypatch.setenv('B2_SNAP_STREAM', stream)
    _check((scheme, 8, 'vp', KC.SUBBOX if box == 'sub' else None), 'iso_tma<4,vp>', resident=False)


def test_snapshots_resident():
    _check(('snap', 8, 'vp', KC.SUBBOX), 'iso_tma<4,vp>')


@pytest.mark.parametrize('scheme', ['plain', 'fs', 'snap'])
@pytest.mark.parametrize('param', ['scalar', 'vp'])
def test_2d(scheme, param):
    """2-D grid (45, 68), spacing (12.5, 8): the generic kernel with a unit x axis."""
    _check((scheme, 8, param, None, 0, 'linear', KC.SHAPE[1:]), 'iso_generic', resident=scheme != 'snap')


# ---------------------------------------------------------------------------------------------------------------
# The streamed time loop of host-staged applies (b2_api_iso.cu::iso_forward_streamed), forced on this small grid
# ---------------------------------------------------------------------------------------------------------------
def _disjoint_source_traces(c, tables):
    """The source traces with every point zeroed whose support shares a cell with an earlier kept point: each cell
    then receives at most one deposit per step, so the result does not depend on the order of the atomics."""
    S = ref64._Support(tables, c['lo'], c['hi'], c['so'])
    flat = np.ravel_multi_index(S.idx, c['u'].shape[1:])
    used, data = set(), np.array(tables['data'])
    for p in range(S.npoint):
        cells = set(flat[S.p == p].tolist())
        if cells & used:
            data[:, p] = 0.0
        used |= cells
    return data


@pytest.mark.parametrize('rec_fwd', [False, True], ids=['rec_u', 'rec_u_forward'])
@pytest.mark.parametrize('interpolation', ['linear', 'sinc'])
@pytest.mark.parametrize('box', list(BOXES))
@pytest.mark.parametrize('so', [4, 8])
@pytest.mark.parametrize('dim', [0, 1])
def test_streamed_loop(dim, so, box, interpolation, rec_fwd, monkeypatch):
    """Chunks of 12 planes (16 at so = 8) cut along x (dim 0) or y (dim 1); the KC points sit on the cuts' faces.
    With SUBBOX the box starts at x = 1, y = 2: every range, upload and download is offset by that origin; tail3
    starts there too and ends every row in a partial float4 group, which every range must keep.
    Against float64 with every KC point; against the resident apply bit for bit with the points whose supports
    overlap switched off (deposits of two points into one cell are atomics in either order, which moves the last
    bit); the traces up to the order of the partial sums."""
    key = ('plain', so, 'vp', BOXES[box], 0, interpolation, KC.SHAPE, rec_fwd)
    _, _, c, tables = _setup(*key)
    resident = _apply(key, _tma(so, 'vp'))
    assert not _last_call_streamed()
    monkeypatch.setenv('B2_STREAM', '2')
    monkeypatch.setenv('B2_STREAM_W', '12')
    monkeypatch.setenv('B2_STREAM_DIM', str(dim))
    got = _apply(key, _tma(so, 'vp'), resident=False)
    assert _last_call_streamed()
    w64 = [ref64.fd2_weights(so, h) for h in KC.SPACING]
    want, traces = ref64.iso_forward(c['u'], so, w64, c['dt'], 1, KC.K, damp=c['damp'], param=c['param'],
                                     lo=c['lo'], hi=c['hi'], src=tables, rec=dict(tables, data=np.zeros_like(
                                         tables['data'])), rec_toff=int(rec_fwd))
    assert rel_linf(got['u'], want) < KC.TOL['iso']
    assert rel_linf(got['traces'], traces) < KC.TOL['iso']
    assert rel_linf(got['u'], resident['u']) < 1e-6
    assert rel_linf(got['traces'], resident['traces']) < 1e-6
    data = _disjoint_source_traces(c, tables)
    assert np.count_nonzero(data.any(axis=0)) >= 10
    got = _apply(key, _tma(so, 'vp'), src_data=data, resident=False)
    assert _last_call_streamed()
    resident = _apply(key, _tma(so, 'vp'), src_data=data)
    assert not _last_call_streamed()
    assert np.array_equal(got['u'], resident['u'])
    assert rel_linf(got['traces'], resident['traces']) < 1e-6
