"""The self-adjoint variable-density visco-acoustic update (`b2_sa_forward`) against the float64 restatement
(tests/sa_ref.py) on the anisotropic, non-cubic grid of tests/kernel_cases.py: (37, 45, 68), spacing (10, 12.5, 8).

The operators are built with the DSL in the formulation of devito_b200/seismic/self_adjoint.py (`iso_stencil`, the
sources injected with dt^2 vp^2/b into the level written, receivers sampling u). Every time slot starts as white
noise, halo included; b, vp and w/Q are positive white noise (or scalars). The sparse points of
kernel_cases.sparse_coordinates reach into the halo and beyond the grid. Each case asserts from `b2_last_sweep_kernel`
which sweep variant ran. Tolerance: rel L-inf 1e-5 for u and the traces.
"""
import functools
from types import SimpleNamespace

import numpy as np
import pytest

from helpers import rel_linf
import kernel_cases as KC
import sa_ref as SA

pytestmark = pytest.mark.gpu

TOL = 1e-5
DT = 0.9


def _last_kernel():
    from devito_b200 import _lib
    return _lib.lib().b2_last_sweep_kernel().decode()


def sa_case(so, arrays, nd=3, seed=0, shape=None):
    shape = shape or (KC.SHAPE if nd == 3 else (KC.SHAPE[0], KC.SHAPE[2]))
    alloc = tuple(n + 2 * so for n in shape)
    rng = np.random.default_rng(seed + 10 * so + nd)
    c = dict(so=so, shape=shape, spacing=KC.SPACING if nd == 3 else (KC.SPACING[0], KC.SPACING[2]))
    c['u'] = rng.standard_normal((3,) + alloc).astype(np.float32)
    c['b'] = rng.uniform(0.4, 1.2, alloc).astype(np.float32) if arrays else np.float32(0.7)
    c['vp'] = rng.uniform(1.5, 3.0, alloc).astype(np.float32) if arrays else np.float32(2.2)
    c['w'] = rng.uniform(0.0, 0.3, alloc).astype(np.float32)
    return c


@functools.lru_cache(maxsize=None)
def _setup(so, arrays, adjoint, nd=3, shape=None, seams=None):
    """(operator, u, rec, case, source tables); `seams` (3-D): KC.sparse_coordinates' points beside the tile and
    x-chunk seams, added to its usual points"""
    from devito_b200 import Constant, Function, Grid, Operator, SparseTimeFunction, TimeFunction
    from devito_b200.seismic.self_adjoint import iso_stencil
    c = sa_case(so, arrays, nd, shape=shape)
    grid = Grid(shape=c['shape'], extent=tuple((n - 1) * h for n, h in zip(c['shape'], c['spacing'])))

    def param(name, values):
        if np.ndim(values) == 0:
            return Constant(name=name, value=float(values))
        f = Function(name=name, grid=grid, space_order=so)
        f.data_with_halo[:] = values
        return f
    model = SimpleNamespace(vp=param('vp', c['vp']), b=param('b', c['b']), damp=param('damp', c['w']), grid=grid)
    u = TimeFunction(name='u', grid=grid, time_order=2, space_order=so)
    eqs = iso_stencil(u, model, forward=not adjoint)
    interpolation = 'sinc' if so >= 8 else 'linear'
    coords = KC.sparse_coordinates(shape=c['shape'], seams=seams) if nd == 3 else KC.sparse_coordinates()
    if nd == 2:
        coords = np.ascontiguousarray(coords[:, [0, 2]])
    tables = sparse_tables(coords, interpolation, KC.K + 2, c['spacing'])
    sp = lambda n: SparseTimeFunction(name=n, grid=grid, npoint=len(coords), nt=KC.K + 2, interpolation=interpolation,
                                      r=tables['r'], coordinates=coords)
    src, rec = sp('src'), sp('rec')
    src.data[:] = tables['data']
    dt = grid.stepping_dim.spacing
    eqs += src.inject(field=u.backward if adjoint else u.forward, expr=src * dt ** 2 * model.vp ** 2 / model.b)
    eqs += rec.interpolate(expr=u)
    op = Operator(eqs)
    assert op.backend == 'cuda-sm90a', op._why_not
    return op, u, rec, c, tables


def sparse_tables(coords, interpolation, nt, spacing):
    from oracle import oracle as O
    r = 1 if interpolation == 'linear' else 4
    gp, ws = O.tabulate(coords, (0.0,) * len(spacing), spacing, r, interpolation, dtype=np.float64)
    rng = np.random.default_rng(11)
    return dict(data=rng.standard_normal((nt, coords.shape[0])).astype(np.float32), gp=gp, w=ws, r=r)


def _reference(key, lo, hi):
    _, _, _, c, tables = _setup(*key)
    so = c['so']
    weights = [SA.sa_weights(so // 2, h) for h in c['spacing']]
    return SA.sa_forward(c['u'], so, weights, DT, 1, KC.K, c['b'], c['vp'], c['w'], lo=lo, hi=hi, src=tables,
                         rec=dict(tables, data=np.zeros_like(tables['data'])), adjoint=key[2])


def _check(key, sweep, box, **kw):
    """box: 'full', a name of KC.BOXES (3-D; 2-D: an interior box) or a 3-D (lo, hi)"""
    op, u, rec, c, _ = _setup(*key)
    u.data_with_halo[:] = c['u']
    rec.data[:] = 0.0
    nd = len(c['shape'])
    if box == 'full':
        lo, hi = [0] * nd, [n - 1 for n in c['shape']]
    elif nd == 3:
        lo, hi = map(list, KC.BOXES[box] if isinstance(box, str) else box)
    else:
        lo, hi = [1, 4], [c['shape'][0] - 3, c['shape'][1] - 9]
    bounds = {}
    for d, l, h in zip('xyz', lo, hi):
        bounds[f'{d}_m'], bounds[f'{d}_M'] = l, h
    op.apply(time_m=1, time_M=KC.K, dt=DT, **bounds, **kw)
    assert _last_kernel() == sweep
    want_u, want_rec = _reference(key, lo, hi)
    assert rel_linf(np.array(u.data_ro_with_halo), want_u) < TOL
    assert rel_linf(np.array(rec.data), want_rec) < TOL


CASES = [
    # (so, arrays, adjoint, nd, kernel=): kernel 0 picks sa_tma<R> on these 3-D so=4 / so=8 layouts (z extent and z
    # start multiples of 4), k_sa_generic otherwise; the (37, 45, 68) grid cuts into 3 x 2 yz-tiles of 16 x 64, the
    # last of each partial, and the interior box shifts and shortens them
    (4, True, False, 3, 0), (8, True, False, 3, 0), (4, True, True, 3, 0), (8, True, True, 3, 0),
    (4, False, False, 3, 2), (8, False, True, 3, 2),
    (4, True, False, 3, 1), (8, True, True, 3, 1), (8, False, False, 3, 1),
    (8, True, False, 2, 0), (4, True, True, 2, 1), (16, True, False, 3, 0),
]


def _variant(so, nd, kernel, adjoint):
    name = f'sa_tma<{so // 2}>' if nd == 3 and so in (4, 8) and kernel != 1 else 'sa_generic'
    return name + ('+adj' if adjoint else '')


def _case_id(c):
    return f"so{c[0]}-{'arr' if c[1] else 'scalar'}-{'adj' if c[2] else 'fwd'}-{c[3]}d-k{c[4]}"


# 3-D cases also run the z-tail boxes of kernel_cases.ZTAIL: every row ends in a partial float4 group
SA_BOXES = [pytest.param(c, box, id=f'{_case_id(c)}-{box}') for c in CASES
            for box in ['full', 'sub'] + (list(KC.ZTAIL) if c[3] == 3 else [])]


@pytest.mark.parametrize('case,box', SA_BOXES)
def test_sa_kernel(case, box):
    so, arrays, adjoint, nd, kernel = case
    _check((so, arrays, adjoint, nd), _variant(so, nd, kernel, adjoint), box, kernel=kernel)


@pytest.mark.parametrize('box', list(KC.TINY) + ['xplane'])
@pytest.mark.parametrize('adjoint', [False, True], ids=['fwd', 'adj'])
@pytest.mark.parametrize('so', [4, 8])
def test_tma_tiny_boxes(so, adjoint, box):
    """sa_plan_init has no size gate: boxes of (1, 1, 1), (1, 1, 4) and (2, 5, 7) points at the corners and inside,
    and one x-plane, run the TMA sweep."""
    _check((so, True, adjoint, 3), _variant(so, 3, 0, adjoint), box)


def test_tma_and_generic_agree():
    """The two sweeps on the same so=8 case, forward: both within 1e-5 of float64 and of each other."""
    key = (8, True, False, 3)
    op, u, rec, c, _ = _setup(*key)
    out = {}
    for kernel in (1, 2):
        u.data_with_halo[:] = c['u']
        rec.data[:] = 0.0
        op.apply(time_m=1, time_M=KC.K, dt=DT, kernel=kernel)
        out[kernel] = (np.array(u.data_ro_with_halo), np.array(rec.data))
    assert rel_linf(out[2][0], out[1][0]) < TOL and rel_linf(out[2][1], out[1][1]) < TOL


@pytest.mark.parametrize('adjoint', [False, True], ids=['fwd', 'adj'])
def test_tma_several_x_chunks(adjoint):
    """A grid long in x and small in y/z: the sweep is cut into several x-chunks (CTAs marching the same yz-tile over
    consecutive x-ranges, each re-reading 4R - 2 priming planes)."""
    _check((8, True, adjoint, 3, (150, 20, 24)), 'sa_tma<4>' + ('+adj' if adjoint else ''), 'full')


def test_forced_tma_on_a_layout_it_does_not_take_is_refused():
    """kernel=2 on a 2-D grid (the TMA sweep is 3-D only) fails with a message instead of running another kernel."""
    from devito_b200.exceptions import ExecutionError
    op, u, rec, c, _ = _setup(8, True, False, 2)
    u.data_with_halo[:] = c['u']
    with pytest.raises(ExecutionError, match='TMA kernel forced'):
        op.apply(time_m=1, time_M=KC.K, dt=DT, kernel=2)
