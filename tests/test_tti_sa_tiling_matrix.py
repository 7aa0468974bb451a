"""The TTI and self-adjoint (SA) sweeps against float64 on grids that cut them into several y- and z-tiles, on grids of
full tiles only, and with the x-chunks the default selection picks on a grid long in x.

The layouts (tests/kernel_cases.py; tests/test_tti_sa_tiling.py checks the tilings they give every sweep):
- multi: TTI_MULTI (13, 71, 364): 3 to 5 y-tiles and 6 z-tiles for every sweep, the last of each partial, and never as
  many y-tiles as z-tiles, so exchanged tile counts or origins visit other tiles;
- multi_tail: the box TTI_MULTI_TAIL on it, z extent 362: every row ends in a partial float4 group of 2;
- multi_sub: the box TTI_MULTI_SUB, y extent 65 (a last y-tile of one row for TY 32 and 16), z extent 352;
- exact: (9, 3 TY, 256) for the sweep's tile height TY: 3 x 4 full tiles;
- longx: LONGX (150, 30, 64) with nothing forced: the default x-chunks (38, 38, 38, 36 planes on 132 SMs).
The multi layouts run with B2_TTI_LX=5 (x-chunks of 5 planes, the last partial) and, for forward and Born, also without
(one chunk); exact runs with B2_TTI_LX=5. The SA sweep has no chunk switch. Every time slot holds white noise, halo
included, as in the other matrices, and the sources and receivers include points half a cell either side of every
tile and x-chunk seam (KC.sparse_coordinates(seams=...)). The builders are those of test_kernel_matrix (forward),
test_tti_adjoint_matrix, test_tti_born_matrix and test_sa_matrix; the float64 result of a (configuration, layout) is
computed once and shared by its B2_TTI_LX settings. Every case asserts the sweep that ran. Tolerance: rel L-inf 1e-4
(TTI) and 1e-5 (SA), traces and srca included.
"""
import pytest

import kernel_cases as KC
import test_kernel_matrix as KM
import test_sa_matrix as SAM
import test_tti_adjoint_matrix as ADJ
import test_tti_born_matrix as BORN

pytestmark = pytest.mark.gpu

MULTI = {'multi': None, 'multi_tail': KC.TTI_MULTI_TAIL, 'multi_sub': KC.TTI_MULTI_SUB}


def _layout(layout, tiles):
    """(shape, box, seams) of a layout; `tiles`: the KC.TILES name whose exact grid 'exact' means"""
    if layout in MULTI:
        shape, box = KC.TTI_MULTI, MULTI[layout]
    elif layout == 'exact':
        shape, box = KC.TTI_EXACT[tiles], None
    else:
        shape, box = KC.LONGX, None
    lo, hi = box if box is not None else ((0, 0, 0), tuple(n - 1 for n in shape))
    lx = KC.LONGX_LX if layout == 'longx' else 5
    return shape, box, (tuple(lo), tuple(range(lo[0] + lx, hi[0] + 1, lx)))


def _env(monkeypatch, lx, env):
    if lx is not None:
        monkeypatch.setenv('B2_TTI_LX', str(lx))
    for k, val in env.items():
        monkeypatch.setenv(k, val)


# (so, arrays, environment) of the default selection of every fused TTI sweep
SWEEPS = {
    'tti_fused<2>': (4, False, {}),
    'tti_fused<4>': (8, False, {'B2_TTI_KERNEL': '2'}),
    'tti_ws<pf1>': (8, False, {}),
    'tti_arr_ct2<2>': (4, True, {}),
    'tti_arr_ct2<4>': (8, True, {}),
}
FWD_LAYOUTS = [(layout, lx) for layout in MULTI for lx in (5, None)] + [('exact', 5), ('longx', None)]


def _lx_id(lx):
    return f'lx{lx}' if lx else 'default'


@pytest.mark.parametrize('layout,lx', FWD_LAYOUTS, ids=[f'{a}-{_lx_id(b)}' for a, b in FWD_LAYOUTS])
@pytest.mark.parametrize('sweep', list(SWEEPS))
def test_tti_forward(sweep, layout, lx, monkeypatch):
    """u, v (every slot, halo included) and the traces of u + v"""
    so, arrays, env = SWEEPS[sweep]
    _env(monkeypatch, lx, env)
    shape, box, seams = _layout(layout, sweep)
    KM._check_tti(('tti', so, arrays, box, shape, seams), sweep)


@pytest.mark.parametrize('layout', ['multi', 'multi_tail', 'multi_sub', 'longx'])
@pytest.mark.parametrize('so,arrays', [(4, False), (8, True)], ids=['so4-scalar', 'so8-arr'])
def test_tti_two_pass_control(so, arrays, layout):
    """The two-pass sweep (no yz-tiles) on the same layouts and inputs: the control of the fused sweeps above."""
    shape, box, seams = _layout(layout, None)
    KM._check_tti(('tti', so, arrays, box, shape, seams), 'tti_two_pass', kernel=1)


ADJ_SWEEPS = [
    # (so, arrays, environment, sweep variant)
    (4, False, {}, 'tti_fused<2>+adj'),
    (8, False, {'B2_TTI_KERNEL': '2'}, 'tti_fused<4>+adj'),
    (8, False, {}, 'tti_fused<4>+adj'),          # the forward runs k_tti_ws here
    (4, True, {}, 'tti_arr_ct2<2>+adj'),
    (8, True, {}, 'tti_arr_ct2<4>+adj'),
]


@pytest.mark.parametrize('layout', list(MULTI) + ['exact'])
@pytest.mark.parametrize('gradient', [False, True], ids=['adjoint', 'gradient'])
@pytest.mark.parametrize('so,arrays,env,sweep', ADJ_SWEEPS,
                         ids=[f"{v[3]}-{'-'.join(v[2].values()) or 'default'}" for v in ADJ_SWEEPS])
def test_tti_adjoint(so, arrays, env, sweep, gradient, layout, monkeypatch):
    """p, r and srca (adjoint) or p, r and grad (gradient), B2_TTI_LX=5"""
    _env(monkeypatch, 5, env)
    shape, box, seams = _layout(layout, sweep.split('+')[0])
    ADJ._check((so, arrays, gradient, box, shape, seams), sweep, kernel=0)


@pytest.mark.parametrize('layout,lx', FWD_LAYOUTS, ids=[f'{a}-{_lx_id(b)}' for a, b in FWD_LAYOUTS])
@pytest.mark.parametrize('sweep', list(SWEEPS))
def test_tti_born(sweep, layout, lx, monkeypatch):
    """u0, v0, du, dv and the traces of du + dv; dm without halo"""
    so, arrays, env = SWEEPS[sweep]
    _env(monkeypatch, lx, env)
    shape, box, seams = _layout(layout, sweep)
    BORN._check((so, arrays, box, 0, shape, seams), sweep, kernel=0)


@pytest.mark.parametrize('layout', list(MULTI) + ['exact'])
@pytest.mark.parametrize('adjoint', [False, True], ids=['fwd', 'adj'])
@pytest.mark.parametrize('so', [4, 8])
def test_sa(so, adjoint, layout):
    """u (every slot, halo included) and the traces, array parameters"""
    shape, box, seams = _layout(layout, f'sa_tma<{so // 2}>')
    sweep = f'sa_tma<{so // 2}>' + ('+adj' if adjoint else '')
    SAM._check((so, True, adjoint, 3, shape, seams), sweep, box or 'full', kernel=0)
