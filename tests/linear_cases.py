"""Inputs of the generic-update matrix (tests/test_linear_matrix.py on the GPU; tests/test_linear_ref.py and
tests/test_zz_emulation.py on the CPU).

A case is a seeded tap table, a time configuration and a box on a 1-D, 2-D or 3-D grid with anisotropic spacing
(the last nd entries of kernel_cases.SPACING). Shapes (301,), (45, 68) and (37, 45, 68): no x/y extent is a multiple
of k_linear's 4-row block and no z extent a multiple of its 64-wide block. Every slot and every halo cell starts as
white noise. K = 6 steps, so that even T = 5 slots rotate.

The equation is built with `f.subs` on the time and space dimensions. Part of each coefficient is written through
the Constant `a` (in two of every five taps), `b * dt` or a spacing (FACTORS); the numeric factor is chosen so that the
coefficient takes the table's value at the default values below. So a tap the recogniser drops, merges wrongly,
mis-signs or puts on the wrong axis changes the answer as much as a kernel bug does.
"""
import numpy as np

import kernel_cases as KC
import linear_ref as LR
from helpers import rel_linf

SHAPES = {1: (301,), 2: (45, 68), 3: (37, 45, 68)}
K = 6
TIME_M = 3                                       # steps TIME_M .. TIME_M + K - 1 (every configuration reads t - 3 at most)
TOL = 1e-5                                       # rel L-inf against float64 on the box of every slot

# name: (time_order, wshift, levels read)
TIMES = {
    'fwd1': (1, 1, (0,)),
    'fwd2': (2, 1, (0, -1)),
    'fwd4': (4, 1, (0, -1, -2, -3)),             # 4 levels, T = 5
    'bwd2': (2, -1, (0, 1)),
    'bwd3': (3, -1, (0, 1, 2)),
}
# tables: a star reaching exactly +-so on every axis; 64 distinct (level, offset) taps in [-so, so]^nd including every
# corner; a star with one access written twice (the recogniser must add the two coefficients)
STAR_SO = {1: (2, 8, 16), 2: (2, 4, 8), 3: (2, 4, 8)}
CLOUD_SO = {1: 32, 2: 4, 3: 2}
TABLES = ('star', 'cloud', 'merge')
BOXES = ('whole', 'interior', 'custom', 'override', 'point')

# every table with every time configuration on every grid, the boxes in turn, plus the other two star radii
MATRIX = ([(nd, tab, tm, BOXES[(i + nd) % len(BOXES)]) for nd in (1, 2, 3)
           for i, (tab, tm) in enumerate((tab, tm) for tab in TABLES for tm in TIMES)] +
          [(nd, ('star', so), tm, box) for nd in (1, 2, 3) for so, tm, box in
           zip((STAR_SO[nd][0], STAR_SO[nd][2]), ('fwd4', 'bwd3'), ('whole', 'point'))])


def case_id(m):
    nd, tab, tm, box = m
    return f"{nd}d-{tab if isinstance(tab, str) else f'{tab[0]}{tab[1]}'}-{tm}-{box}"


DEFAULTS = dict(a=0.75, b=1.25, dt=0.375)        # exact in float32, like the spacings
OVERRIDES = dict(a=0.625, b=1.5, dt=0.3125, h_x=9.0)


def spacing(nd):
    return tuple(KC.SPACING[3 - nd:])


def values(nd, **over):
    """The scalar environment of the coefficients: Constants, dt and spacings by name."""
    v = dict(DEFAULTS)
    v.update({'h_' + n: h for n, h in zip('xyz', spacing(nd))})
    v.update(over)
    return v


# the symbolic factor of tap k is FACTORS[k % 5]: a number, a Constant, a Constant times dt, a spacing, a Constant
# times a spacing; `a` is in two of every five taps
FACTORS = ('1', 'a', 'b*dt', '1/h0**2', 'a*hl')


def _factor_value(kind, v, nd):
    h0, hl = v['h_x'], v['h_' + 'xyz'[nd - 1]]
    return {'1': 1.0, 'a': v['a'], 'b*dt': v['b'] * v['dt'], '1/h0**2': 1.0 / h0 ** 2, 'a*hl': v['a'] * hl}[kind]


def table(kind, nd, so, levels, seed=0):
    """[(tshift, offsets, number, factor)]: the coefficient of a tap is number * factor, the coefficients at the
    default values have random signs and sum to 1.2 in absolute value."""
    rng = np.random.default_rng(seed + 1000 * nd + 10 * so + len(levels))
    acc = []
    if kind in ('star', 'merge'):
        for d in range(nd):
            for r in range(1, so + 1):
                for sgn in (1, -1):
                    o = [0] * nd
                    o[d] = sgn * r
                    acc.append((levels[0], tuple(o)))
        acc.insert(0, (levels[0], (0,) * nd))
        for s in levels[1:]:                       # the older levels: the centre and one random offset
            acc.append((s, (0,) * nd))
            acc.append((s, tuple(int(x) for x in rng.integers(-so, so + 1, nd))))
        if kind == 'merge':
            acc.append(acc[1])                     # written a second time (with another factor, below)
    else:
        corners = [tuple(so * (1 if (i >> d) & 1 else -1) for d in range(nd)) for i in range(2 ** nd)]
        acc = [(levels[0], c) for c in corners]
        seen = set(acc)
        while len(acc) < 64:
            t = (int(levels[rng.integers(len(levels))]), tuple(int(x) for x in rng.integers(-so, so + 1, nd)))
            if t not in seen:
                seen.add(t)
                acc.append(t)
    target = rng.uniform(0.5, 1.0, len(acc)) * rng.choice((-1.0, 1.0), len(acc))
    target *= 1.2 / np.abs(target).sum()
    kinds = [FACTORS[k % 5] for k in range(len(acc))]
    if kind == 'merge':
        kinds[-1] = '1/h0**2'
    v = values(nd)
    return [(s, o, float(c / _factor_value(fk, v, nd)), fk) for (s, o), c, fk in zip(acc, target, kinds)]


def coefficients(tab, nd, v):
    """The tap table the update applies at the scalar values v: float64, one entry per access (duplicates added),
    sorted by (tshift, offsets) like the recogniser's."""
    out = {}
    for s, o, num, kind in tab:
        out[(s, o)] = out.get((s, o), 0.0) + num * _factor_value(kind, v, nd)
    return [(s, o, c) for (s, o), c in sorted(out.items())]


def case(nd, tab, times, box, seed=0, shape=None):
    """One matrix case: tab in TABLES (or ('star', so)), times in TIMES, box in BOXES."""
    to, wshift, levels = TIMES[times]
    if isinstance(tab, tuple):
        tab, so = tab
    else:
        so = {'star': STAR_SO[nd][1], 'cloud': CLOUD_SO[nd], 'merge': 2}[tab]
    shape = shape or SHAPES[nd]
    rng = np.random.default_rng(seed + 7 * nd + 31 * so + 101 * to)
    f = rng.standard_normal((to + 1,) + tuple(n + 2 * so for n in shape)).astype(np.float32)
    return dict(nd=nd, so=so, shape=shape, time_order=to, wshift=wshift, levels=levels, box=box, f=f,
                table=table(tab, nd, so, levels, seed), time_m=TIME_M, time_M=TIME_M + K - 1)


def custom_spec(shape):
    """An asymmetric SubDomain: ('middle', 2, 5) on x, ('right', ny - 4) on y, ('left', nz - 7) on z."""
    spec = [('middle', 2, 5), ('right', shape[1] - 4) if len(shape) > 1 else None,
            ('left', shape[2] - 7) if len(shape) > 2 else None]
    return spec[:len(shape)]


def bounds(c):
    """(lo, hi) of the case's box, computed here rather than read from the operator, and the apply overrides it
    needs."""
    shape, box = c['shape'], c['box']
    lo, hi = [0] * len(shape), [n - 1 for n in shape]
    over = {}
    if box == 'interior':
        lo, hi = [1] * len(shape), [n - 2 for n in shape]
    elif box == 'custom':
        for d, (sp, n) in enumerate(zip(custom_spec(shape), shape)):
            if sp[0] == 'middle':
                lo[d], hi[d] = sp[1], n - 1 - sp[2]
            elif sp[0] == 'right':
                lo[d] = n - sp[1]
            else:
                hi[d] = sp[1] - 1
    elif box == 'override':
        lo[0], hi[0] = 3, shape[0] - 6
        over = dict(x_m=lo[0], x_M=hi[0])
    elif box == 'point':
        p = [1, shape[1] - 1 if len(shape) > 1 else 0, 0][:len(shape)]
        lo, hi = list(p), list(p)
        over = {f'{n}_{e}': x for n, x in zip('xyz', p) for e in ('m', 'M')}
    return lo, hi, over


def reference(c, v=None, mut=None, dtype=np.float64):
    lo, hi, _ = bounds(c)
    taps = coefficients(c['table'], c['nd'], v or values(c['nd']))
    return LR.run(c['f'], c['so'], taps, c['wshift'], lo, hi, c['time_m'], c['time_M'], mut=mut, dtype=dtype)


def written_slots(c):
    T = c['time_order'] + 1
    return {(t + c['wshift']) % T for t in range(c['time_m'], c['time_M'] + 1)}


def box_error(c, got, want):
    """rel L-inf difference on the case's box, in every slot (relative to the largest value there, so that a
    single-point box is not measured against one value that happens to be small)"""
    lo, hi, _ = bounds(c)
    box = (slice(None),) + LR.box_slices(lo, hi, c['so'])
    return rel_linf(got[box], want[box])


def check(c, got, want):
    """The box of every slot within TOL of float64; every cell outside the box, halo included, and every slot not
    written bit-identical to the input; the written boxes changed."""
    lo, hi, _ = bounds(c)
    box = LR.box_slices(lo, hi, c['so'])
    outside = np.ones(c['f'].shape[1:], dtype=bool)
    outside[box] = False
    assert box_error(c, got, want) < TOL
    written = written_slots(c)
    for s in range(c['f'].shape[0]):
        if s in written:
            assert np.array_equal(got[s][outside], c['f'][s][outside]), s
            assert not np.array_equal(got[s][box], c['f'][s][box]), s
        else:
            assert np.array_equal(got[s], c['f'][s]), s


def reaches_halo(c):
    """Whether some tap read from the box lands in the halo."""
    lo, hi, _ = bounds(c)
    return any(l + o[d] < 0 or h + o[d] > n - 1 for _, o, _, _ in c['table']
               for d, (l, h, n) in enumerate(zip(lo, hi, c['shape'])))


def build(c, name='u', grid_spacing=None):
    """(operator, field, Constants, grid) of the case's equation; the field holds the case's initial data."""
    from devito_b200 import Constant, Eq, Grid, Operator, SubDomain, TimeFunction
    nd, shape = c['nd'], c['shape']
    h = grid_spacing or spacing(nd)
    sds = []
    if c['box'] == 'custom':
        spec = custom_spec(shape)

        class Custom(SubDomain):
            name = 'custom'

            def define(self, dimensions):
                return dict(zip(dimensions, spec))
        sds.append(Custom())
    g = Grid(shape=shape, extent=tuple((n - 1) * x for n, x in zip(shape, h)), subdomains=sds)
    f = TimeFunction(name=name, grid=g, time_order=c['time_order'], space_order=c['so'])
    f.data_with_halo[:] = c['f']
    a = Constant(name='a', value=DEFAULTS['a'])
    b = Constant(name='b', value=DEFAULTS['b'])
    t, dims, hs = g.stepping_dim, g.dimensions, g.spacing_symbols
    dt = t.spacing
    sym = {'1': 1, 'a': a, 'b*dt': b * dt, '1/h0**2': 1 / hs[0] ** 2, 'a*hl': a * hs[-1]}
    rhs = None
    for s, o, num, kind in c['table']:
        acc = f.subs(t, t + s) if s else f
        for d, x in zip(dims, o):
            if x:
                acc = acc.subs(d, d + x)
        term = num * sym[kind] * acc
        rhs = term if rhs is None else rhs + term
    lhs = f.forward if c['wshift'] > 0 else f.backward
    sd = {'whole': None, 'override': None, 'point': None, 'interior': g.interior}.get(c['box'], None)
    if c['box'] == 'custom':
        sd = g.subdomains['custom']
    op = Operator([Eq(lhs, rhs, subdomain=sd)])
    return op, f, (a, b), g

