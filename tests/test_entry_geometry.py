"""How a call's iteration box becomes device geometry, and what the wave entry points check around their time loop.

CPU (tests/support/emu_box.cu, nvcc host build): the box of `x_m .. z_M` in the internal 3-dim convention (a 1-D or
2-D grid gets leading dummy dims of extent 1) against numpy's own view of that box, and the reach rule of the wave
calls: a box grown by the stencil's reach (iso: radius r, TTI: R, SA and SLS: 2R-1) must stay inside the allocation,
dim 0, 1, 2 in turn, where an empty extent means "nothing to do".

GPU, called through the ABI on tiny 2-D and 3-D grids (host arrays, `dmap` NULL): for b2_iso_forward, b2_tti_forward,
b2_sa_forward and b2_visco_forward, a box whose reach passes the allocation by one cell is refused (210) with every
host array byte-identical, the box one cell smaller matches the float64 references (ref64, tti2d_ref, sa_ref,
visco_ref), an empty box writes nothing, and a sparse radius beyond the halo is refused; errctl stops TTI, SA and SLS
on an Inf (100) and still writes the arrays back; the timers report section0 for TTI, SA and the linear update.
"""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

import ref64
import sa_ref
import tti2d_ref
import visco_ref
from helpers import rel_linf
from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B2_OK, B2_ERR_NAN, B2_ERR_INVALID = 0, 100, 210


# ---- CPU: the box and the reach rule ---------------------------------------------------------------------------

@pytest.fixture(scope='module')
def emu(tmp_path_factory):
    if shutil.which('nvcc') is None:
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp('emu_box') / 'libemu_box.so'
    cmd = ['nvcc', '-O1', '-std=c++17', '-shared', '-Xcompiler', '-fPIC', '-I', os.path.join(ROOT, 'include'),
           '-I', os.path.join(ROOT, 'devito_b200', 'csrc'), os.path.join(ROOT, 'tests', 'support', 'emu_box.cu'),
           '-o', str(out)]
    env = dict(os.environ)
    env.pop('CC', None)
    r = subprocess.run(cmd, capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    lib = ctypes.CDLL(str(out))
    ip = ctypes.POINTER(ctypes.c_int)
    lib.emu_make_box.argtypes = [ip, ip, ctypes.c_int, ip, ctypes.c_int, ctypes.POINTER(ctypes.c_longlong)]
    lib.emu_check_reach.argtypes = [ctypes.c_char_p, ip, ip, ctypes.c_int, ip, ctypes.c_int, ctypes.c_int, ip]
    lib.emu_last_error.restype = ctypes.c_char_p
    return lib


def _ints(v):
    v = list(v) + [0] * (3 - len(v)) if len(v) < 3 else list(v)
    return (ctypes.c_int * len(v))(*v)


def _make_box(emu, lo, hi, size, halo):
    out = (ctypes.c_longlong * 14)()
    emu.emu_make_box(_ints(lo), _ints(hi), len(lo), _ints(size), halo, out)
    v = list(out)
    return dict(a=v[0:3], n=v[3:6], o=v[6:9], sx=v[9], sy=v[10], slot_elems=v[11], tsize=v[12], so=v[13])


def _reach(emu, lo, hi, size, halo, reach, who=b'b2_test'):
    empty = ctypes.c_int(-1)
    rc = emu.emu_check_reach(who, _ints(lo), _ints(hi), len(lo), _ints(size), halo, reach, ctypes.byref(empty))
    return rc, empty.value, emu.emu_last_error().decode()


BOXES = {
    1: ((23,), 2, (3,), (17,)),
    2: ((11, 19), 4, (-2, 1), (9, 16)),
    3: ((7, 10, 13), 3, (1, -1, 0), (5, 11, 12)),
}


@pytest.mark.parametrize('nd', [1, 2, 3])
def test_box_layout(emu, nd):
    """extents, origins, strides and slot size against numpy's view of the box in a (T, space...) array"""
    shape, halo, lo, hi = BOXES[nd]
    alloc = tuple(n + 2 * halo for n in shape)
    u = np.zeros((4,) + alloc, dtype=np.float32)
    b = _make_box(emu, lo, hi, (4,) + alloc, halo)
    slot = u[0].reshape((1,) * (3 - nd) + alloc)                    # the internal 3-dim convention
    view = slot[(slice(None),) * (3 - nd) + tuple(slice(l + halo, h + halo + 1) for l, h in zip(lo, hi))]
    assert b['a'] == list(slot.shape)
    assert b['n'] == list(view.shape)
    first = (view.ctypes.data - slot.ctypes.data) // 4
    assert first == b['o'][0] * b['sx'] + b['o'][1] * b['sy'] + b['o'][2]
    assert [b['o'][d] for d in range(3 - nd)] == [0] * (3 - nd)
    assert [b['sx'], b['sy'], 1] == [s // 4 for s in slot.strides]
    assert b['slot_elems'] == u[0].size and b['tsize'] == 4 and b['so'] == halo


# reach of each wave update at space order 8: (name, reach)
RULES = [('iso', 4), ('tti', 4), ('sa', 2 * 4 - 1), ('visco', 2 * 4 - 1), ('iso_r1', 1)]


@pytest.mark.parametrize('rule,reach', RULES, ids=[r for r, _ in RULES])
@pytest.mark.parametrize('nd', [1, 2, 3])
def test_reach_touching_and_one_past(emu, nd, rule, reach):
    so = 8
    shape = (12, 15, 17)[:nd]
    size = (3,) + tuple(n + 2 * so for n in shape)
    lo = [reach - so] * nd                                          # the reach touches index 0 ...
    hi = [n - 1 + so - reach for n in shape]                        # ... and the last allocated index
    assert _reach(emu, lo, hi, size, so, reach) == (B2_OK, 0, '')
    for d in range(nd):
        for end, step in ((lo, -1), (hi, 1)):
            end[d] += step
            rc, empty, msg = _reach(emu, lo, hi, size, so, reach, b'b2_' + rule.encode())
            end[d] -= step
            assert (rc, empty) == (B2_ERR_INVALID, 0), msg
            assert msg == (f"b2_{rule}: iteration range [{lo[d] + min(step, 0)},{hi[d] + max(step, 0)}] + reach "
                           f"{reach} leaves the allocated array (extent {size[d + 1]}) on dim {d}")


@pytest.mark.parametrize('nd', [1, 2, 3])
def test_empty_extent_means_nothing_to_do(emu, nd):
    so, shape = 4, (9, 10, 11)[:nd]
    size = (3,) + tuple(n + 2 * so for n in shape)
    for d in range(nd):
        lo, hi = [0] * nd, [n - 1 for n in shape]
        hi[d] = lo[d] - 1
        assert _reach(emu, lo, hi, size, so, 2) == (B2_OK, 1, '')


def test_refusal_before_a_later_empty_extent(emu):
    """dims are taken in order: out of range on x refuses even though y is empty; empty x wins over a bad y"""
    so, shape = 4, (9, 10, 11)
    size = (3,) + tuple(n + 2 * so for n in shape)
    rc, empty, msg = _reach(emu, (-3, 5, 0), (8, 4, 10), size, so, 2)
    assert (rc, empty) == (B2_ERR_INVALID, 0) and 'on dim 0' in msg
    assert _reach(emu, (5, -3, 0), (4, 9, 10), size, so, 2) == (B2_OK, 1, '')


# ---- GPU: the wave entry points through the ABI ----------------------------------------------------------------

H = 10.0
SO = 4
K = 4                                   # time steps 1 .. K
NT = K + 2
SHAPES = {2: (14, 12), 3: (9, 10, 12)}
TOL = {'iso': 1e-5, 'tti': 1e-4, 'sa': 1e-5, 'visco': 2e-5}
REACH = {'iso': SO // 2, 'tti': SO // 2, 'sa': SO - 1, 'visco': SO - 1}   # radius SO/2; the nested stencil 2R-1
FN = {'iso': 'b2_iso_forward', 'tti': 'b2_tti_forward', 'sa': 'b2_sa_forward', 'visco': 'b2_visco_forward'}
F0 = 0.01                               # the SLS reference frequency


def _L():
    from devito_b200 import _lib
    return _lib


class Call:
    """The host arrays of one call (by name), its args, and the float64 reference of a run."""

    def __init__(self, kind, nd, lo, hi, seed=0, errctl=0, born=False):
        self.kind, self.nd, self.keep = kind, nd, []
        self.rng = np.random.default_rng(seed)
        self.shape = SHAPES[nd]
        self.alloc = tuple(n + 2 * SO for n in self.shape)
        self.lo, self.hi = tuple(lo), tuple(hi)
        self.host = {'u': self.noise((3,) + self.alloc), 'damp': (0.1 * self.rng.uniform(0, 1, self.alloc)).astype(
            np.float32)}
        self.src = self.sparse(2)
        self.rec = self.sparse(5)
        self.host['src'], self.host['rec'] = self.src['data'], self.rec['data']
        getattr(self, '_' + kind)(errctl, born)
        a = self.a
        (a.x_m, a.y_m, a.z_m), (a.x_M, a.y_M, a.z_M) = (tuple(lo) + (0,))[:3], (tuple(hi) + (0,))[:3]
        a.time_m, a.time_M, a.errctl = 1, K, errctl
        a.src, a.rec = self.sparse_args(self.src), self.sparse_args(self.rec)

    def noise(self, shape, scale=1.0):
        return (scale * self.rng.standard_normal(shape)).astype(np.float32)

    def obj(self, arr):
        d = _L().make_dataobj(host=arr)
        self.keep.append(d)
        return d.ptr

    def weights(self, ws):
        arr = (ctypes.POINTER(ctypes.c_float) * 3)()
        for d, w in enumerate(ws):
            c = (ctypes.c_float * len(w))(*np.asarray(w, dtype=np.float32))
            self.keep.append(c)
            arr[d] = ctypes.cast(c, ctypes.POINTER(ctypes.c_float))
        return arr

    def sparse(self, npoint):
        pos = self.rng.uniform(0.2, np.array(self.shape) - 1.2, (npoint, self.nd)) * H
        gp, ws = O.tabulate(pos.astype(np.float32), (0.0,) * self.nd, (np.float32(H),) * self.nd, 1, 'linear')
        return dict(data=self.noise((NT, npoint)), gp=np.ascontiguousarray(gp, dtype=np.int32),
                    w=[np.ascontiguousarray(w, dtype=np.float32) for w in ws], r=1)

    def sparse_args(self, sp):
        s = _L().Sparse()
        s.data, s.gp = self.obj(sp['data']), self.obj(sp['gp'])
        for d in range(self.nd):
            s.w[d] = self.obj(sp['w'][d])
        s.p_m, s.p_M, s.r = 0, sp['data'].shape[1] - 1, sp['r']
        self.keep.append(s)
        return ctypes.pointer(s)

    def _iso(self, errctl, born):
        a = self.a = _L().IsoArgs()
        a.ndim, a.space_order, a.radius = self.nd, SO, SO // 2
        self.w64 = [ref64.fd2_weights(SO, H)] * self.nd
        a.w = self.weights(self.w64)
        a.u, a.damp = self.obj(self.host['u']), self.obj(self.host['damp'])
        a.param_kind, a.vp = 0, 2.0
        a.dt = self.dt = float(O.critical_dt(SO, self.nd, H, 2.0))

    def _tti(self, errctl, born):
        a = self.a = _L().TtiArgs()
        a.ndim, a.space_order, a.radius = self.nd, SO, SO // 2
        self.w2 = [ref64.fd2_weights(SO, H)] * self.nd
        self.w1 = [ref64.fd1_half_weights(SO, H)] * self.nd
        a.w2, a.w1 = self.weights(self.w2), self.weights(self.w1)
        self.host['v'] = self.noise((3,) + self.alloc)
        a.u, a.v, a.damp = self.obj(self.host['u']), self.obj(self.host['v']), self.obj(self.host['damp'])
        self.params = dict(vp=2.0, epsilon=0.2, delta=0.1, theta=0.6, phi=0.35 if self.nd == 3 else 0.0)
        a.vp, a.epsilon, a.delta, a.theta, a.phi = (self.params[k] for k in ('vp', 'epsilon', 'delta', 'theta', 'phi'))
        a.dt = self.dt = float(O.critical_dt(SO, self.nd, H, 2.0, eps_max=0.3))
        if born:
            for name in ('born_du', 'born_dv'):
                self.host[name] = self.noise((3,) + self.alloc)
            self.host['born_dm'] = self.noise(self.shape, 0.05)             # no halo
            a.born_du, a.born_dv, a.born_dm = (self.obj(self.host[n]) for n in ('born_du', 'born_dv', 'born_dm'))

    def _sa(self, errctl, born):
        a = self.a = _L().SaArgs()
        R = SO // 2
        a.ndim, a.space_order, a.radius = self.nd, SO, R
        self.c64 = [sa_ref.sa_weights(R, H)] * self.nd
        a.c = self.weights(self.c64)
        a.u, a.damp = self.obj(self.host['u']), self.obj(self.host['damp'])
        a.b_value, a.vp_value, a.dt = 1.25, 2.0, 0.9
        self.dt = 0.9

    def _visco(self, errctl, born):
        a = self.a = _L().ViscoArgs()
        R = SO // 2
        a.ndim, a.space_order, a.radius = self.nd, SO, R
        self.c64 = [sa_ref.sa_weights(R, H)] * self.nd
        a.c = self.weights(self.c64)
        self.host['r'] = self.noise((3,) + self.alloc, 0.1)
        self.host['damp'] = 1.0 - self.host['damp']                         # a mask profile in [0.9, 1]
        a.u, a.r, a.damp = (self.obj(self.host[k]) for k in ('u', 'r', 'damp'))
        a.b_value, a.vp_value, a.qp_value, a.f0, a.dt = 1.25, 2.0, 30.0, F0, 0.9
        self.dt = 0.9

    def run(self):
        """(return code, message, host arrays before the call); the call releases its staging"""
        L = _L().lib()
        before = {k: v.copy() for k, v in self.host.items()}
        rc = getattr(L, FN[self.kind])(ctypes.byref(self.a))
        assert L.b2_staging_outstanding() == 0, rc
        return rc, L.b2_last_error().decode(), before

    def sparse64(self, sp):
        return dict(sp, w=[np.asarray(w, dtype=np.float64) for w in sp['w']])

    def reference(self, before):
        """float64 (fields by name, traces) from the arrays as they were before the call"""
        src, rec = self.sparse64(dict(self.src, data=before['src'])), self.sparse64(dict(self.rec, data=before['rec']))
        kw = dict(lo=self.lo, hi=self.hi, src=src, rec=rec)
        if self.kind == 'iso':
            u, tr = ref64.iso_forward(before['u'], SO, self.w64, self.dt, 1, K, damp=before['damp'], param=('vp', 2.0),
                                      **kw)
            return dict(u=u), tr
        if self.kind == 'sa':
            u, tr = sa_ref.sa_forward(before['u'], SO, self.c64, self.dt, 1, K, 1.25, 2.0, w=before['damp'], **kw)
            return dict(u=u), tr
        if self.kind == 'visco':
            u, r, tr = visco_ref.visco_forward(before['u'], before['r'], SO, self.c64, self.dt,
                                               float(np.float32(F0)), 1, K, 1.25, 2.0, 30.0, damp=before['damp'], **kw)
            return dict(u=u, r=r), tr
        if self.nd == 3:
            u, v, tr = ref64.tti_forward(before['u'], before['v'], SO, self.w2, self.w1, self.dt, 1, K,
                                         before['damp'], self.params, **kw)
        else:
            p2 = {k: x for k, x in self.params.items() if k != 'phi'}
            u, v, _, _, tr = tti2d_ref.forward(before['u'], before['v'], SO, self.w2, self.w1, self.dt, 1, K,
                                               before['damp'], p2, **kw)
        return dict(u=u, v=v), tr


def _touching(nd, reach):
    """the box whose reach touches both ends of the allocation on every dim"""
    return [reach - SO] * nd, [n - 1 + SO - reach for n in SHAPES[nd]]


CASES = [(k, nd) for k in ('iso', 'tti', 'sa', 'visco') for nd in (2, 3)]
IDS = [f'{k}-{nd}d' for k, nd in CASES]


@pytest.mark.gpu
@pytest.mark.parametrize('kind,nd', CASES, ids=IDS)
def test_box_one_past_the_allocation_is_refused(kind, nd):
    lo, hi = _touching(nd, REACH[kind])
    for d in range(nd):
        for end, step in ((lo, -1), (hi, 1)):
            end[d] += step
            c = Call(kind, nd, lo, hi)
            end[d] -= step
            rc, msg, before = c.run()
            assert rc == B2_ERR_INVALID, (rc, msg)
            assert 'leaves the allocated array' in msg and FN[kind] in msg, msg
            for k in c.host:
                assert np.array_equal(c.host[k], before[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize('kind,nd', CASES, ids=IDS)
def test_box_touching_the_allocation_matches_float64(kind, nd):
    c = Call(kind, nd, *_touching(nd, REACH[kind]))
    rc, msg, before = c.run()
    assert rc == B2_OK, msg
    fields, traces = c.reference(before)
    for k, ref in fields.items():
        assert rel_linf(c.host[k], ref) < TOL[kind], k
    assert rel_linf(c.host['rec'], traces) < TOL[kind]


@pytest.mark.gpu
@pytest.mark.parametrize('kind,nd', CASES, ids=IDS)
def test_empty_box_writes_nothing(kind, nd):
    lo, hi = [0] * nd, [n - 1 for n in SHAPES[nd]]
    hi[-1] = -1
    c = Call(kind, nd, lo, hi)
    rc, msg, before = c.run()
    assert rc == B2_OK, msg
    for k in c.host:
        assert np.array_equal(c.host[k], before[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize('kind,nd', CASES, ids=IDS)
def test_sparse_radius_beyond_the_halo_is_refused(kind, nd):
    c = Call(kind, nd, [0] * nd, [n - 1 for n in SHAPES[nd]])
    c.a.src.contents.r = SO + 1
    rc, msg, before = c.run()
    assert rc == B2_ERR_INVALID and 'exceeds the halo' in msg and FN[kind] in msg, (rc, msg)
    for k in c.host:
        assert np.array_equal(c.host[k], before[k]), k


def _plant_inf(c, name):
    mid = tuple(SO + n // 2 for n in c.shape)
    c.host[name][(slice(None),) + mid] = np.inf


def _stopped_on_nan(c, field, written):
    rc, msg, before = c.run()
    assert rc == B2_ERR_NAN and f'NaN/Inf detected in {field} at time=' in msg, (rc, msg)
    for k in written:                      # the Inf spread over the steps taken, and that came back
        assert np.count_nonzero(~np.isfinite(c.host[k])) > np.count_nonzero(~np.isfinite(before[k])), k


@pytest.mark.gpu
@pytest.mark.parametrize('kind,nd', [(k, nd) for k, nd in CASES if k != 'iso'],
                         ids=[i for i in IDS if not i.startswith('iso')])
def test_errctl_stops_on_inf_in_u(kind, nd):
    c = Call(kind, nd, [0] * nd, [n - 1 for n in SHAPES[nd]], errctl=1)
    _plant_inf(c, 'u')
    _stopped_on_nan(c, 'p' if kind == 'visco' else 'u', ['u'])


@pytest.mark.gpu
def test_errctl_tti_born_names_du():
    c = Call('tti', 3, [0] * 3, [n - 1 for n in SHAPES[3]], errctl=1, born=True)
    _plant_inf(c, 'born_du')
    _stopped_on_nan(c, 'du', ['born_du'])


@pytest.mark.gpu
@pytest.mark.parametrize('kind', ['tti', 'sa', 'linear'])
def test_timers_report_section0(kind):
    L = _L()
    prof = L.Profiler()
    if kind == 'linear':
        f = np.random.default_rng(0).standard_normal((2, 40, 50)).astype(np.float32)
        taps = (L.Tap * 2)()
        taps[0].coef, taps[1].coef, taps[1].off[1] = 0.5, 0.25, 1
        a = L.LinearArgs()
        keep = L.make_dataobj(host=f)
        a.ndim, a.f, a.halo, a.ntaps, a.taps, a.wshift = 2, keep.ptr, 1, 2, taps, 1
        a.x_m, a.x_M, a.y_m, a.y_M, a.time_m, a.time_M = 0, 37, 0, 47, 0, 9
        a.timers = ctypes.pointer(prof)
        rc = L.lib().b2_linear_forward(ctypes.byref(a))
    else:
        c = Call(kind, 3, [0] * 3, [n - 1 for n in SHAPES[3]])
        c.a.timers = ctypes.pointer(prof)
        rc, _, _ = c.run()
    assert rc == B2_OK, L.lib().b2_last_error().decode()
    assert prof.section0 > 0
