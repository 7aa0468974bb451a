"""Host staging of the C entry points, called directly through the ABI on tiny 3-D grids (`dmap` = NULL, i.e.
`resident=False`): every call releases every staging buffer it took (`b2_staging_outstanding`), whatever it returns;
refused calls (210) leave every host array byte-identical; a call that stops on a NaN (100) still writes its
written arrays back (include/b200stencil.h, `struct b2_dataobj`).
"""
import ctypes

import numpy as np
import pytest

from oracle import oracle as O

pytestmark = pytest.mark.gpu

B2_ERR_NAN, B2_ERR_INVALID = 100, 210
H = 10.0
N = (20, 12, 16)                      # domain; x long enough for the streamed loop at radius 2
NT = 8


def _L():
    from devito_b200 import _lib
    return _lib


class Call:
    """The arrays of one call, kept alive next to their `struct b2_dataobj`s."""

    def __init__(self, so, seed=0):
        self.so, self.keep, self.rng = so, [], np.random.default_rng(seed)
        self.alloc = tuple(n + 2 * so for n in N)

    def obj(self, arr):
        halo = None
        if arr.ndim >= 3:                             # a grid array: its halo in `hsize`
            h = (arr.shape[-1] - N[2]) // 2
            halo = ((0, 0),) * (arr.ndim - 3) + ((h, h),) * 3
        d = _L().make_dataobj(host=arr, halo=halo)
        self.keep.append(d)
        return d.ptr

    def field(self, lead=(3,), halo=None, scale=1e-3):
        h = self.so if halo is None else halo
        return (scale * self.rng.standard_normal(tuple(lead) + tuple(n + 2 * h for n in N))).astype(np.float32)

    def sparse(self, npoint, p_M=None):
        L = _L()
        pos = np.array([[(n - 1) * H * f for n in N] for f in np.linspace(0.3, 0.7, npoint)], dtype=np.float32)
        gp, ws = O.tabulate(pos, (0.0,) * 3, (np.float32(H),) * 3, 1, 'linear')
        data = (self.rng.standard_normal((NT, npoint))).astype(np.float32)
        s = L.Sparse()
        s.data, s.gp = self.obj(data), self.obj(np.ascontiguousarray(gp, dtype=np.int32))
        for d in range(3):
            s.w[d] = self.obj(np.ascontiguousarray(ws[d], dtype=np.float32))
        s.p_m, s.p_M, s.r = 0, npoint - 1 if p_M is None else p_M, 1
        self.keep.append(s)
        return ctypes.pointer(s), data

    def weights(self, w):
        arr = (ctypes.POINTER(ctypes.c_float) * 3)()
        for d in range(3):
            c = (ctypes.c_float * len(w))(*w)
            self.keep.append(c)
            arr[d] = ctypes.cast(c, ctypes.POINTER(ctypes.c_float))
        return arr

    def box(self, a):
        a.x_m, a.x_M, a.y_m, a.y_M, a.z_m, a.z_M = 0, N[0] - 1, 0, N[1] - 1, 0, N[2] - 1
        a.time_m, a.time_M = 1, NT - 2


def _iso(c, **kw):
    """An iso call: (args, host arrays by name). kw: `adjoint`, `grad`/`usave`/`born_U`/`born_dm`/`snap` arrays
    (or None), `rec_p_M`, `errctl`."""
    L = _L()
    a = L.IsoArgs()
    a.ndim, a.space_order, a.radius = 3, c.so, c.so // 2
    a.w = c.weights(O.fd2_weights(c.so, H))
    host = {'u': c.field(), 'damp': np.zeros(c.alloc, dtype=np.float32)}
    a.u, a.damp = c.obj(host['u']), c.obj(host['damp'])
    a.param_kind, a.vp, a.dt = 0, 1.5, 1.0
    c.box(a)
    a.src, host['src'] = c.sparse(1)
    a.rec, host['rec'] = c.sparse(5, kw.pop('rec_p_M', None))
    a.errctl = kw.pop('errctl', 0)
    a.adjoint = kw.pop('adjoint', 0)
    for name in ('grad', 'usave', 'born_U', 'born_dm', 'snap'):
        arr = kw.pop(name, None)
        if arr is not None:
            host[name] = arr
            setattr(a, name, c.obj(arr))
    a.snap_factor = kw.pop('snap_factor', 0)
    assert not kw, kw
    return a, host


def _tti(c, **kw):
    L = _L()
    a = L.TtiArgs()
    a.space_order, a.radius = c.so, c.so // 2
    a.w2 = c.weights(O.fd2_weights(c.so, H))
    a.w1 = c.weights(O.fd1_half_weights(c.so, H))
    host = {'u': c.field(), 'v': c.field(), 'damp': np.zeros(c.alloc, dtype=np.float32)}
    a.u, a.v, a.damp = c.obj(host['u']), c.obj(host['v']), c.obj(host['damp'])
    a.vp, a.epsilon, a.delta, a.theta, a.phi, a.dt = 1.5, 0.2, 0.1, 0.3, 0.2, 1.0
    c.box(a)
    a.src, host['src'] = c.sparse(1)
    a.rec, host['rec'] = c.sparse(5, kw.pop('rec_p_M', None))
    a.adjoint = kw.pop('adjoint', 0)
    for name in ('born_du', 'born_dv', 'born_dm', 'grad', 'usave', 'vsave'):
        arr = kw.pop(name, None)
        if arr is not None:
            host[name] = arr
            setattr(a, name, c.obj(arr))
    assert not kw, kw
    return a, host


def _call(fn, a, host):
    """(return code, host arrays before the call); checks that the call released its staging."""
    L = _L().lib()
    before = {k: v.copy() for k, v in host.items()}
    rc = getattr(L, fn)(ctypes.byref(a))
    assert L.b2_staging_outstanding() == 0, (fn, rc)
    return rc, before


def _runs(fn, a, host, written):
    rc, before = _call(fn, a, host)
    assert rc == 0, _L().lib().b2_last_error().decode()
    for k in written:
        assert not np.array_equal(host[k], before[k]), k
    assert all(np.isfinite(host[k]).all() for k in written)


def _refused(fn, a, host, what):
    rc, before = _call(fn, a, host)
    msg = _L().lib().b2_last_error().decode()
    assert rc == B2_ERR_INVALID, (rc, msg)
    assert what in msg, msg
    for k in host:
        assert np.array_equal(host[k], before[k]), k


# ---- successful host-staged calls ------------------------------------------------------------------------------

@pytest.mark.parametrize('stream', [None, '2'])
def test_iso_forward(stream, monkeypatch):
    if stream:
        monkeypatch.setenv('B2_STREAM', stream)
    c = Call(4)
    a, host = _iso(c)
    _runs('b2_iso_forward', a, host, ['u', 'rec'])
    prof = (ctypes.c_double * 5)()
    _L().lib().b2_last_call_profile(prof)
    assert (prof[4] == 1.0) == bool(stream)


def test_iso_adjoint_gradient():
    c = Call(4)
    a, host = _iso(c, adjoint=1, grad=np.zeros(N, dtype=np.float32), usave=c.field((NT,)))
    _runs('b2_iso_forward', a, host, ['u', 'rec', 'grad'])


def test_iso_born():
    c = Call(4)
    a, host = _iso(c, born_U=c.field(), born_dm=c.field((), halo=1, scale=0.1))
    _runs('b2_iso_forward', a, host, ['u', 'rec', 'born_U'])


def test_iso_streamed_snapshots():
    c = Call(4)
    a, host = _iso(c, snap=np.zeros((NT // 2,) + tuple(n + 2 for n in N), dtype=np.float32), snap_factor=2)
    _runs('b2_iso_forward', a, host, ['u', 'rec', 'snap'])


def test_tti_forward():
    c = Call(8)
    a, host = _tti(c)
    _runs('b2_tti_forward', a, host, ['u', 'v', 'rec'])


def test_tti_born():
    c = Call(8)
    a, host = _tti(c, born_du=c.field(), born_dv=c.field(), born_dm=c.field((), halo=0, scale=0.1))
    _runs('b2_tti_forward', a, host, ['u', 'v', 'rec', 'born_du', 'born_dv'])


def test_tti_adjoint_gradient():
    c = Call(8)
    a, host = _tti(c, adjoint=1, grad=np.zeros(N, dtype=np.float32), usave=c.field((NT,)), vsave=c.field((NT,)))
    _runs('b2_tti_forward', a, host, ['u', 'v', 'rec', 'grad'])


def test_linear():
    L = _L()
    c = Call(1)
    f = c.field((2,))
    taps = (L.Tap * 3)()
    for i, (off, coef) in enumerate([((0, 0, 0), 0.5), ((1, 0, 0), 0.25), ((0, 0, -1), 0.25)]):
        taps[i].tshift, taps[i].coef = 0, coef
        for d in range(3):
            taps[i].off[d] = off[d]
    a = L.LinearArgs()
    a.ndim, a.f, a.halo, a.ntaps, a.taps, a.wshift = 3, c.obj(f), 1, 3, taps, 1
    c.box(a)
    _runs('b2_linear_forward', a, {'f': f}, ['f'])


# ---- refusals: 210 before anything is written back -------------------------------------------------------------

def test_iso_rec_point_range():
    c = Call(4)
    a, host = _iso(c, rec_p_M=5)                       # = npoint_total
    _refused('b2_iso_forward', a, host, 'point range')


def test_tti_rec_point_range():
    c = Call(8)
    a, host = _tti(c, rec_p_M=5)
    _refused('b2_tti_forward', a, host, 'point range')


def test_iso_grad_without_usave():
    c = Call(4)
    a, host = _iso(c, adjoint=1, grad=np.zeros(N, dtype=np.float32))
    _refused('b2_iso_forward', a, host, 'needs both grad and usave')


def test_iso_grad_of_wrong_extent():
    c = Call(4)
    a, host = _iso(c, adjoint=1, grad=np.zeros((N[0], N[1], N[2] + 1), dtype=np.float32), usave=c.field((NT,)))
    _refused('b2_iso_forward', a, host, 'grad extent')


def test_iso_usave_of_wrong_layout():
    c = Call(4)
    a, host = _iso(c, adjoint=1, grad=np.zeros(N, dtype=np.float32), usave=c.field((NT,), halo=2))
    _refused('b2_iso_forward', a, host, 'usave extent')


def test_tti_born_du_without_born_dm():
    c = Call(8)
    a, host = _tti(c, born_du=c.field(), born_dv=c.field())
    _refused('b2_tti_forward', a, host, 'born_du, born_dv and born_dm together')


@pytest.mark.parametrize('T,taps,wshift,what', [
    (3, [(0, (0, 0, 0)), (-2, (1, 0, 0))], 1, 'the slot being written'),      # t - 2 is t + 1 modulo 3
    (2, [(0, (0, 0, 0)), (1, (0, 0, -1))], -1, 'the slot being written'),     # t + 1 is t - 1 modulo 2
    (2, [(1, (0, 0, 0))], 1, 'the slot being written'),                        # implicit
    (2, [(0, (0, 0, 0)), (0, (0, 2, 0))], 1, 'leaves the allocated array'),    # halo 1
    (2, [], 1, '0 taps'),
    (2, [(0, (0, 0, 0))] * 65, 1, '65 taps'),
    (6, [(-k, (0, 0, 0)) for k in range(5)], 1, 'more than 4 time levels'),
    (2, [(-1, (0, 0, 0))], 0, 'wshift must be'),
], ids=['alias-fwd', 'alias-bwd', 'implicit', 'beyond-alloc', '0-taps', '65-taps', '5-levels', 'wshift-0'])
def test_linear_refusals(T, taps, wshift, what):
    L = _L()
    c = Call(1)
    f = c.field((T,))
    arr = (L.Tap * max(len(taps), 1))()
    for i, (s, off) in enumerate(taps):
        arr[i].tshift, arr[i].coef = s, 0.5
        for d in range(3):
            arr[i].off[d] = off[d]
    a = L.LinearArgs()
    a.ndim, a.f, a.halo, a.ntaps, a.taps, a.wshift = 3, c.obj(f), 1, len(taps), arr, wshift
    c.box(a)
    _refused('b2_linear_forward', a, {'f': f}, what)


# ---- a NaN stops the call (100), and the written arrays still come back ----------------------------------------

def test_iso_gradient_nan_writes_back():
    c = Call(4)
    a, host = _iso(c, adjoint=1, grad=np.zeros(N, dtype=np.float32), usave=c.field((NT,)), errctl=1)
    host['u'][:, c.so + N[0] // 2, c.so + N[1] // 2, c.so + N[2] // 2] = np.inf
    rc, before = _call('b2_iso_forward', a, host)
    assert rc == B2_ERR_NAN, (rc, _L().lib().b2_last_error().decode())
    assert not np.isfinite(host['grad']).all()
    assert not np.array_equal(host['rec'], before['rec'])
