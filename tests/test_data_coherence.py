"""Views of a function's data that the caller keeps across applies, on the CPU.

Dense arrays stay on the device between applies (devito_b200/types.py::FieldStorage); the host copy and the device copy
are reconciled when an accessor is called. A view the caller keeps must still be coherent in both directions, as in
the reference, which copies every array in and out of every apply (devito/passes/iet/definitions.py:636-671):
(a) a write through the kept view is in the next upload, (b) what a kernel wrote is in the kept view as soon as the
write is marked. A CPU tensor stands in for the device copy (`to_device(torch.device('cpu'))`): the protocol the CUDA
path runs, without a GPU. Every accessor a caller can keep, and views derived from each (a slice, an integer-indexed
sub-view, `np.asarray`, `.view(np.ndarray)`), on both host allocations: the page-locked one (`_pinned.numpy()`, a
torch CPU tensor's array standing in where CUDA is absent) and the plain NumPy one.

Also: `SeismicModel.critical_dt` after a write through a kept view of vp / epsilon equals a fresh float64 evaluation
of the CFL formula, and with no view held nothing is copied that was not copied before (two uploads make one copy,
marking a kernel write downloads nothing), which is what keeps the resident applies copy-free.
"""
import numpy as np
import pytest
import torch

from devito_b200 import Grid, Function, TimeFunction
from devito_b200.types import FieldStorage
from oracle import oracle as O

CPU = torch.device('cpu')

ACCESSORS = {
    'data': lambda f: f.data,
    'data_with_halo': lambda f: f.data_with_halo,
    'data_allocated': lambda f: f.data_allocated,
    '_data_allocated': lambda f: f._data_allocated,
    'data_ro_domain': lambda f: f.data_ro_domain,
    'data_ro_with_halo': lambda f: f.data_ro_with_halo,
}
DOMAIN_ONLY = ('data', 'data_ro_domain')

# views derived from an accessor's result; the accessor's own object is dropped at once
DERIVED = {
    'whole': lambda v: v,
    'slice': lambda v: v[1:, 2:-1],
    'index': lambda v: v[1],
    'asarray': np.asarray,
    'ndarray_view': lambda v: v.view(np.ndarray),
}

# shapes: the pinned one holds 1 MiB or more (the size from which the storage pins when CUDA is present)
SHAPES = {'numpy': (6, 7, 9), 'pinned': (64, 64, 64)}
SO = 2


@pytest.fixture(params=['numpy', 'pinned'])
def host_kind(request, monkeypatch):
    if request.param == 'pinned' and not torch.cuda.is_available():
        def pinned_standin(self):
            self._pinned = torch.zeros(self.shape, dtype=torch.float32)
            return self._pinned.numpy()
        monkeypatch.setattr(FieldStorage, '_new_host', pinned_standin)
    return request.param


def _function(host_kind, time=True):
    grid = Grid(shape=SHAPES[host_kind])
    if time:
        f = TimeFunction(name='u', grid=grid, time_order=2, space_order=SO)
    else:
        f = Function(name='vp', grid=grid, space_order=SO)
    rng = np.random.default_rng(5)
    f.data_with_halo[:] = rng.standard_normal(f.shape_allocated).astype(np.float32)
    assert (f.storage._pinned is not None) == (host_kind == 'pinned')
    return f


def _region(f, accessor, arr):
    """The part of an allocation-shaped array `arr` that `accessor` exposes."""
    return arr[f._domain_slices()] if accessor in DOMAIN_ONLY else arr


def _noise(shape, seed):
    return np.random.default_rng(seed).standard_normal(shape).astype(np.float32)


def _kernel_write(st, values):
    """What an apply does to a storage it writes: upload, write on the device, mark the write."""
    t = st.to_device(CPU)
    t.copy_(torch.from_numpy(values))
    st.mark_device_written()


@pytest.mark.parametrize('derive', list(DERIVED))
@pytest.mark.parametrize('accessor', list(ACCESSORS))
def test_write_through_a_kept_view_reaches_the_device(host_kind, accessor, derive):
    f = _function(host_kind)
    st = f.storage
    view = DERIVED[derive](ACCESSORS[accessor](f))
    st.to_device(CPU)                                     # first apply
    dev = _noise(st.shape, 1)
    _kernel_write(st, dev)                                # it writes the array
    pattern = (1000.0 + np.arange(view.size, dtype=np.float32)).reshape(view.shape)
    view[...] = pattern                                   # the caller writes through the view it kept
    got = st.to_device(CPU).numpy()                       # second apply
    want = dev.copy()
    DERIVED[derive](_region(f, accessor, want))[...] = pattern
    assert np.array_equal(got, want)


@pytest.mark.parametrize('derive', list(DERIVED))
@pytest.mark.parametrize('accessor', list(ACCESSORS))
def test_kept_view_sees_what_a_kernel_wrote(host_kind, accessor, derive):
    f = _function(host_kind)
    st = f.storage
    view = DERIVED[derive](ACCESSORS[accessor](f))
    for seed in (1, 2):                                   # two applies, the view kept across both
        dev = _noise(st.shape, seed)
        _kernel_write(st, dev)
        got = np.array(view)                              # read before any fresh accessor
        want = DERIVED[derive](_region(f, accessor, dev))
        assert np.array_equal(got, want)
        assert np.array_equal(got, DERIVED[derive](ACCESSORS[accessor](f)))


def test_views_of_a_parameter_and_of_a_sub_view(host_kind):
    """A Function (parameter: read by the kernels, never written) and `f.data[1]` of a TimeFunction kept over several
    round trips, written between them."""
    vp = _function(host_kind, time=False)
    u = _function(host_kind)
    kept_vp = vp.data
    kept_u1 = u.data[1]
    for k in range(3):
        kept_vp[...] = 1.5 + k
        assert np.array_equal(vp.storage.to_device(CPU).numpy()[vp._domain_slices()],
                              np.full(vp.shape, 1.5 + k, np.float32))
        dev = _noise(u.storage.shape, 10 + k)
        _kernel_write(u.storage, dev)
        assert np.array_equal(kept_u1, dev[u._domain_slices()][1])
        kept_u1[...] = -k
        assert np.all(u.storage.to_device(CPU).numpy()[u._domain_slices()][1] == -k)


def _count_copies(monkeypatch):
    counts = {'up': 0, 'down': 0}
    up, down = FieldStorage._upload, FieldStorage.sync_to_host

    def counted_up(self):
        counts['up'] += 1
        return up(self)

    def counted_down(self):
        counts['down'] += 1
        return down(self)
    monkeypatch.setattr(FieldStorage, '_upload', counted_up)
    monkeypatch.setattr(FieldStorage, 'sync_to_host', counted_down)
    return counts


def test_no_view_held_makes_no_copy(host_kind, monkeypatch):
    """The resident applies' fast path: with no view alive an array is uploaded once, a kernel write is not
    downloaded, and a fresh accessor (dropped at once) costs one download and the next apply one upload."""
    counts = _count_copies(monkeypatch)
    u = _function(host_kind)
    st = u.storage
    assert not st.views_held()
    st.to_device(CPU)
    st.to_device(CPU)
    assert counts == {'up': 1, 'down': 0}
    for _ in range(3):
        _kernel_write(st, _noise(st.shape, 4))
    assert counts == {'up': 1, 'down': 0}
    assert float(np.abs(u.data_ro_with_halo).max()) > 0  # a fresh read: one download, nothing kept
    assert counts == {'up': 1, 'down': 1}
    assert not st.views_held()
    _kernel_write(st, _noise(st.shape, 5))               # the read did not expose the host copy for writing
    assert counts == {'up': 1, 'down': 1}
    u.data[:] = 0.0                                       # a fresh write (after a download of the kernel's values):
    st.to_device(CPU)                                     # the next apply uploads once
    st.to_device(CPU)
    assert counts == {'up': 2, 'down': 2}
    kept = u.data
    assert st.views_held()
    _kernel_write(st, _noise(st.shape, 6))               # with a view kept: one upload, one download per apply
    assert counts == {'up': 3, 'down': 3}
    del kept
    assert not st.views_held()
    _kernel_write(st, _noise(st.shape, 7))
    assert counts == {'up': 3, 'down': 3}


def test_a_model_and_its_solver_keep_no_view():
    """Building a model, a geometry and a solver leaves no view of any array alive: the resident applies of the
    solvers stay copy-free."""
    from devito_b200.seismic import SeismicModel, AcquisitionGeometry, AcousticWaveSolver, AnisotropicWaveSolver
    shape = (24, 20, 22)
    v = np.full(shape, 1.5, dtype=np.float32)
    v[..., 11:] = 2.5
    m = SeismicModel(origin=(0., 0., 0.), spacing=(10., 10., 10.), shape=shape, space_order=4, vp=v, nbl=4,
                     bcs='damp', epsilon=0.1 * (v - 1.5), delta=0.05 * (v - 1.5), theta=0.3 * (v - 1.5),
                     phi=0.1 * (v - 1.5))
    geometry = AcquisitionGeometry(m, np.array([[100., 100., 20.]]), np.array([[120., 90., 10.]]), t0=0.0, tn=50.0,
                                   src_type='Ricker', f0=0.010)
    solvers = [AcousticWaveSolver(m, geometry, space_order=4), AnisotropicWaveSolver(m, geometry, space_order=4)]
    solvers[0].op_fwd()
    solvers[1].op_fwd()
    for name in ('vp', 'damp', 'epsilon', 'delta', 'theta', 'phi'):
        f = getattr(m, name)
        assert not f.storage.views_held(), name
    _ = m.critical_dt
    assert not m.vp.storage.views_held()


def _cfl(so, spacing, vmax, emax=None):
    return O.critical_dt(so, 3, float(min(spacing)), float(vmax), eps_max=None if emax is None else float(emax))


@pytest.mark.parametrize('derive', ['whole', 'asarray', 'slice'])
def test_critical_dt_after_a_write_through_a_kept_view_of_vp(derive):
    from devito_b200.seismic import SeismicModel
    shape = (24, 20, 22)
    v = np.full(shape, 1.5, dtype=np.float32)
    v[..., 11:] = 2.5
    m = SeismicModel(origin=(0., 0., 0.), spacing=(10., 10., 12.5), shape=shape, space_order=4, vp=v, nbl=4,
                     bcs='damp')
    kept = DERIVED[derive](m.vp.data)
    dt0 = m.critical_dt
    assert dt0 == _cfl(4, m.spacing, 2.5)
    assert m.critical_dt == dt0
    kept[...] *= 2                                        # doubles the maximum wherever the view reaches
    assert m.critical_dt == _cfl(4, m.spacing, 5.0)
    kept[...] = 1.0
    want = _cfl(4, m.spacing, float(np.max(np.asarray(m.vp.data_ro_domain, dtype=np.float64))))
    assert m.critical_dt == want


def test_critical_dt_after_a_write_through_a_kept_view_of_epsilon():
    from devito_b200.seismic import SeismicModel
    shape = (24, 20, 22)
    v = np.full(shape, 1.5, dtype=np.float32)
    v[..., 11:] = 2.5
    m = SeismicModel(origin=(0., 0., 0.), spacing=(10., 10., 10.), shape=shape, space_order=8, vp=v, nbl=4,
                     bcs='damp', epsilon=0.1 * (v - 1.5), delta=0.05 * (v - 1.5), theta=0.3 * (v - 1.5),
                     phi=0.1 * (v - 1.5))
    eps = m.epsilon.data
    vp = np.asarray(m.vp.data)
    dt0 = m.critical_dt
    assert dt0 == _cfl(8, m.spacing, 2.5, np.float32(0.1))
    eps[...] = 0.4
    assert m.critical_dt == _cfl(8, m.spacing, 2.5, np.float32(0.4))
    vp[3, 4, 5] = 4.0
    assert m.critical_dt == _cfl(8, m.spacing, 4.0, np.float32(0.4))
