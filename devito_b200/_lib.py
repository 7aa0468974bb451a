"""ctypes binding of libb200stencil.so — the C-ABI drop-in boundary (include/b200stencil.h).

The reference reaches its generated kernel the same way: `ctypes` load of a shared object,
`argtypes` from each parameter's `_C_ctype`, one blocking call per `Operator.apply`
(devito/operator/operator.py:857-869, :1029-1032).  There is NO fallback: if the library or a
GPU is missing, `lib()` raises `BackendUnavailable`.
"""
import ctypes
import os
from ctypes import (POINTER, Structure, c_char_p, c_double, c_float, c_int, c_ulong, c_ulonglong,
                    c_void_p)

import numpy as np

from .exceptions import BackendUnavailable

__all__ = ['lib', 'have_lib', 'have_gpu', 'Dataobj', 'Profiler', 'Sparse', 'IsoArgs', 'TtiArgs', 'SaArgs', 'ViscoArgs', 'Tap', 'LinearArgs',
           'SysTap', 'SysStage', 'SysInject', 'SysInterp', 'SystemArgs',
           'make_dataobj', 'ForeignDataobj', 'ForeignSparse', 'nccl_library_path', 'LIB_PATH']

LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'libb200stencil.so')


class Dataobj(Structure):
    """`struct dataobj` (devito/types/dense.py:737-746)."""
    _fields_ = [('data', c_void_p), ('size', POINTER(c_int)), ('nbytes', c_ulong),
                ('npsize', POINTER(c_ulong)), ('dsize', POINTER(c_ulong)),
                ('hsize', POINTER(c_int)), ('hofs', POINTER(c_int)), ('oofs', POINTER(c_int)),
                ('dmap', c_void_p)]


class Profiler(Structure):
    _fields_ = [('section0', c_double), ('section1', c_double), ('section2', c_double),
                ('haloupdate0', c_double)]


class Sparse(Structure):
    _fields_ = [('data', POINTER(Dataobj)), ('gp', POINTER(Dataobj)),
                ('w', POINTER(Dataobj) * 3), ('p_m', c_int), ('p_M', c_int), ('r', c_int)]


class IsoArgs(Structure):
    _fields_ = [('ndim', c_int), ('space_order', c_int), ('radius', c_int),
                ('w', POINTER(c_float) * 3),
                ('u', POINTER(Dataobj)), ('damp', POINTER(Dataobj)),
                ('param_kind', c_int), ('param', POINTER(Dataobj)), ('vp', c_float),
                ('dt', c_float),
                ('x_m', c_int), ('x_M', c_int), ('y_m', c_int), ('y_M', c_int),
                ('z_m', c_int), ('z_M', c_int), ('time_m', c_int), ('time_M', c_int),
                ('src', POINTER(Sparse)), ('rec', POINTER(Sparse)), ('rec_toff', c_int),
                ('errctl', c_int), ('deviceid', c_int), ('kernel', c_int),
                ('halo', c_void_p), ('timers', POINTER(Profiler)), ('adjoint', c_int),
                ('grad', POINTER(Dataobj)), ('usave', POINTER(Dataobj)), ('free_surface', c_int), ('ot4', c_int),
                ('born_U', POINTER(Dataobj)), ('born_dm', POINTER(Dataobj)),
                ('snap', POINTER(Dataobj)), ('snap_factor', c_int), ('snap_toff', c_int), ('host_io', c_int)]


class TtiArgs(Structure):
    _fields_ = [('space_order', c_int), ('radius', c_int),
                ('w2', POINTER(c_float) * 3), ('w1', POINTER(c_float) * 3),
                ('u', POINTER(Dataobj)), ('v', POINTER(Dataobj)), ('damp', POINTER(Dataobj)),
                ('vp', c_float), ('epsilon', c_float), ('delta', c_float), ('theta', c_float),
                ('phi', c_float), ('dt', c_float),
                ('x_m', c_int), ('x_M', c_int), ('y_m', c_int), ('y_M', c_int),
                ('z_m', c_int), ('z_M', c_int), ('time_m', c_int), ('time_M', c_int),
                ('src', POINTER(Sparse)), ('rec', POINTER(Sparse)), ('rec_toff', c_int),
                ('errctl', c_int), ('deviceid', c_int), ('kernel', c_int),
                ('halo', c_void_p), ('timers', POINTER(Profiler)),
                ('vp_arr', POINTER(Dataobj)), ('epsilon_arr', POINTER(Dataobj)),
                ('delta_arr', POINTER(Dataobj)), ('theta_arr', POINTER(Dataobj)),
                ('phi_arr', POINTER(Dataobj)),
                ('born_du', POINTER(Dataobj)), ('born_dv', POINTER(Dataobj)), ('born_dm', POINTER(Dataobj)),
                ('adjoint', c_int), ('grad', POINTER(Dataobj)), ('usave', POINTER(Dataobj)),
                ('vsave', POINTER(Dataobj)), ('ndim', c_int)]


class SaArgs(Structure):
    _fields_ = [('ndim', c_int), ('space_order', c_int), ('radius', c_int),
                ('c', POINTER(c_float) * 3),
                ('u', POINTER(Dataobj)), ('b', POINTER(Dataobj)), ('b_value', c_float),
                ('vp', POINTER(Dataobj)), ('vp_value', c_float), ('damp', POINTER(Dataobj)),
                ('dt', c_float),
                ('x_m', c_int), ('x_M', c_int), ('y_m', c_int), ('y_M', c_int),
                ('z_m', c_int), ('z_M', c_int), ('time_m', c_int), ('time_M', c_int),
                ('src', POINTER(Sparse)), ('rec', POINTER(Sparse)), ('rec_toff', c_int),
                ('adjoint', c_int), ('errctl', c_int), ('deviceid', c_int), ('kernel', c_int),
                ('halo', c_void_p), ('free_surface', c_int), ('timers', POINTER(Profiler))]


class ViscoArgs(Structure):
    _fields_ = [('ndim', c_int), ('space_order', c_int), ('radius', c_int),
                ('c', POINTER(c_float) * 3),
                ('u', POINTER(Dataobj)), ('r', POINTER(Dataobj)), ('b', POINTER(Dataobj)), ('b_value', c_float),
                ('vp', POINTER(Dataobj)), ('vp_value', c_float), ('qp', POINTER(Dataobj)), ('qp_value', c_float),
                ('damp', POINTER(Dataobj)), ('f0', c_float), ('dt', c_float),
                ('x_m', c_int), ('x_M', c_int), ('y_m', c_int), ('y_M', c_int),
                ('z_m', c_int), ('z_M', c_int), ('time_m', c_int), ('time_M', c_int),
                ('src', POINTER(Sparse)), ('rec', POINTER(Sparse)), ('rec_toff', c_int),
                ('adjoint', c_int), ('errctl', c_int), ('deviceid', c_int), ('kernel', c_int),
                ('halo', c_void_p), ('free_surface', c_int), ('timers', POINTER(Profiler))]


class Tap(Structure):
    _fields_ = [('tshift', c_int), ('off', c_int * 3), ('coef', c_float)]


class SysTap(Structure):
    _fields_ = [('field', c_int), ('tshift', c_int), ('off', c_int * 3), ('coef', c_float), ('cfield', c_int)]


class SysStage(Structure):
    _fields_ = [('out_field', c_int), ('out_tshift', c_int), ('ntaps', c_int), ('taps', POINTER(SysTap)),
                ('ext', c_int)]


class SysInject(Structure):
    _fields_ = [('s', POINTER(Sparse)), ('nfields', c_int), ('fields', c_int * 3), ('tshift', c_int),
                ('scale', c_float), ('param_kind', c_int), ('param', POINTER(Dataobj))]


class SysInterp(Structure):
    _fields_ = [('s', POINTER(Sparse)), ('field', c_int), ('tshift', c_int)]


class SystemArgs(Structure):
    _fields_ = [('ndim', c_int), ('halo', c_int), ('nfields', c_int), ('fields', POINTER(POINTER(Dataobj))),
                ('ncoefs', c_int), ('coefs', POINTER(POINTER(Dataobj))),
                ('nstages', c_int), ('stages', POINTER(SysStage)),
                ('ninject', c_int), ('ninterp', c_int), ('inject', POINTER(SysInject)), ('interp', POINTER(SysInterp)),
                ('x_m', c_int), ('x_M', c_int), ('y_m', c_int), ('y_M', c_int), ('z_m', c_int), ('z_M', c_int),
                ('time_m', c_int), ('time_M', c_int), ('deviceid', c_int), ('timers', POINTER(Profiler))]


SYS_MAX_FIELDS, SYS_MAX_COEFS, SYS_MAX_TAPS = 24, 48, 160


class LinearArgs(Structure):
    _fields_ = [('ndim', c_int), ('f', POINTER(Dataobj)), ('halo', c_int), ('ntaps', c_int),
                ('taps', POINTER(Tap)), ('wshift', c_int),
                ('x_m', c_int), ('x_M', c_int), ('y_m', c_int), ('y_M', c_int), ('z_m', c_int), ('z_M', c_int),
                ('time_m', c_int), ('time_M', c_int), ('deviceid', c_int), ('timers', POINTER(Profiler))]


MAX_TAPS = 64

# action kinds of b2_iso_gradient_revolve
REVOLVE_ACTIONS = {'advance': 0, 'takeshot': 1, 'restore': 2, 'reverse': 3}

_lib = None

# every symbol include/b200stencil.h declares
SYMBOLS = ['b2_iso_forward', 'b2_iso_gradient_revolve', 'b2_revolve_check', 'b2_tti_forward', 'b2_sa_forward', 'b2_visco_forward', 'b2_linear_forward', 'b2_system_forward', 'b2_nccl_unique_id', 'b2_halo_create',
           'b2_halo_destroy', 'b2_halo_update', 'b2_device_count', 'b2_last_error', 'b2_version',
           'b2_launch_count', 'b2_last_sweep_kernel', 'b2_last_iso_coef_reuse', 'b2_kernel_timing_reset', 'b2_kernel_timing_ms',
           'b2_kernel_timing_enable', 'b2_malloc_device', 'b2_free_device', 'b2_memcpy_h2d',
           'b2_memcpy_d2h', 'b2_memset_device', 'b2_synchronize', 'b2_set_stream',
           'b2_staging_cache_release', 'b2_staging_outstanding', 'b2_last_call_profile', 'b2_device_pci_bus_id',
           'b2_ipc_get_handle', 'b2_ipc_open', 'b2_ipc_close', 'b2_halo_p2p_setup',
           'b2_halo_p2p_register']


def have_lib():
    return os.path.exists(LIB_PATH)


def load_library():
    """Load the shared object and declare signatures (no GPU needed for this)."""
    global _lib
    if _lib is not None:
        return _lib
    if not have_lib():
        raise BackendUnavailable(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C devito_b200/csrc`). The wave-propagation path has no CPU fallback.")
    L = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
    L.b2_iso_forward.argtypes = [POINTER(IsoArgs)]
    L.b2_iso_forward.restype = c_int
    L.b2_iso_gradient_revolve.argtypes = [POINTER(IsoArgs), POINTER(IsoArgs), POINTER(c_int), c_int, c_int]
    L.b2_iso_gradient_revolve.restype = c_int
    L.b2_revolve_check.argtypes = [POINTER(c_int), c_int, c_int, c_int, c_int, c_int, c_int]
    L.b2_revolve_check.restype = c_int
    L.b2_tti_forward.argtypes = [POINTER(TtiArgs)]
    L.b2_tti_forward.restype = c_int
    L.b2_sa_forward.argtypes = [POINTER(SaArgs)]
    L.b2_sa_forward.restype = c_int
    L.b2_visco_forward.argtypes = [POINTER(ViscoArgs)]
    L.b2_visco_forward.restype = c_int
    L.b2_linear_forward.argtypes = [POINTER(LinearArgs)]
    L.b2_linear_forward.restype = c_int
    L.b2_system_forward.argtypes = [POINTER(SystemArgs)]
    L.b2_system_forward.restype = c_int
    L.b2_nccl_unique_id.argtypes = [c_char_p, c_char_p]
    L.b2_nccl_unique_id.restype = c_int
    L.b2_halo_create.argtypes = [c_char_p, c_char_p, c_int, c_int, c_int]
    L.b2_halo_create.restype = c_void_p
    L.b2_halo_destroy.argtypes = [c_void_p]
    L.b2_halo_destroy.restype = None
    L.b2_halo_update.argtypes = [c_void_p, POINTER(Dataobj), c_int, c_int]
    L.b2_halo_update.restype = c_int
    L.b2_device_count.restype = c_int
    L.b2_last_error.restype = c_char_p
    L.b2_version.restype = c_char_p
    L.b2_launch_count.restype = c_ulonglong
    L.b2_last_sweep_kernel.argtypes = []
    L.b2_last_sweep_kernel.restype = c_char_p
    L.b2_last_iso_coef_reuse.argtypes = []
    L.b2_last_iso_coef_reuse.restype = c_int
    L.b2_kernel_timing_reset.restype = None
    L.b2_kernel_timing_ms.argtypes = [POINTER(c_int)]
    L.b2_kernel_timing_ms.restype = c_double
    L.b2_kernel_timing_enable.argtypes = [c_int]
    L.b2_kernel_timing_enable.restype = None
    L.b2_malloc_device.argtypes = [c_ulong, c_int]
    L.b2_malloc_device.restype = c_void_p
    L.b2_free_device.argtypes = [c_void_p, c_int]
    L.b2_free_device.restype = None
    L.b2_memcpy_h2d.argtypes = [c_void_p, c_void_p, c_ulong, c_int]
    L.b2_memcpy_h2d.restype = c_int
    L.b2_memcpy_d2h.argtypes = [c_void_p, c_void_p, c_ulong, c_int]
    L.b2_memcpy_d2h.restype = c_int
    L.b2_memset_device.argtypes = [c_void_p, c_int, c_ulong, c_int]
    L.b2_memset_device.restype = c_int
    L.b2_synchronize.argtypes = [c_int]
    L.b2_synchronize.restype = c_int
    L.b2_set_stream.argtypes = [c_void_p]
    L.b2_set_stream.restype = None
    L.b2_staging_cache_release.argtypes = []
    L.b2_staging_cache_release.restype = None
    L.b2_staging_outstanding.argtypes = []
    L.b2_staging_outstanding.restype = c_ulonglong
    L.b2_last_call_profile.argtypes = [POINTER(c_double)]
    L.b2_last_call_profile.restype = None
    L.b2_device_pci_bus_id.argtypes = [c_int, c_char_p, c_int]
    L.b2_device_pci_bus_id.restype = c_int
    L.b2_ipc_get_handle.argtypes = [c_void_p, c_char_p]
    L.b2_ipc_get_handle.restype = c_int
    L.b2_ipc_open.argtypes = [c_char_p]
    L.b2_ipc_open.restype = c_void_p
    L.b2_ipc_close.argtypes = [c_void_p]
    L.b2_ipc_close.restype = c_int
    L.b2_halo_p2p_setup.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p]
    L.b2_halo_p2p_setup.restype = c_int
    L.b2_halo_p2p_register.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int]
    L.b2_halo_p2p_register.restype = c_int
    _lib = L
    return L


_gpu_checked = None


def have_gpu():
    global _gpu_checked
    if _gpu_checked is None:
        try:
            _gpu_checked = load_library().b2_device_count() > 0
        except BackendUnavailable:
            _gpu_checked = False
    return _gpu_checked


def lib():
    """The library, ready to compute. Raises BackendUnavailable without a GPU."""
    L = load_library()
    if not have_gpu():
        raise BackendUnavailable("no CUDA device visible: the wave-propagation path runs only on the "
                                 "GPU (there is deliberately no CPU fallback)")
    return L


def nccl_library_path():
    try:
        import nvidia.nccl as n
        p = os.path.join(list(n.__path__)[0], 'lib', 'libnccl.so.2')
        if os.path.exists(p):
            return p.encode()
    except Exception:
        pass
    return b'libnccl.so.2'


class DataobjHolder:
    """Keeps the ctypes arrays (and the ndarray) alive next to the struct, like the reference
    stashes the ndarray on the ctypes object (devito/types/dense.py:774-776)."""

    def __init__(self, host=None, dev_ptr=None, shape=None, halo=None, itemsize=4):
        if host is not None:
            assert host.flags['C_CONTIGUOUS']
            shape = host.shape
            itemsize = host.dtype.itemsize
        self.host = host
        nd = len(shape)
        self._size = (c_int * nd)(*[int(s) for s in shape])
        halo = halo or tuple((0, 0) for _ in shape)
        flat = [int(v) for pair in halo for v in pair]
        self._hsize = (c_int * (2 * nd))(*flat)
        self._hofs = (c_int * (2 * nd))(*[0] * (2 * nd))
        self._oofs = (c_int * (2 * nd))(*[0] * (2 * nd))
        self.obj = Dataobj()
        self.obj.data = host.ctypes.data if host is not None else None
        self.obj.size = ctypes.cast(self._size, POINTER(c_int))
        self.obj.nbytes = int(np.prod(shape)) * itemsize
        self.obj.npsize = None
        self.obj.dsize = None
        self.obj.hsize = ctypes.cast(self._hsize, POINTER(c_int))
        self.obj.hofs = ctypes.cast(self._hofs, POINTER(c_int))
        self.obj.oofs = ctypes.cast(self._oofs, POINTER(c_int))
        self.obj.dmap = dev_ptr

    @property
    def ptr(self):
        return ctypes.pointer(self.obj)


def make_dataobj(host=None, dev_ptr=None, shape=None, halo=None):
    return DataobjHolder(host=host, dev_ptr=dev_ptr, shape=shape, halo=halo)


class ForeignDataobj:
    """A `struct dataobj` somebody else built — the reference's own `_C_make_dataobj`
    (devito/types/dense.py:749-777) when its Operator hands its arguments to this backend
    (devito_b200/refplugin.py). The struct is used as it is: same field layout, `data` = host array,
    `size` = allocated extents (halo included), `dmap` = NULL (host-staged by the library)."""

    def __init__(self, address, keep=None):
        self.obj = Dataobj.from_address(int(address))
        self._keep = keep                      # whatever owns the struct's memory

    @property
    def ptr(self):
        return ctypes.pointer(self.obj)

    def shape(self, ndim):
        return tuple(int(self.obj.size[i]) for i in range(ndim))


class ForeignSparse:
    """A sparse time function described by foreign structs: traces `data` (nt, npoint), base cells `gp`
    (npoint, ndim, int32) and per-dimension weight tables (npoint, 2r) — the arguments `src, src_gp,
    src_wx, ...` the reference computes for its own generated kernel
    (devito/operations/interpolators.py:674-718)."""
    is_SparseTimeFunction = True
    is_foreign = True

    def __init__(self, name, data, gp, ws, p_m, p_M, r):
        self.name, self.data, self.gp, self.ws = name, data, gp, list(ws)
        self.p_m, self.p_M, self.r = int(p_m), int(p_M), int(r)
        self.nt, self.npoint = data.shape(2)
