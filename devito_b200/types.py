"""Dimensions, Grid, SubDomain, dense discrete functions and their data.

API surface mirrors what `examples/seismic` touches in the reference (SURVEY Appendix B):
`Grid` (devito/types/grid.py:72), `SubDomain`, `Dimension` family
(devito/types/dimension.py), `Function`/`TimeFunction` (devito/types/dense.py:971, :1478),
`Constant` (devito/types/constant.py).  Memory layout is the reference's: C row-major, halo =
`space_order` points per side on every space dimension (dense.py:1256-1259), time buffer of
`time_order+1` slots unless `save` is given (dense.py:1539-1540).

Data residency: every function owns a host array and, once a CUDA operator touched it, a
device mirror (a torch tensor used purely as an allocation).  `.data` access synchronises
device -> host lazily; the next CUDA operator re-uploads only if the host side was exposed.
Views the caller keeps across applies stay coherent in both directions: while a view of an
array is alive, every apply uploads that array before it runs and downloads it after writing
it, so an apply costs a copy of an array only while a view of it is held.
(The reference copies every array H2D/D2H on every `apply`, devito/passes/iet/definitions.py:636-671.)
"""
import sys

import numpy as np

from .symbolics import Symbol, Access, Index

__all__ = ['Dimension', 'SpaceDimension', 'TimeDimension', 'SteppingDimension', 'SubDimension',
           'DefaultDimension', 'ConditionalDimension', 'Grid', 'SubDomain', 'Function',
           'TimeFunction', 'Constant', 'Buffer', 'NODE', 'CELL']

NODE = 'node'
CELL = 'cell'


class Buffer:
    def __init__(self, val):
        self.val = int(val)


# ---------------------------------------------------------------------------------------------
# dimensions
# ---------------------------------------------------------------------------------------------
class Dimension(Symbol):
    is_Dimension = True
    is_Time = False
    is_Space = False
    is_Sub = False
    is_Stepping = False
    is_Conditional = False

    def __init__(self, name, spacing=None):
        super().__init__(name, dtype=np.int32)
        self._spacing = spacing if spacing is not None else Symbol(f'h_{name}')

    @property
    def spacing(self):
        return self._spacing

    @property
    def root(self):
        return self

    @property
    def parent(self):
        return None

    @property
    def symbolic_min(self):
        return Symbol(f'{self.name}_m', dtype=np.int32)

    @property
    def symbolic_max(self):
        return Symbol(f'{self.name}_M', dtype=np.int32)

    @property
    def symbolic_size(self):
        return Symbol(f'{self.name}_size', dtype=np.int32)

    @property
    def min_name(self):
        return f'{self.name}_m'

    @property
    def max_name(self):
        return f'{self.name}_M'


class SpaceDimension(Dimension):
    is_Space = True


class TimeDimension(Dimension):
    is_Time = True

    def __init__(self, name, spacing=None):
        super().__init__(name, spacing if spacing is not None else Symbol('dt'))


class SteppingDimension(Dimension):
    """Modulo-buffered time dimension `t` (devito/types/dimension.py:1753)."""
    is_Time = True
    is_Stepping = True

    def __init__(self, name, parent):
        super().__init__(name, parent.spacing)
        self._parent = parent

    @property
    def parent(self):
        return self._parent

    @property
    def root(self):
        return self._parent


class DefaultDimension(Dimension):
    def __init__(self, name, default_value=None):
        super().__init__(name)
        self.default_value = default_value


class SubDimension(Dimension):
    """A contiguous sub-range of a parent dimension (devito/types/dimension.py SubDimension):
    `left`: [m, m+thickness-1]; `right`: [M-thickness+1, M]; `middle`: [m+tl, M-tr]."""
    is_Sub = True

    def __init__(self, name, parent, kind, thickness_left=0, thickness_right=0):
        super().__init__(name, parent.spacing)
        self._parent = parent
        self.kind = kind
        self.thickness = (int(thickness_left), int(thickness_right))
        self.is_Space = parent.is_Space

    @classmethod
    def left(cls, name, parent, thickness, local=True):
        return cls(name, parent, 'left', thickness, 0)

    @classmethod
    def right(cls, name, parent, thickness, local=True):
        return cls(name, parent, 'right', 0, thickness)

    @classmethod
    def middle(cls, name, parent, thickness_left, thickness_right, local=False):
        return cls(name, parent, 'middle', thickness_left, thickness_right)

    @property
    def parent(self):
        return self._parent

    @property
    def root(self):
        return self._parent.root

    def bounds(self, pmin, pmax):
        """Inclusive index range given the parent's range."""
        tl, tr = self.thickness
        if self.kind == 'left':
            return pmin, pmin + tl - 1
        if self.kind == 'right':
            return pmax - tr + 1, pmax
        return pmin + tl, pmax - tr


class ConditionalDimension(Dimension):
    """Sub-sampled dimension (`factor`) — only time sub-sampling in the NumPy interpreter."""
    is_Conditional = True

    def __init__(self, name, parent, factor=None, condition=None):
        super().__init__(name, parent.spacing)
        self._parent = parent
        self.factor = factor
        self.condition = condition
        self.is_Time = parent.is_Time

    @property
    def parent(self):
        return self._parent

    @property
    def root(self):
        return self._parent.root


# ---------------------------------------------------------------------------------------------
# grid
# ---------------------------------------------------------------------------------------------
class SubDomain:
    """User-defined sub-region (devito/types/grid.py SubDomain). Subclasses provide `name` and
    `define(dimensions) -> {d: d | ('middle', l, r) | ('left', n) | ('right', n)}`."""
    name = None

    def __init__(self, *args, **kwargs):
        self._dimensions = None
        self.grid = kwargs.get('grid')

    def define(self, dimensions):
        return {d: d for d in dimensions}

    def __subdomain_finalize__(self, grid):
        self.grid = grid
        dims = []
        for d, v in self.define(grid.dimensions).items():
            if isinstance(v, Dimension):
                dims.append(v)
                continue
            kind = v[0]
            nm = f'i{self.name or "sd"}_{d.name}' if False else f'i{d.name}'
            if kind == 'middle':
                dims.append(SubDimension.middle(nm, d, v[1], v[2]))
            elif kind == 'left':
                dims.append(SubDimension.left(nm, d, v[1]))
            elif kind == 'right':
                dims.append(SubDimension.right(nm, d, v[1]))
            else:
                raise ValueError(f"unknown SubDomain spec {v!r}")
        self._dimensions = tuple(dims)

    @property
    def dimensions(self):
        return self._dimensions

    @property
    def dimension_map(self):
        return {d.root: d for d in self._dimensions}


class _Domain(SubDomain):
    name = 'domain'


class _Interior(SubDomain):
    name = 'interior'

    def define(self, dimensions):
        return {d: ('middle', 1, 1) for d in dimensions}


class Grid:
    """Cartesian grid (devito/types/grid.py:72)."""
    _default_names = ('x', 'y', 'z')

    def __init__(self, shape, extent=None, origin=None, dimensions=None, time_dimension=None,
                 dtype=np.float32, subdomains=None, comm=None, topology=None):
        shape = tuple(int(s) for s in (shape if np.iterable(shape) else (shape,)))
        self._glb_shape = shape
        ndim = len(shape)
        self._dtype = np.dtype(dtype).type
        extent = tuple(extent) if extent is not None else tuple(1.0 for _ in shape)
        origin = tuple(origin) if origin is not None else tuple(0.0 for _ in shape)
        self._extent = tuple(self._dtype(e) for e in extent)
        self._origin = tuple(self._dtype(o) for o in origin)
        if dimensions is None:
            if ndim > 3:
                raise ValueError("provide `dimensions` for grids with more than 3 dimensions")
            names = self._default_names[:ndim]
            dimensions = tuple(SpaceDimension(n) for n in names)
        self._dimensions = tuple(dimensions)
        self.time_dim = time_dimension or TimeDimension('time')
        self.stepping_dim = SteppingDimension('t', self.time_dim)
        # domain decomposition (x-slabs), see distributed.py
        from .distributed import Distributor
        self._distributor = Distributor(shape, self._dimensions, topology=topology)
        self._shape = self._distributor.shape
        # subdomains
        sds = [_Domain(), _Interior()] + list(subdomains or [])
        self._subdomains = {}
        for sd in sds:
            sd.__subdomain_finalize__(self)
            self._subdomains[sd.name] = sd

    def __repr__(self):
        return f"Grid[extent={self.extent}, shape={self.shape}, dimensions={self.dimensions}]"

    @property
    def dimensions(self): return self._dimensions
    @property
    def dim(self): return len(self._glb_shape)
    @property
    def shape(self): return self._shape                 # local (per-rank) shape
    @property
    def shape_local(self): return self._shape
    @property
    def shape_global(self): return self._glb_shape
    @property
    def extent(self): return self._extent
    @property
    def origin(self): return self._origin
    @property
    def dtype(self): return self._dtype
    @property
    def distributor(self): return self._distributor
    @property
    def subdomains(self): return self._subdomains
    @property
    def interior(self): return self._subdomains['interior']

    @property
    def spacing(self):
        return tuple(self._dtype(e / (s - 1)) if s > 1 else self._dtype(e)
                     for e, s in zip(self._extent, self._glb_shape))

    @property
    def spacing_symbols(self):
        return tuple(d.spacing for d in self._dimensions)

    @property
    def spacing_map(self):
        """{h_x: value} with the values in the grid dtype (devito/types/grid.py:311, 319-338)."""
        return dict(zip(self.spacing_symbols, self.spacing))

    @property
    def origin_map(self):
        return {Symbol(f'o_{d.name}'): o for d, o in zip(self._dimensions, self._origin)}

    @property
    def origin_offset(self):
        """Physical origin of this rank's sub-domain."""
        return tuple(self._dtype(o + off * h) for o, off, h in
                     zip(self._origin, self._distributor.offsets, self.spacing))

    @property
    def volume_cell(self):
        return float(np.prod(self.spacing))


# ---------------------------------------------------------------------------------------------
# data holder with lazy host/device mirrors
# ---------------------------------------------------------------------------------------------
class Data(np.ndarray):
    """ndarray view returned by `.data` (devito/data/data.py:14). Plain NumPy semantics."""

    def __new__(cls, array):
        return np.asarray(array).view(cls)


class RawDeviceBuffer:
    """Plain cudaMalloc allocation made through the C library (not torch's caching allocator), so
    that its CUDA IPC handle can be exported to the neighbour ranks (peer-memory halo path)."""

    def __init__(self, nbytes, deviceid):
        from ._lib import lib
        self.nbytes, self.deviceid = int(nbytes), int(deviceid)
        self.ptr = lib().b2_malloc_device(self.nbytes, self.deviceid)
        if not self.ptr:
            raise MemoryError(f"b2_malloc_device({self.nbytes}) failed")

    def data_ptr(self):
        return self.ptr

    @property
    def device(self):
        import torch
        return torch.device('cuda', self.deviceid)

    def __del__(self):
        try:
            from ._lib import lib
            if self.ptr:
                lib().b2_free_device(self.ptr, self.deviceid)
                self.ptr = None
        except Exception:
            pass


class FieldStorage:
    """Host array and device mirror of one dense function.

    `host_valid` / `dev_valid` say which copy is current. Views handed out by the accessors may be kept by the caller
    across applies: every NumPy view of the host array, however derived, holds a reference to it (NumPy points a
    view's `base` at the array that owns the data, here `_host` itself), so the host array's reference count above
    the storage's own says whether such a view is alive (`views_held`). While one is, the host array is the copy the
    caller reads and writes at any time: `to_device` uploads it even if the device copy looks current, and
    `mark_device_written` downloads the device copy at once."""
    raw = False          # True: device copy is a RawDeviceBuffer (IPC-exportable)
    p2p_registered = False
    _host_refs = 0       # references to `_host` with no caller view alive; 0: a host array the caller passed in

    def __init__(self, shape, dtype):
        self.shape = tuple(int(s) for s in shape)
        self.dtype = np.dtype(dtype)
        self._host = None
        self._pinned = None
        self.dev = None            # torch tensor (allocation only)
        self.host_valid = True
        self.dev_valid = False
        self.version = 0           # bumped whenever somebody obtains write access (host) or a kernel writes (device)

    def _alloc_host(self):
        if self._host is not None:
            return
        self._host = self._new_host()
        self._host_refs = sys.getrefcount(self._host)

    def _new_host(self):
        """A zeroed host array: page-locked (`_pinned`, a torch tensor sharing its memory) for arrays of 1 MiB or
        more when CUDA is present, else a plain NumPy array."""
        n = int(np.prod(self.shape))
        try:
            import torch
            if torch.cuda.is_available() and n * self.dtype.itemsize >= (1 << 20):
                tdt = {np.dtype(np.float32): torch.float32, np.dtype(np.int32): torch.int32,
                       np.dtype(np.float64): torch.float64}[self.dtype]
                try:
                    from .numa import bind_to_gpu
                    from .parameters import configuration
                    dev = configuration['deviceid']
                    bind_to_gpu(torch.cuda.current_device() if dev is None or dev < 0 else dev)
                except Exception:
                    pass
                self._pinned = torch.zeros(self.shape, dtype=tdt, pin_memory=True)
                return self._pinned.numpy()
        except Exception:
            self._pinned = None
        return np.zeros(self.shape, dtype=self.dtype)

    def views_held(self):
        """Whether a view of the host array is alive outside this storage."""
        return self._host is not None and sys.getrefcount(self._host) > self._host_refs

    @property
    def host(self):
        """Host array, up to date; the caller may write to it (device copy is invalidated)."""
        self._alloc_host()
        if not self.host_valid:
            self.sync_to_host()
        self.dev_valid = False
        self.version += 1
        return self._host

    @property
    def host_ro(self):
        """Host array, up to date; the caller promises not to write."""
        self._alloc_host()
        if not self.host_valid:
            self.sync_to_host()
        return self._host

    def sync_to_host(self):
        import torch
        self._alloc_host()
        if isinstance(self.dev, RawDeviceBuffer):
            from ._lib import lib
            rc = lib().b2_memcpy_d2h(self._host.ctypes.data, self.dev.ptr, self._host.nbytes, self.dev.deviceid)
            if rc:
                raise RuntimeError("device -> host copy failed")
            self.host_valid = True
            return
        src = self.dev
        if self._pinned is not None:
            self._pinned.copy_(src, non_blocking=False)
        else:
            self._host[...] = src.cpu().numpy()
        self.host_valid = True

    def to_device(self, device):
        """Device tensor holding current data (upload if the host copy is newer, or may be: while the caller keeps a
        view of the host array). A function whose host array was never touched is all zeros: it is created directly on
        the device."""
        import torch
        if self.raw:
            from ._lib import lib
            L = lib()
            nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
            if not isinstance(self.dev, RawDeviceBuffer):
                if self.dev is not None and not self.host_valid:
                    self.sync_to_host()
                self.dev = RawDeviceBuffer(nbytes, device.index)
                self.p2p_registered = False
                if self._host is None:
                    L.b2_memset_device(self.dev.ptr, 0, nbytes, device.index)
                    L.b2_synchronize(device.index)
                    self.dev_valid, self.host_valid = True, False
                    return self.dev
                self.dev_valid = False
            if not self.dev_valid or (self.host_valid and self.views_held()):
                self._upload()
            return self.dev
        tdt = {np.dtype(np.float32): torch.float32, np.dtype(np.int32): torch.int32,
               np.dtype(np.float64): torch.float64}[self.dtype]
        if self.dev is None or self.dev.device != device:
            if self._host is None:
                self.dev = torch.zeros(self.shape, dtype=tdt, device=device)
                # the fill runs on torch's current stream, the library launches on its own non-blocking
                # stream: finish the fill before anyone else touches the array
                torch.cuda.current_stream(device).synchronize()
                self.dev_valid = True
                self.host_valid = False
                return self.dev
            self.dev = torch.empty(self.shape, dtype=tdt, device=device)
            self.dev_valid = False
        if not self.dev_valid or (self.host_valid and self.views_held()):
            self._upload()
        return self.dev

    def _upload(self):
        """Host -> device copy of the whole array into the existing device allocation."""
        import torch
        self._alloc_host()
        if isinstance(self.dev, RawDeviceBuffer):
            from ._lib import lib
            if lib().b2_memcpy_h2d(self.dev.ptr, self._host.ctypes.data, self._host.nbytes, self.dev.deviceid):
                raise RuntimeError("host -> device copy failed")
        elif self._pinned is not None:
            self.dev.copy_(self._pinned, non_blocking=False)
        else:
            self.dev.copy_(torch.from_numpy(self._host))
        self.dev_valid = True

    def device_scratch(self, device):
        """A device buffer of this array's size WITHOUT uploading: staging space for a host-staged apply that moves
        the data itself (b2_iso_args.host_io). Raw (cudaMalloc) when `self.raw`, so that it can be CUDA-IPC
        registered with the neighbour ranks; kept across calls."""
        import torch
        nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        if self.raw:
            if not isinstance(self.dev, RawDeviceBuffer):
                if self.dev is not None and not self.host_valid:
                    self.sync_to_host()
                self.dev = RawDeviceBuffer(nbytes, device.index)
                self.p2p_registered = False
        elif self.dev is None or getattr(self.dev, 'device', None) != device:
            tdt = {np.dtype(np.float32): torch.float32, np.dtype(np.int32): torch.int32,
                   np.dtype(np.float64): torch.float64}[self.dtype]
            if self.dev is not None and not self.host_valid:
                self.sync_to_host()
            self.dev = torch.empty(self.shape, dtype=tdt, device=device)
        self.dev_valid = False
        return self.dev

    def mark_device_written(self):
        """A kernel wrote the device copy. Called once the write is complete: a view the caller keeps is brought up to
        date at once."""
        self.dev_valid = True
        self.host_valid = False
        self.version += 1
        if self.views_held():
            self.sync_to_host()

    def drop_device(self):
        if self.dev is not None and not self.host_valid:
            self.sync_to_host()
        self.dev = None
        self.dev_valid = False


# ---------------------------------------------------------------------------------------------
# discrete functions
# ---------------------------------------------------------------------------------------------
class DiscreteFunction(Access):
    """Base of Function/TimeFunction/SparseFunction. An instance *is* the access at its own
    dimensions, so it can be used directly in expressions (like in the reference)."""
    is_Function = False
    is_TimeFunction = False
    is_SparseFunction = False
    is_SparseTimeFunction = False
    is_DiscreteFunction = True
    time_dim = None
    time_order = 0

    __rkwargs__ = ('name', 'grid', 'dtype', 'space_order', 'shape', 'dimensions')

    def __new__(cls, *args, **kwargs):
        args, kwargs = cls.__args_setup__(*args, **kwargs)
        obj = object.__new__(cls)
        obj._ctor_kwargs = dict(kwargs)
        obj.__init_finalize__(*args, **kwargs)
        return obj

    def __init__(self, *args, **kwargs):
        pass

    @classmethod
    def __args_setup__(cls, *args, **kwargs):
        return args, kwargs

    def __init_finalize__(self, *args, **kwargs):
        raise NotImplementedError

    # Access protocol ---------------------------------------------------------------------------
    __hash__ = Access.__hash__

    @property
    def function(self):
        return self

    @function.setter
    def function(self, v):
        pass

    @property
    def name(self):
        return self._name

    @property
    def alias(self):
        return self._alias

    def __repr__(self):
        return f"{self._name}({', '.join(d.name for d in self.dimensions)})"

    __str__ = __repr__

    @property
    def is_Constant(self):
        return False

    # data -------------------------------------------------------------------------------------
    @property
    def dimensions(self): return self._dimensions
    @property
    def grid(self): return self._grid
    @property
    def dtype(self): return self._dtype
    @property
    def space_order(self): return self._space_order
    @property
    def shape(self): return self._shape
    @property
    def shape_domain(self): return self._shape
    @property
    def ndim(self): return len(self._shape)
    @property
    def shape_with_halo(self):
        return tuple(s + l + r for s, (l, r) in zip(self._shape, self._halo))
    shape_allocated = shape_with_halo

    @property
    def halo(self): return self._halo
    _size_halo = halo

    @property
    def _offset_domain(self):
        return tuple(l for l, _ in self._halo)

    @property
    def storage(self):
        if self._storage is None:
            self._storage = FieldStorage(self.shape_allocated, self._dtype)
        return self._storage

    def _domain_slices(self):
        return tuple(slice(l, l + s) for s, (l, _) in zip(self._shape, self._halo))

    @property
    def data(self):
        return Data(self.storage.host[self._domain_slices()])

    @data.setter
    def data(self, value):
        self.storage.host[self._domain_slices()] = value

    @property
    def data_ro_domain(self):
        return self.storage.host_ro[self._domain_slices()]

    @property
    def data_with_halo(self):
        return Data(self.storage.host)

    @property
    def data_ro_with_halo(self):
        return self.storage.host_ro

    _data_allocated = data_with_halo
    data_allocated = data_with_halo

    @property
    def _data(self):
        return self.storage.host


class Function(DiscreteFunction):
    """Space-varying discrete function (devito/types/dense.py:971)."""
    is_Function = True

    def __init_finalize__(self, *args, **kwargs):
        self._name = kwargs['name']
        self._alias = kwargs.get('alias', False)
        self._grid = kwargs.get('grid')
        self._space_order = int(kwargs.get('space_order', 1))
        dims = kwargs.get('dimensions')
        if dims is None:
            if self._grid is None:
                raise TypeError("Function needs `grid` or `dimensions`")
            dims = self._grid.dimensions
        self._dimensions = tuple(dims)
        shape = kwargs.get('shape')
        if shape is None:
            if self._grid is not None and all(d in self._grid.dimensions for d in self._dimensions):
                shape = tuple(self._grid.shape[self._grid.dimensions.index(d)] for d in self._dimensions)
            else:
                raise TypeError("Function needs `shape` when not defined on grid dimensions")
        self._shape = tuple(int(s) for s in shape)
        dtype = kwargs.get('dtype')
        self._dtype = np.dtype(dtype if dtype is not None else
                               (self._grid.dtype if self._grid is not None else np.float32)).type
        so = self._space_order
        self._halo = tuple((so, so) if d.is_Space else (0, 0) for d in self._dimensions)
        self._staggered = kwargs.get('staggered')
        self.avg_mode = kwargs.get('avg_mode', 'arithmetic')
        self._storage = None
        self._indices = tuple(Index(d, 0) for d in self._dimensions)
        init = kwargs.get('initializer')
        if init is not None:
            if callable(init):
                init(self.data_with_halo)
            else:
                self.data[:] = init

    @property
    def staggered(self):
        return self._staggered

    @property
    def is_parameter(self):
        return True


class TimeFunction(Function):
    """Time-varying discrete function (devito/types/dense.py:1478)."""
    is_TimeFunction = True

    def __init_finalize__(self, *args, **kwargs):
        grid = kwargs.get('grid')
        self.time_order = int(kwargs.get('time_order', 1))
        save = kwargs.get('save')
        self.save = save
        if isinstance(save, Buffer):
            self._time_size = save.val
            self.time_dim = kwargs.get('time_dim') or grid.stepping_dim
            self._stepping = True
        elif save is None:
            self._time_size = self.time_order + 1
            self.time_dim = kwargs.get('time_dim') or grid.stepping_dim
            self._stepping = True
        else:
            self._time_size = int(save)
            self.time_dim = kwargs.get('time_dim') or grid.time_dim
            self._stepping = False
        kw = dict(kwargs)
        kw['dimensions'] = (self.time_dim,) + tuple(kwargs.get('dimensions') or grid.dimensions)
        kw['shape'] = (self._time_size,) + tuple(kwargs.get('shape') or grid.shape)
        super().__init_finalize__(*args, **kw)

    @property
    def time_size(self):
        return self._time_size

    @property
    def is_buffered(self):
        return self._stepping

    @property
    def _time_buffering(self):
        return self._stepping


class Constant(Symbol):
    """Scalar runtime parameter (devito/types/constant.py)."""
    is_Constant = True

    def __init__(self, name=None, value=0, dtype=np.float32, **kwargs):
        super().__init__(name, dtype=dtype)
        self._value = np.dtype(dtype).type(value)
        self._dtype = np.dtype(dtype).type

    def _key(self):
        return ('K', self.name, id(self))

    @property
    def data(self):
        return self._value

    @data.setter
    def data(self, val):
        self._value = self._dtype(val)

    @property
    def value(self):
        return self._value

    @property
    def dtype_(self):
        return self._dtype

    @property
    def is_parameter(self):
        return True
