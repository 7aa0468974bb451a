"""Physical model for seismic wave propagation (host-side mirror of the reference's
`examples/seismic/model.py`, written against this package's DSL).

Numerical definitions that matter for parity with the reference:
  * absorbing-layer profile `damp` — examples/seismic/model.py:25-63 (`initialize_damp`);
  * CFL time step — model.py:353-382 (`_cfl_coeff`, `critical_dt`: weights over +-space_order,
    value rounded through "%.3e" to the model dtype);
  * squared slowness m = 1/vp^2 — model.py:407-411;
  * parameters given as arrays are edge-padded into the absorbing layers — `_gen_phys_param`
    (model.py:180-191) via `initialize_function`.
"""
import numpy as np
from sympy import finite_diff_weights

from .. import (Grid, SubDomain, Function, Constant, Eq, Inc, Operator, SubDimension, Abs, sin,
                warning, mmax, mmin, initialize_function, gaussian_smooth)

__all__ = ['SeismicModel', 'Model', 'demo_model', 'initialize_damp']


def initialize_damp(damp, padsizes, spacing, abc_type="damp", fs=False):
    """Fill `damp` with the absorbing-layer profile. Written with the DSL (SubDimensions + Inc)
    exactly like the reference does, so that it exercises the generic operator path."""
    eqs = [Eq(damp, 1.0 if abc_type == "mask" else 0.0)]
    for (nbl, nbr), d in zip(padsizes, damp.dimensions):
        if not fs or d is not damp.dimensions[-1]:
            coeff = 1.5 * np.log(1.0 / 0.001) / nbl
            left = SubDimension.left(name=f'abc_{d.name}_l', parent=d, thickness=nbl)
            pos = Abs((nbl - (left - d.symbolic_min) + 1) / float(nbl))
            val = coeff * (pos - sin(2 * np.pi * pos) / (2 * np.pi))
            val = -val if abc_type == "mask" else val
            eqs.append(Inc(damp.subs({d: left}), val / d.spacing))
        coeff = 1.5 * np.log(1.0 / 0.001) / nbr
        right = SubDimension.right(name=f'abc_{d.name}_r', parent=d, thickness=nbr)
        pos = Abs((nbr - (d.symbolic_max - right) + 1) / float(nbr))
        val = coeff * (pos - sin(2 * np.pi * pos) / (2 * np.pi))
        val = -val if abc_type == "mask" else val
        eqs.append(Inc(damp.subs({d: right}), val / d.spacing))
    Operator(eqs, name='initdamp')()


class PhysicalDomain(SubDomain):
    """Where the wave equation is solved: the whole grid, or — with a free surface — everything
    below the top `space_order` rows, which `FSDomain` covers (examples/seismic/model.py:67-98)."""
    name = 'physdomain'

    def __init__(self, so, fs=False):
        super().__init__()
        self.so, self.fs = so, fs

    def define(self, dimensions):
        spec = dict.fromkeys(dimensions)
        for d in dimensions:
            spec[d] = d
        if self.fs:
            spec[dimensions[-1]] = ('middle', self.so, 0)
        return spec


class FSDomain(SubDomain):
    """The top `space_order` rows of the last dimension, updated with mirrored vertical taps."""
    name = 'fsdomain'

    def __init__(self, so):
        super().__init__()
        self.size = so

    def define(self, dimensions):
        spec = {d: d for d in dimensions}
        spec[dimensions[-1]] = ('left', self.size)
        return spec


_PARAMETER_NAMES = ('vp', 'damp', 'vs', 'b', 'epsilon', 'delta', 'theta', 'phi', 'qp', 'qs', 'lam', 'mu')


class SeismicModel:
    """Physical model on a grid extended by `nbl` absorbing points per side.

    Same constructor as the reference's `SeismicModel` (examples/seismic/model.py:238-322):
    `origin, spacing, shape, space_order, vp, nbl, dtype, bcs, **parameters` where every physical
    parameter is either a scalar (-> `Constant`) or an ndarray over the physical `shape`
    (-> `Function`, edge-padded into the absorbing layers and the halo)."""
    _known_parameters = list(_PARAMETER_NAMES)

    def __init__(self, origin, spacing, shape, space_order, vp, nbl=20, fs=False, dtype=np.float32,
                 subdomains=(), bcs="mask", grid=None, topology=None, **kwargs):
        if 'vs' in kwargs:
            raise NotImplementedError("elastic models are outside this backend's scope (SURVEY §8f)")
        self.shape = tuple(int(n) for n in shape)
        self.space_order = int(space_order)
        self.nbl = int(nbl)
        self.fs = bool(fs)
        self.origin = tuple(dtype(o) for o in origin)
        # free surface: no absorbing layer above the last dimension, whose origin stays put
        # (examples/seismic/model.py:113-131)
        ext_shape = [n + 2 * self.nbl for n in self.shape]
        ext_origin = [dtype(o - hh * self.nbl) for o, hh in zip(origin, spacing)]
        extra = (PhysicalDomain(space_order, fs=self.fs),)
        if self.fs:
            ext_shape[-1] -= self.nbl
            ext_origin[-1] = dtype(origin[-1])
            extra += (FSDomain(space_order),)
        ext_shape = tuple(ext_shape)
        if grid is not None:
            self.grid = grid
        else:
            h = np.asarray(spacing, dtype=np.float64)
            self.grid = Grid(shape=ext_shape, extent=tuple(h * (np.asarray(ext_shape) - 1)),
                             origin=tuple(ext_origin), dtype=dtype, topology=topology,
                             subdomains=tuple(subdomains) + extra)
        self._physical_parameters = set()
        self._dt = kwargs.get('dt')
        self._dt_scale = 1
        self.damp = None
        self._initialize_bcs(bcs=bcs)
        self.vp = self._gen_phys_param(vp, 'vp', space_order)
        for name in _PARAMETER_NAMES:
            value = kwargs.get(name)
            if value is not None and name not in ('vp', 'damp'):
                setattr(self, name, self._gen_phys_param(value, name, space_order))

    # -- absorbing boundary -------------------------------------------------------------------------
    def _initialize_bcs(self, bcs="damp"):
        """(Re-)build the damping field; wave solvers ask for the `"damp"` profile even when the
        model was created with the `"mask"` default (examples/seismic/model.py:138-162)."""
        if self.nbl == 0:
            self.damp = 1 if bcs == "mask" else 0
            return
        fresh = self.damp is None
        if fresh:
            self.damp = Function(name="damp", grid=self.grid, space_order=self.space_order)
        if callable(bcs):
            bcs(self.damp, self.nbl)
        else:
            wrong_kind = (mmin(self.damp) == 0) if bcs == "mask" else (mmax(self.damp) == 1)
            if fresh or wrong_kind:
                if not fresh:
                    warning(f"Re-initializing damp profile from {'damp' if bcs == 'mask' else 'mask'} to {bcs}")
                self._fill_damp(bcs)
        self._physical_parameters.add('damp')

    def _fill_damp(self, bcs):
        dist = self.grid.distributor
        if dist.is_parallel:
            # the profile follows GLOBAL indices: evaluate only this rank's x-slab
            self.damp.data[:] = damp_profile(self.grid.shape_global, self.padsizes, self.grid.spacing, bcs,
                                             x_range=dist.x_range)
        else:
            initialize_damp(self.damp, self.padsizes, self.spacing, abc_type=bcs, fs=self.fs)

    @property
    def padsizes(self):
        """(left, right) absorbing points per dimension; none above a free surface (model.py:166-172)."""
        pads = [(self.nbl, self.nbl)] * (self.dim - 1)
        return pads + [(0 if self.fs else self.nbl, self.nbl)]

    # -- parameters ------------------------------------------------------------------------------------
    def _gen_phys_param(self, field, name, space_order, default_value=0, **kwargs):
        if field is None:
            return default_value
        if isinstance(field, np.ndarray):
            obj = Function(name=name, grid=self.grid, space_order=space_order)
            initialize_function(obj, field, self.padsizes)
        else:
            obj = Constant(name=name, value=field, dtype=self.grid.dtype)
        self._physical_parameters.add(name)
        return obj

    @property
    def physical_parameters(self):
        return tuple(self._physical_parameters)

    def physical_params(self, **overrides):
        """{name: object} of all parameters, with user overrides by name."""
        out = {}
        for name in self._physical_parameters:
            obj = getattr(self, name)
            out[obj.name] = overrides.get(obj.name, obj) or obj
        return out

    def update(self, name, value):
        if not hasattr(self, name):
            setattr(self, name, self._gen_phys_param(value, name, self.space_order))
            return
        param = getattr(self, name)
        if not isinstance(value, np.ndarray):
            param.data = value
        elif value.shape == param.shape:
            param.data[:] = value
        elif value.shape == self.shape:
            initialize_function(param, value, self.nbl)
        else:
            raise ValueError(f"Incorrect input size {value.shape} for model {self.shape}")

    def smooth(self, physical_parameters, sigma=5.0):
        objs = self.physical_params()
        for name in physical_parameters:
            gaussian_smooth(objs[name], sigma=sigma)

    # -- geometry shortcuts ------------------------------------------------------------------------------
    dim = property(lambda self: self.grid.dim)
    spacing = property(lambda self: self.grid.spacing)
    space_dimensions = property(lambda self: self.grid.dimensions)
    spacing_map = property(lambda self: self.grid.spacing_map)
    dtype = property(lambda self: self.grid.dtype)

    @property
    def domain_size(self):
        return tuple((n - 1) * h for n, h in zip(self.shape, self.spacing))

    @property
    def m(self):
        """Squared slowness 1/vp^2 (examples/seismic/model.py:407-411)."""
        return 1 / (self.vp * self.vp)

    # -- time step ------------------------------------------------------------------------------------------
    dt_scale = property(lambda self: self._dt_scale, lambda self, v: setattr(self, '_dt_scale', v))

    @property
    def _cfl_coeff(self):
        """sqrt(4 / (ndim * sum|w|)) with w = second-derivative weights over +-space_order points
        (examples/seismic/model.py:353-367)."""
        w = finite_diff_weights(2, range(-self.space_order, self.space_order + 1), 0)[-1][-1]
        return np.sqrt(4.0 / float(self.grid.dim * np.sum(np.abs(np.array(w, dtype=np.float64)))))

    @property
    def critical_dt(self):
        """CFL time step, rounded through "%.3e" to the model dtype (model.py:370-382)."""
        if self._dt:
            return self._dt
        # the maxima are full-array reductions (80 ms per apply for vp and epsilon at 512^3, more than a third of a
        # 32-step propagation): recomputed only after somebody obtained write access to the parameter arrays
        pars = [self.vp] + ([self.epsilon] if 'epsilon' in self._physical_parameters else [])
        key = tuple((id(p), getattr(getattr(p, 'storage', None), 'version', None) if hasattr(p, 'storage')
                     else float(getattr(p, 'data', p))) for p in pars) + (self.dt_scale,)
        cached = getattr(self, '_critical_dt_cache', None)
        # under decomposition the maxima are collectives: every rank must take the same branch, so no rank-local
        # shortcut there
        parallel = self.grid.distributor.is_parallel
        # a view of a parameter kept by the caller may have been written since without a new access
        viewed = any(p.storage.views_held() for p in pars if hasattr(p, 'storage'))
        if not parallel and not viewed and cached is not None and cached[0] == key and \
                None not in [k[1] for k in key[:-1]]:
            return cached[1]
        vmax = mmax(self.vp)
        aniso = np.sqrt(1 + 2 * mmax(self.epsilon)) if 'epsilon' in self._physical_parameters else 1
        dt = self._cfl_coeff * np.min(self.spacing) / (aniso * vmax)
        out = self.dtype("%.3e" % (self.dt_scale * dt))
        # the key is taken again AFTER the reductions: `data` accessors used by a reduction may count as accesses
        key = tuple((id(p), getattr(getattr(p, 'storage', None), 'version', None) if hasattr(p, 'storage')
                     else float(getattr(p, 'data', p))) for p in pars) + (self.dt_scale,)
        self._critical_dt_cache = (key, out)
        return out


Model = SeismicModel


def damp_profile(shape, padsizes, spacing, abc_type="damp", x_range=None):
    """NumPy evaluation of the same profile as `initialize_damp`: the sum over dimensions of 1-D
    layer profiles in GLOBAL indices. `x_range=(lo, hi)` returns only that x-slab (used under
    slab decomposition, where each rank must not materialise the global array)."""
    lo, hi = x_range if x_range is not None else (0, shape[0])
    lshape = (hi - lo,) + tuple(shape[1:])
    out = np.full(lshape, 1.0 if abc_type == "mask" else 0.0, dtype=np.float32)
    for ax, ((nbl, nbr), h) in enumerate(zip(padsizes, spacing)):
        n = shape[ax]
        prof = np.zeros(n)
        if nbl > 0:
            i = np.arange(nbl)
            pos = np.abs((nbl - i + 1) / float(nbl))
            prof[:nbl] += 1.5 * np.log(1000.0) / nbl * (pos - np.sin(2 * np.pi * pos) / (2 * np.pi)) / float(h)
        j = np.arange(n - nbr, n)
        pos = np.abs((nbr - (n - 1 - j) + 1) / float(nbr))
        prof[n - nbr:] += 1.5 * np.log(1000.0) / nbr * (pos - np.sin(2 * np.pi * pos) / (2 * np.pi)) / float(h)
        if ax == 0:
            prof = prof[lo:hi]
        sh = [1] * len(shape)
        sh[ax] = len(prof)
        out += (-prof if abc_type == "mask" else prof).astype(np.float32).reshape(sh)
    return out


def demo_model(preset, **kwargs):
    """Preset models with the reference's names and defaults
    (examples/seismic/preset_models.py:20-238): `constant-isotropic`, `constant-tti`,
    `layers-isotropic`, `layers-tti`, `layers-viscoacoustic`."""
    space_order = kwargs.pop('space_order', 2)
    shape = kwargs.pop('shape', (101, 101))
    spacing = kwargs.pop('spacing', tuple(10. for _ in shape))
    origin = kwargs.pop('origin', tuple(0. for _ in shape))
    nbl = kwargs.pop('nbl', 10)
    dtype = kwargs.pop('dtype', np.float32)
    vp = kwargs.pop('vp', 1.5)
    nlayers = kwargs.pop('nlayers', 3)
    fs = kwargs.pop('fs', False)
    p = preset.lower()
    if fs and 'tti' in p:
        raise NotImplementedError("free-surface TTI models are not on this backend's path yet")
    if p == 'constant-isotropic':
        return SeismicModel(space_order=space_order, vp=vp, origin=origin, shape=shape, dtype=dtype,
                            spacing=spacing, nbl=nbl, fs=fs, **kwargs)
    if p in ('constant-tti', 'constant-tti-noazimuth'):
        phi = .35 if (len(shape) > 2 and p != 'constant-tti-noazimuth') else None
        return SeismicModel(space_order=space_order, vp=vp, origin=origin, shape=shape, dtype=dtype,
                            spacing=spacing, nbl=nbl, epsilon=.3, delta=.2, theta=.7, phi=phi,
                            bcs="damp", **kwargs)
    if p == 'layers-isotropic':
        vp_top = kwargs.pop('vp_top', 1.5)
        vp_bottom = kwargs.pop('vp_bottom', 3.5)
        v = np.empty(shape, dtype=dtype)
        v[:] = vp_top
        vp_i = np.linspace(vp_top, vp_bottom, nlayers)
        for i in range(1, nlayers):
            v[..., i * int(shape[-1] / nlayers):] = vp_i[i]
        return SeismicModel(space_order=space_order, vp=v, origin=origin, shape=shape, dtype=dtype,
                            spacing=spacing, nbl=nbl, bcs="damp", fs=fs, **kwargs)
    if p in ('layers-tti', 'layers-tti-noazimuth'):
        vp_top = kwargs.pop('vp_top', 1.5)
        vp_bottom = kwargs.pop('vp_bottom', 3.5)
        v = np.empty(shape, dtype=dtype)
        v[:] = vp_top
        vp_i = np.linspace(vp_top, vp_bottom, nlayers)
        for i in range(1, nlayers):
            v[..., i * int(shape[-1] / nlayers):] = vp_i[i]
        phi = .25 * (v - vp_top) if (len(shape) > 2 and p != 'layers-tti-noazimuth') else None
        return SeismicModel(space_order=space_order, vp=v, origin=origin, shape=shape, dtype=dtype,
                            spacing=spacing, nbl=nbl, epsilon=.1 * (v - vp_top), delta=.05 * (v - vp_top),
                            theta=.5 * (v - vp_top), phi=phi, bcs="damp", **kwargs)
    if p == 'layers-viscoacoustic':
        vp_top = kwargs.pop('vp_top', 1.5)
        vp_bottom = kwargs.pop('vp_bottom', 3.5)
        v = np.empty(shape, dtype=dtype)
        v[:] = vp_top
        vp_i = np.linspace(vp_top, vp_bottom, nlayers)
        for i in range(1, nlayers):
            v[..., i * int(shape[-1] / nlayers):] = vp_i[i]
        qp = (3.516 * ((v * 1000.) ** 2.2) * 10 ** (-6)).astype(dtype)     # Li's empirical formula
        b = (1.0 / (0.31 * (1e3 * v) ** 0.25)).astype(dtype)               # Gardner's density, not normalised
        return SeismicModel(space_order=space_order, vp=v, qp=qp, b=b, nbl=nbl, dtype=dtype, origin=origin,
                            shape=shape, spacing=spacing, **kwargs)
    raise ValueError(f"unknown or unsupported preset {preset!r}")
