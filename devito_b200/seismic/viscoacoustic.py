"""Second-order SLS viscoacoustic modelling (mirror of examples/seismic/viscoacoustic/operators.py and wavesolver.py at
kernel='sls', time_order=2): forward and adjoint operators on the CUDA path (`b2_visco_forward`). With
t_s = (sqrt(1 + 1/qp^2) - 1/qp)/f0, tt = 1/(f0^2 t_s^2) - 1, rho = 1/b and L(f) = div(b grad(f, shift=.5), shift=-.5):

    r.forward = damp * solve(r.dt - (tt/t_s) rho L(p) + r/t_s, r.forward)
    p.forward = damp * solve(m p.dt2 - rho (1+tt) L(p) + r.forward + (1-damp) p.dt, p.forward)

and the adjoint pair of operators.py:176-190. `damp` is the model's "mask" profile. The first-order kernels, the
Kelvin-Voigt and Maxwell rheologies and the linearised operators are not on this path yet.
"""
from .. import Eq, Operator, TimeFunction, solve, sqrt
from ..tools import memoized_meth

__all__ = ['sls_2nd_order', 'ForwardOperator', 'AdjointOperator', 'ViscoacousticWaveSolver']

_SUPPORTED = "only kernel='sls' with time_order=2 (forward and adjoint) is on this backend's path"


def _check_kernel(kernel, time_order):
    if str(kernel).lower() != 'sls' or time_order != 2:
        raise NotImplementedError(f"viscoacoustic kernel={kernel!r} time_order={time_order}: {_SUPPORTED}")


def _nested(f, b, dims):
    """div(b * grad(f, shift=.5), shift=-.5) of a field or an expression: per dimension the half-node derivative at
    d + h/2, times b at the node, differentiated back at d - h/2 (the reference's staggered `grad` / `div`)."""
    out = 0
    for d, deriv in zip(dims, ('dx', 'dy', 'dz')):
        inner = getattr(f, deriv)(x0=d + d.spacing / 2)
        out = out + getattr(b * inner, deriv)(x0=d - d.spacing / 2)
    return out


def sls_2nd_order(model, geometry, p, r=None, **kwargs):
    """operators.py:124-192: [Eq(r.forward|backward, ...), Eq(p.forward|backward, ...)]."""
    forward = kwargs.get('forward', True)
    save = kwargs.get('save', False)
    b, m, damp, qp = model.b, model.m, model.damp, model.qp
    f0 = geometry._f0
    q = kwargs.get('q', 0)
    t_s = (sqrt(1. + 1. / qp ** 2) - 1. / qp) / f0
    t_ep = 1. / (f0 ** 2 * t_s)
    tt = (t_ep / t_s) - 1.
    rho = 1. / b
    r = r or TimeFunction(name="r", grid=model.grid, time_order=2, space_order=p.space_order,
                          save=geometry.nt if save else None)
    dims = p.dimensions[1:]
    if forward:
        pde_r = r.dt - (tt / t_s) * rho * _nested(p, b, dims) + (1. / t_s) * r
        u_r = Eq(r.forward, damp * solve(pde_r, r.forward))
        pde_p = m * p.dt2 - rho * (1. + tt) * _nested(p, b, dims) + r.forward - q + (1 - damp) * p.dt
        u_p = Eq(p.forward, damp * solve(pde_p, p.forward))
        return [u_r, u_p]
    pde_r = r.dt.T + (tt / t_s) * p + (1. / t_s) * r
    u_r = Eq(r.backward, damp * solve(pde_r, r.backward))
    pde_p = m * p.dt2 - _nested((1. + tt) * rho * p, b, dims) - _nested(rho * r.backward, b, dims) + \
        (1 - damp) * p.dt.T
    u_p = Eq(p.backward, damp * solve(pde_p, p.backward))
    return [u_r, u_p]


def _src_rec(p, model, geometry, forward=True):
    """operators.py:9-37: injection scaled by dt^2/m, interpolation of p."""
    dt = model.grid.time_dim.spacing
    scale = dt ** 2 / model.m
    src, rec = geometry.src, geometry.rec
    if forward:
        return src.inject(field=p.forward, expr=src * scale) + rec.interpolate(expr=p)
    return src.interpolate(expr=p) + rec.inject(field=p.backward, expr=rec * scale)


def ForwardOperator(model, geometry, space_order=4, kernel='sls', time_order=2, save=False, **kwargs):
    """operators.py:482-528."""
    _check_kernel(kernel, time_order)
    p = TimeFunction(name="p", grid=model.grid, time_order=2, space_order=space_order,
                     save=geometry.nt if save else None)
    eqn = sls_2nd_order(model, geometry, p, save=save)
    return Operator(eqn + _src_rec(p, model, geometry), subs=model.spacing_map, name='ViscoIsoAcousticForward',
                    **kwargs)


def AdjointOperator(model, geometry, space_order=4, kernel='sls', time_order=2, **kwargs):
    """operators.py:531-569."""
    _check_kernel(kernel, time_order)
    pa = TimeFunction(name="pa", grid=model.grid, time_order=2, space_order=space_order)
    eqn = sls_2nd_order(model, geometry, pa, forward=False)
    return Operator(eqn + _src_rec(pa, model, geometry, forward=False), subs=model.spacing_map, name='Adjoint',
                    **kwargs)


class ViscoacousticWaveSolver:
    """wavesolver.py:11-227 at kernel='sls', time_order=2: forward and adjoint modelling. The model's damping field
    becomes the "mask" profile (1 inside, below 1 in the absorbing layers)."""

    def __init__(self, model, geometry, space_order=4, kernel='sls', time_order=2, **kwargs):
        _check_kernel(kernel, time_order)
        self.model = model
        self.model._initialize_bcs(bcs="mask")
        self.geometry = geometry
        self.space_order = space_order
        self.kernel = kernel
        self.time_order = time_order
        self._kwargs = kwargs

    @property
    def dt(self):
        return self.model.critical_dt

    @memoized_meth
    def op_fwd(self, save=None):
        return ForwardOperator(self.model, save=save, geometry=self.geometry, space_order=self.space_order,
                               kernel=self.kernel, time_order=self.time_order, **self._kwargs)

    @memoized_meth
    def op_adj(self):
        return AdjointOperator(self.model, geometry=self.geometry, space_order=self.space_order,
                               kernel=self.kernel, time_order=self.time_order, **self._kwargs)

    def forward(self, src=None, rec=None, v=None, r=None, p=None, model=None, save=None, **kwargs):
        """wavesolver.py:78-149: returns (rec, p, v, summary); v is None at time_order=2."""
        src = src or self.geometry.src
        rec = rec or self.geometry.rec
        save_t = src.nt if save else None
        p = p or TimeFunction(name="p", grid=self.model.grid, save=save_t, time_order=2,
                              space_order=self.space_order)
        r = r or TimeFunction(name="r", grid=self.model.grid, save=save_t, time_order=2,
                              space_order=self.space_order)
        model = model or self.model
        kwargs.update(model.physical_params(**kwargs))
        summary = self.op_fwd(save).apply(src=src, rec=rec, r=r, p=p, dt=kwargs.pop('dt', self.dt), **kwargs)
        return rec, p, v, summary

    def adjoint(self, rec, srca=None, va=None, pa=None, r=None, model=None, **kwargs):
        """wavesolver.py:151-209: returns (srca, pa, va, summary); va is None at time_order=2."""
        srca = srca or self.geometry.new_src(name='srca', src_type=None)
        pa = pa or TimeFunction(name="pa", grid=self.model.grid, time_order=2, space_order=self.space_order)
        r = r or TimeFunction(name="r", grid=self.model.grid, time_order=2, space_order=self.space_order)
        model = model or self.model
        kwargs.update(model.physical_params(**kwargs))
        summary = self.op_adj().apply(src=srca, rec=rec, pa=pa, r=r, dt=kwargs.pop('dt', self.dt), **kwargs)
        return srca, pa, va, summary

    def jacobian(self, *args, **kwargs):
        raise NotImplementedError(f"the viscoacoustic Born operator is not on this backend's path yet; {_SUPPORTED}")

    def jacobian_adjoint(self, *args, **kwargs):
        raise NotImplementedError(f"the viscoacoustic gradient operator is not on this backend's path yet; "
                                  f"{_SUPPORTED}")
