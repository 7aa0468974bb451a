"""Self-adjoint variable-density visco-acoustic modelling (mirror of examples/seismic/self_adjoint/operators.py,
wavesolver.py, utils.py and example_iso.py): forward and adjoint operators on the CUDA path (`b2_sa_forward`).

The update, with b = 1/rho the buoyancy and w = w/Q the dissipation-only attenuation (`model.damp`),

    u.forward = dt^2 vp^2/b * sum_d (b u.d(x0=d+h/2)).d(x0=d-h/2) + (2 - dt w) u + (dt w - 1) u.backward

is self-adjoint: the adjoint is the same stencil run backwards in time. The linearised pair (`jacobian`,
`jacobian_adjoint`) is not on this path yet.
"""
import numpy as np

from .. import Eq, Operator, TimeFunction
from ..tools import memoized_meth
from .geometry import setup_geometry
from .model import Model

__all__ = ['iso_stencil', 'IsoFwdOperator', 'IsoAdjOperator', 'SaIsoAcousticWaveSolver', 'setup_w_over_q',
           'acoustic_sa_setup']


def iso_stencil(field, model, **kwargs):
    """operators.py:4-65: the time update of `field` (forward=True: field.forward from field, field.backward)."""
    vp, b, wOverQ = model.vp, model.b, model.damp
    forward = kwargs.get('forward', True)
    field_next = field.forward if forward else field.backward
    field_prev = field.backward if forward else field.forward
    q = kwargs.get('q', 0)
    t = field.dimensions[0]
    div = q
    for d, deriv in zip(field.dimensions[1:], ('dx', 'dy', 'dz')):
        inner = getattr(field, deriv)(x0=d + d.spacing / 2)
        div = div + getattr(b * inner, deriv)(x0=d - d.spacing / 2)
    update = (t.spacing ** 2 * vp ** 2 / b) * div + (2 - t.spacing * wOverQ) * field + \
        (t.spacing * wOverQ - 1) * field_prev
    return [Eq(field_next, update)]


def IsoFwdOperator(model, geometry, space_order=8, save=False, **kwargs):
    """operators.py:68-113: source injected into u.forward with dt^2 vp^2/b, receivers sample u."""
    src, rec = geometry.src, geometry.rec
    vp, b = model.vp, model.b
    u = TimeFunction(name='u', grid=model.grid, save=geometry.nt if save else None, time_order=2,
                     space_order=space_order)
    eqn = iso_stencil(u, model, forward=True)
    t = u.grid.time_dim
    src_term = src.inject(field=u.forward, expr=src * t.spacing ** 2 * vp ** 2 / b)
    rec_term = rec.interpolate(expr=u)
    return Operator(eqn + src_term + rec_term, subs=model.spacing_map, name='IsoFwdOperator', **kwargs)


def IsoAdjOperator(model, geometry, space_order=8, save=False, **kwargs):
    """operators.py:116-160: receiver data injected into v.backward with dt^2 vp^2/b, the adjoint source
    samples v."""
    rec, src = geometry.rec, geometry.src
    vp, b = model.vp, model.b
    v = TimeFunction(name='v', grid=model.grid, save=geometry.nt if save else None, time_order=2,
                     space_order=space_order)
    eqn = iso_stencil(v, model, forward=False)
    t = model.grid.time_dim
    rec_term = rec.inject(field=v.backward, expr=rec * t.spacing ** 2 * vp ** 2 / b)
    src_term = src.interpolate(expr=v)
    return Operator(eqn + rec_term + src_term, subs=model.spacing_map, name='IsoAdjOperator', **kwargs)


_JACOBIAN_LATER = ("the linearised self-adjoint operators (IsoJacobianFwdOperator / IsoJacobianAdjOperator: "
                   "u0.dt(x0=t-dt/2), the linearised source and the imaging term) are not on this backend's path "
                   "yet")


class SaIsoAcousticWaveSolver:
    """wavesolver.py:7-120: forward and adjoint modelling. The time step is the critical one at dt_scale .5
    (wavesolver.py:48-49)."""

    def __init__(self, model, geometry, space_order=8, **kwargs):
        self.model = model
        self.geometry = geometry
        assert self.model.grid == geometry.grid
        self.space_order = space_order
        # time step is .5 time smaller due to Q
        self.model.dt_scale = .5
        self._kwargs = kwargs

    @property
    def dt(self):
        return self.model.critical_dt

    @memoized_meth
    def op_fwd(self, save=None):
        return IsoFwdOperator(self.model, save=save, geometry=self.geometry, space_order=self.space_order,
                              **self._kwargs)

    @memoized_meth
    def op_adj(self, save=None):
        return IsoAdjOperator(self.model, save=save, geometry=self.geometry, space_order=self.space_order,
                              **self._kwargs)

    def op_jac(self, save=None):
        raise NotImplementedError(_JACOBIAN_LATER)

    def op_jacadj(self, save=True):
        raise NotImplementedError(_JACOBIAN_LATER)

    def forward(self, src=None, rec=None, b=None, vp=None, damp=None, u=None, save=None, **kwargs):
        """wavesolver.py:82-120: returns (rec, u, summary)."""
        src = src or self.geometry.src
        rec = rec or self.geometry.rec
        u = u or TimeFunction(name='u', grid=self.model.grid, save=self.geometry.nt if save else None,
                              time_order=2, space_order=self.space_order)
        kwargs.update(self.model.physical_params(vp=vp, damp=damp, b=b))
        kwargs.update({'dt': kwargs.pop('dt', self.dt)})
        summary = self.op_fwd(save).apply(src=src, rec=rec, u=u, **kwargs)
        return rec, u, summary

    def adjoint(self, rec, src=None, b=None, v=None, damp=None, vp=None, save=None, **kwargs):
        """wavesolver.py:122-165: returns (srca, v, summary)."""
        srca = src or self.geometry.new_src(name='srca', src_type=None)
        v = v or TimeFunction(name='v', grid=self.model.grid, save=self.geometry.nt if save else None,
                              time_order=2, space_order=self.space_order)
        kwargs.update(self.model.physical_params(vp=vp, damp=damp, b=b))
        kwargs.update({'dt': kwargs.pop('dt', self.dt)})
        summary = self.op_adj(save).apply(src=srca, rec=rec, v=v, **kwargs)
        return srca, v, summary

    def jacobian(self, dm, *args, **kwargs):
        raise NotImplementedError(_JACOBIAN_LATER)

    def jacobian_adjoint(self, rec, u0, *args, **kwargs):
        raise NotImplementedError(_JACOBIAN_LATER)


def w_over_q_profile(shape, w, qmin, qmax, npad):
    """NumPy evaluation of the profile `setup_w_over_q` builds (utils.py:8-63): 1 in the interior, the minimum over
    the axes of the distance to the nearest edge over npad inside the absorbing layers, then
    w / exp(log qmin + profile * (log qmax - log qmin))."""
    prof = np.ones(shape, dtype=np.float64)
    for d, n in enumerate(shape):
        i = np.arange(n, dtype=np.float64)
        dist = np.full(n, np.inf)
        dist[:npad] = i[:npad] / float(npad)
        dist[n - npad:] = np.minimum(dist[n - npad:], (n - 1 - i[n - npad:]) / float(npad))
        sh = [1] * len(shape)
        sh[d] = n
        prof = np.minimum(prof, dist.reshape(sh))
    lqmin, lqmax = np.log(qmin), np.log(qmax)
    return w / np.exp(lqmin + prof * (lqmax - lqmin))


def setup_w_over_q(wOverQ, w, qmin, qmax, npad, sigma=0):
    """utils.py:8-63. The reference writes the profile with an Operator using `Min`; this DSL has no `Min`, so the
    same profile is evaluated with NumPy and written into the domain of `wOverQ`."""
    assert w > 0, f"supplied w value [{w:f}] must be positive"
    assert qmin > 0, f"supplied qmin value [{qmin:f}] must be positive"
    assert qmax > 0, f"supplied qmax value [{qmax:f}] must be positive"
    assert npad > 0, f"supplied npad value [{npad:f}] must be positive"
    shape = wOverQ.grid.shape
    for n in shape:
        if n - 2 * npad < 1:
            raise ValueError("2 * npad must not exceed dimension size!")
    wOverQ.data[:] = w_over_q_profile(shape, w, qmin, qmax, npad).astype(wOverQ.grid.dtype)


def acoustic_sa_setup(shape=(50, 50, 50), spacing=(10.0, 10.0, 10.0), tn=500., space_order=8, nbl=10, **kwargs):
    """example_iso.py:9-34: constant vp = 1.5 and b = 1, w/Q from qmin 0.1 to qmax 1000 at 10 Hz."""
    if space_order < 8:
        space_order = 8
    qmin, qmax = 0.1, 1000.0
    fpeak = 0.010
    omega = 2.0 * np.pi * fpeak
    vp = 1.5 * np.ones(shape)
    b = 1.0 * np.ones(shape)

    def init_damp(func, nbl):
        return setup_w_over_q(func, omega, qmin, qmax, nbl, sigma=0)
    o = tuple([0] * len(shape))
    spacing = spacing[:len(shape)]
    model = Model(origin=o, shape=shape, vp=vp, b=b, spacing=spacing, nbl=nbl, space_order=space_order,
                  bcs=init_damp, dtype=kwargs.pop('dtype', np.float32), **kwargs)
    geometry = setup_geometry(model, tn)
    return SaIsoAcousticWaveSolver(model, geometry, space_order=space_order, **kwargs)
