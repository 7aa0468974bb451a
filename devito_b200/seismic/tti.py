"""TTI (centred kernel) forward, adjoint, linearised (Born) and gradient modelling — mirror of
examples/seismic/tti/operators.py:12-247, 431-640 and tti/wavesolver.py (forward, adjoint, jacobian,
jacobian_adjoint)."""
from .. import Eq, Function, Inc, Operator, TimeFunction, solve, cos, sin, sqrt
from ..tools import memoized_meth

__all__ = ['kernel_centered', 'ForwardOperator', 'AdjointOperator', 'JacobianOperator', 'JacobianAdjOperator',
           'AnisotropicWaveSolver']


def trig_func(model):
    """operators.py `trig_func`: (cos theta, sin theta) on a 2-D model, which has no azimuth, and (cos theta, sin theta,
    cos phi, sin phi) in 3-D."""
    theta = getattr(model, 'theta', 0)
    grid = getattr(model, 'grid', None)
    if getattr(model, 'dim', grid.dim if grid is not None else 3) == 2:
        return cos(theta), sin(theta)
    phi = getattr(model, 'phi', 0)
    return cos(theta), sin(theta), cos(phi), sin(phi)


def _order1(field):
    # `field` may be an expression (the adjoint's mixes): its order is that of the fields it reads
    return (field.space_order if hasattr(field, 'space_order') else field._default_fd_order) // 2


def Gzz_centered(model, field):
    """Rotated second derivative along the symmetry axis (operators.py:65-104)."""
    costheta, sintheta, cosphi, sinphi = trig_func(model)
    order1 = _order1(field)
    x, y, z = field.grid.dimensions if hasattr(field, 'grid') else model.grid.dimensions
    dx, dy, dz = x.spacing / 2, y.spacing / 2, z.spacing / 2
    Gz = (sintheta * cosphi * field.dx(fd_order=order1, x0=x + dx) +
          sintheta * sinphi * field.dy(fd_order=order1, x0=y + dy) +
          costheta * field.dz(fd_order=order1, x0=z + dz))
    Gzz = (Gz * costheta).dz(fd_order=order1, x0=z - dz)
    if sintheta != 0:
        Gzz += (Gz * sintheta * cosphi).dx(fd_order=order1, x0=x - dx)
    if sinphi != 0:
        Gzz += (Gz * sintheta * sinphi).dy(fd_order=order1, x0=y - dy)
    return Gzz


def Gzz_centered_2d(model, field):
    """The 2-D rotated second derivative along the symmetry axis (operators.py `Gzz_centered_2d`): the rotation
    (sin theta, cos theta) on (x, z)."""
    costheta, sintheta = trig_func(model)
    order1 = _order1(field)
    x, z = field.grid.dimensions if hasattr(field, 'grid') else model.grid.dimensions
    dx, dz = x.spacing / 2, z.spacing / 2
    Gz = (sintheta * field.dx(fd_order=order1, x0=x + dx) +
          costheta * field.dy(fd_order=order1, x0=z + dz))
    Gzz = (Gz * costheta).dy(fd_order=order1, x0=z - dz)
    if sintheta != 0:
        Gzz += (Gz * sintheta).dx(fd_order=order1, x0=x - dx)
    return Gzz


def _is_zero(q):
    return isinstance(q, (int, float)) and q == 0


def kernel_centered(model, u, v, qu=0, qv=0, forward=True):
    """operators.py:186-247 + :12-39; `qu` / `qv` are extra sources of the u / v equations (the linearised
    operator passes -dm * u0.dt2 / -dm * v0.dt2). `forward=False` builds the adjoint pair: H0 = Gh(e2 u + sd v),
    Hz = Gzz(sd u + v), solved for u.backward / v.backward with the transposed damping term."""
    delta, epsilon = sqrt(1 + 2 * model.delta), 1 + 2 * model.epsilon
    Gzz_centered_ = Gzz_centered_2d if model.dim == 2 else Gzz_centered
    if not forward:
        m, damp = model.m, model.damp
        a, b = epsilon * u + delta * v, delta * u + v
        H0 = a.laplace - Gzz_centered_(model, a)
        Hz = Gzz_centered_(model, b)
        stencilp = solve(m * u.dt2 - H0 - qu + damp * u.dt.T, u.backward)
        stencilr = solve(m * v.dt2 - Hz - qv + damp * v.dt.T, v.backward)
        sd = model.grid.subdomains['physdomain']
        return [Eq(u.backward, stencilp, subdomain=sd), Eq(v.backward, stencilr, subdomain=sd)]
    Gxx = u.laplace - Gzz_centered_(model, u)
    Gzz = Gzz_centered_(model, v)
    H0 = epsilon * Gxx + delta * Gzz
    Hz = delta * Gxx + Gzz
    m, damp = model.m, model.damp
    pdeu = m * u.dt2 - H0 + damp * u.dt
    pdev = m * v.dt2 - Hz + damp * v.dt
    if not _is_zero(qu):
        pdeu = m * u.dt2 - H0 - qu + damp * u.dt
    if not _is_zero(qv):
        pdev = m * v.dt2 - Hz - qv + damp * v.dt
    stencilp = solve(pdeu, u.forward)
    stencilr = solve(pdev, v.forward)
    sd = model.grid.subdomains['physdomain']
    return [Eq(u.forward, stencilp, subdomain=sd), Eq(v.forward, stencilr, subdomain=sd)]


def ForwardOperator(model, geometry, space_order=4, save=False, kernel='centered', **kwargs):
    """operators.py:431-480"""
    if kernel != 'centered':
        raise NotImplementedError("only the centred TTI kernel is on this backend's path")
    dt = model.grid.time_dim.spacing
    m = model.m
    u = TimeFunction(name='u', grid=model.grid, save=geometry.nt if save else None, time_order=2,
                     space_order=space_order)
    v = TimeFunction(name='v', grid=model.grid, save=geometry.nt if save else None, time_order=2,
                     space_order=space_order)
    src, rec = geometry.src, geometry.rec
    stencils = kernel_centered(model, u, v)
    stencils += src.inject(field=(u.forward, v.forward), expr=src * dt ** 2 / m)
    stencils += rec.interpolate(expr=u + v)
    return Operator(stencils, subs=model.spacing_map, name='ForwardTTI', **kwargs)


def AdjointOperator(model, geometry, space_order=4, kernel='centered', **kwargs):
    """operators.py `AdjointOperator`: the adjoint pair (p, r) driven by the receivers, injected into
    (p.backward, r.backward); the adjoint source `srca` samples p + r."""
    if kernel != 'centered':
        raise NotImplementedError("only the centred TTI kernel is on this backend's path")
    dt = model.grid.time_dim.spacing
    m = model.m
    p = TimeFunction(name='p', grid=model.grid, time_order=2, space_order=space_order)
    r = TimeFunction(name='r', grid=model.grid, time_order=2, space_order=space_order)
    srca = geometry.new_src(name='srca', src_type=None)
    rec = geometry.rec
    stencils = kernel_centered(model, p, r, forward=False)
    stencils += rec.inject(field=(p.backward, r.backward), expr=rec * dt ** 2 / m)
    stencils += srca.interpolate(expr=p + r)
    return Operator(stencils, subs=model.spacing_map, name='AdjointTTI', **kwargs)


def JacobianOperator(model, geometry, space_order=4, **kwargs):
    """operators.py:532-586: the background pair (u0, v0) driven by the source, the linearised pair (du, dv) by
    -dm * u0.dt2 / -dm * v0.dt2, the receivers sampling du + dv."""
    dt = model.grid.stepping_dim.spacing
    m = model.m
    mk = lambda n: TimeFunction(name=n, grid=model.grid, save=None, time_order=2, space_order=space_order)
    u0, v0, du, dv = mk('u0'), mk('v0'), mk('du'), mk('dv')
    dm = Function(name='dm', grid=model.grid, space_order=0)
    src, rec = geometry.src, geometry.rec
    eqn1 = kernel_centered(model, u0, v0)
    eqn2 = kernel_centered(model, du, dv, qu=-dm * u0.dt2, qv=-dm * v0.dt2)
    src_term = src.inject(field=(u0.forward, v0.forward), expr=src * dt ** 2 / m)
    rec_term = rec.interpolate(expr=du + dv)
    return Operator(eqn1 + src_term + eqn2 + rec_term, subs=model.spacing_map, name='BornTTI', **kwargs)


def JacobianAdjOperator(model, geometry, space_order=4, save=True, **kwargs):
    """operators.py `JacobianAdjOperator`: the adjoint pair (du, dv) driven by the receivers and the imaging
    condition Inc(dm, -(u0 * du.dt2 + v0 * dv.dt2)) with the saved forward wavefields u0, v0."""
    dt = model.grid.stepping_dim.spacing
    m = model.m
    mk = lambda n, nt: TimeFunction(name=n, grid=model.grid, save=nt, time_order=2, space_order=space_order)
    u0, v0 = mk('u0', geometry.nt if save else None), mk('v0', geometry.nt if save else None)
    du, dv = mk('du', None), mk('dv', None)
    dm = Function(name='dm', grid=model.grid)
    rec = geometry.rec
    eqn = kernel_centered(model, du, dv, forward=False)
    dm_update = Inc(dm, -(u0 * du.dt2 + v0 * dv.dt2))
    rec_term = rec.inject(field=(du.backward, dv.backward), expr=rec * dt ** 2 / m)
    return Operator(eqn + rec_term + [dm_update], subs=model.spacing_map, name='GradientTTI', **kwargs)


class AnisotropicWaveSolver:
    def __init__(self, model, geometry, space_order=4, kernel='centered', **kwargs):
        self.model = model
        self.model._initialize_bcs(bcs="damp")
        self.geometry = geometry
        self.kernel = kernel
        if space_order % 2 != 0:
            raise ValueError("space_order must be even")
        self.space_order = space_order
        self._kwargs = kwargs

    @property
    def dt(self):
        return self.model.critical_dt

    @memoized_meth
    def op_fwd(self, save=False):
        return ForwardOperator(self.model, save=save, geometry=self.geometry,
                               space_order=self.space_order, kernel=self.kernel, **self._kwargs)

    def forward(self, src=None, rec=None, u=None, v=None, model=None, save=False, **kwargs):
        src = src or self.geometry.src
        rec = rec or self.geometry.rec
        mk = lambda n: TimeFunction(name=n, grid=self.model.grid, save=self.geometry.nt if save else None,
                                    time_order=2, space_order=self.space_order)
        u = u or mk('u')
        v = v or mk('v')
        model = model or self.model
        kwargs.update(model.physical_params(**kwargs))
        summary = self.op_fwd(save).apply(src=src, rec=rec, u=u, v=v, dt=kwargs.pop('dt', self.dt), **kwargs)
        return rec, u, v, summary

    @memoized_meth
    def op_jac(self):
        return JacobianOperator(self.model, self.geometry, space_order=self.space_order, **self._kwargs)

    def jacobian(self, dm, src=None, rec=None, u0=None, v0=None, du=None, dv=None, model=None, **kwargs):
        """wavesolver.py:232-293: linearised (Born) modelling for the model perturbation `dm` (a Function, or an
        array of the grid's shape). Returns (rec, u0, v0, du, dv, summary)."""
        dt = kwargs.pop('dt', self.dt)
        src = src or self.geometry.src
        rec = rec or self.geometry.rec
        mk = lambda n: TimeFunction(name=n, grid=self.model.grid, time_order=2, space_order=self.space_order)
        u0 = u0 or mk('u0')
        v0 = v0 or mk('v0')
        du = du or mk('du')
        dv = dv or mk('dv')
        model = model or self.model
        kwargs.update(model.physical_params(**kwargs))
        summary = self.op_jac().apply(dm=dm, u0=u0, v0=v0, du=du, dv=dv, src=src, rec=rec, dt=dt, **kwargs)
        return rec, u0, v0, du, dv, summary

    @memoized_meth
    def op_adj(self):
        return AdjointOperator(self.model, self.geometry, space_order=self.space_order, kernel=self.kernel,
                               **self._kwargs)

    @memoized_meth
    def op_jacadj(self, save=True):
        return JacobianAdjOperator(self.model, self.geometry, space_order=self.space_order, save=save,
                                   **self._kwargs)

    def adjoint(self, rec, srca=None, p=None, r=None, model=None, **kwargs):
        """wavesolver.py `adjoint`: adjoint modelling of the receiver data `rec`. Returns (srca, p, r, summary)."""
        srca = srca or self.geometry.new_src(name='srca', src_type=None)
        mk = lambda n: TimeFunction(name=n, grid=self.model.grid, time_order=2, space_order=self.space_order)
        p = p or mk('p')
        r = r or mk('r')
        model = model or self.model
        kwargs.update(model.physical_params(**kwargs))
        summary = self.op_adj().apply(srca=srca, rec=rec, p=p, r=r, dt=kwargs.pop('dt', self.dt), **kwargs)
        return srca, p, r, summary

    def jacobian_adjoint(self, rec, u0, v0, du=None, dv=None, dm=None, model=None, checkpointing=False, **kwargs):
        """wavesolver.py `jacobian_adjoint`: the gradient (Jacobian adjoint applied to `rec`) from the forward
        wavefields u0, v0 saved by `forward(save=True)`. Returns (dm, summary)."""
        if checkpointing:
            raise NotImplementedError("checkpointing needs pyrevolve, which this package does not provide")
        dt = kwargs.pop('dt', self.dt)
        dm = dm or Function(name='dm', grid=self.model.grid)
        mk = lambda n: TimeFunction(name=n, grid=self.model.grid, time_order=2, space_order=self.space_order)
        du = du or mk('du')
        dv = dv or mk('dv')
        model = model or self.model
        kwargs.update(model.physical_params(**kwargs))
        summary = self.op_jacadj().apply(rec=rec, dm=dm, u0=u0, v0=v0, du=du, dv=dv, dt=dt, **kwargs)
        return dm, summary
