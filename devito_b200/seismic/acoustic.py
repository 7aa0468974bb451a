"""Isotropic acoustic modelling (mirror of examples/seismic/acoustic/operators.py:50-187 and
wavesolver.py:11-156): forward and adjoint operators (gradient/Born are SURVEY §8f)."""
import ctypes
import time as _time
from types import SimpleNamespace

import numpy as np

from .. import Eq, FreeSurface, Inc, Function, Operator, TimeFunction, solve, InvalidArgument
from .. import _lib as L_
from ..revolve import schedule, default_n_checkpoints
from ..tools import memoized_meth

__all__ = ['laplacian', 'iso_stencil', 'ForwardOperator', 'AdjointOperator', 'GradientOperator',
           'BornOperator', 'AcousticWaveSolver']


def laplacian(field, model, kernel):
    """Spatial operator (operators.py:50-68): for the 4th-order-in-time scheme the 4th time derivative
    is traded for a double Laplacian, H = laplace + s**2/12 * laplace(1/m * laplace)."""
    if kernel not in ('OT2', 'OT4'):
        raise ValueError("Unrecognized kernel")
    s = model.grid.time_dim.spacing
    biharmonic = field.biharmonic(1 / model.m) if kernel == 'OT4' else 0
    return field.laplace + s ** 2 / 12 * biharmonic


def iso_stencil(field, model, kernel='OT2', **kwargs):
    """u.dt2 * m - H(u) + damp * u.dt = 0 solved for u.forward (operators.py:71-107)."""
    forward = kwargs.get('forward', True)
    unext = field.forward if forward else field.backward
    udt = field.dt if forward else field.dt.T
    lap = laplacian(field, model, kernel)
    eq_time = solve(model.m * field.dt2 - lap - kwargs.get('q', 0) + model.damp * udt, unext)
    update = Eq(unext, eq_time, subdomain=model.grid.subdomains['physdomain'])
    if model.fs:
        # operators.py:105-106 `freesurface(model, Eq(unext, eq_time))`: the top rows get the same
        # update with vertical taps mirrored about the surface, and the surface row is cleared
        return [update, FreeSurface(update, model.grid.subdomains['fsdomain'])]
    return [update]


def ForwardOperator(model, geometry, space_order=4, save=False, kernel='OT2', **kwargs):
    """operators.py:113-150"""
    m = model.m
    u = TimeFunction(name='u', grid=model.grid, save=geometry.nt if save else None, time_order=2,
                     space_order=space_order)
    src, rec = geometry.src, geometry.rec
    s = model.grid.stepping_dim.spacing
    eqn = iso_stencil(u, model, kernel)
    src_term = src.inject(field=u.forward, expr=src * s ** 2 / m)
    rec_term = rec.interpolate(expr=u)
    return Operator(eqn + src_term + rec_term, subs=model.spacing_map, name='Forward', **kwargs)


def AdjointOperator(model, geometry, space_order=4, kernel='OT2', save=None, **kwargs):
    """operators.py:153-187: the update solved for v.backward, receivers injected, adjoint source
    sampled at the source position."""
    m = model.m
    v = TimeFunction(name='v', grid=model.grid, save=None, time_order=2, space_order=space_order)
    srca = geometry.new_src(name='srca', src_type=None)
    rec = geometry.rec
    s = model.grid.stepping_dim.spacing
    eqn = iso_stencil(v, model, kernel, forward=False)
    receivers = rec.inject(field=v.backward, expr=rec * s ** 2 / m)
    source_a = srca.interpolate(expr=v)
    return Operator(eqn + receivers + source_a, subs=model.spacing_map, name='Adjoint', **kwargs)


def GradientOperator(model, geometry, space_order=4, save=True, kernel='OT2', **kwargs):
    """operators.py:190-232: adjoint propagation of the data + imaging condition grad -= u * v.dt2."""
    if kernel != 'OT2':
        raise NotImplementedError("the OT4 imaging condition (extra biharmonic term, operators.py:225-226) "
                                  "is not on this backend's path yet")
    m = model.m
    grad = Function(name='grad', grid=model.grid)
    u = TimeFunction(name='u', grid=model.grid, save=geometry.nt if save else None, time_order=2,
                     space_order=space_order)
    v = TimeFunction(name='v', grid=model.grid, save=None, time_order=2, space_order=space_order)
    rec = geometry.rec
    s = model.grid.stepping_dim.spacing
    eqn = iso_stencil(v, model, kernel, forward=False)
    gradient_update = Inc(grad, -u * v.dt2)
    receivers = rec.inject(field=v.backward, expr=rec * s ** 2 / m)
    return Operator(eqn + receivers + [gradient_update], subs=model.spacing_map, name='Gradient', **kwargs)


def BornOperator(model, geometry, space_order=4, kernel='OT2', **kwargs):
    """operators.py:235-277: background field u driven by the source, linearised field U driven by
    `-dm * u.dt2`, receivers sampling U."""
    kwargs.pop('save', None)
    m = model.m
    src, rec = geometry.src, geometry.rec
    u = TimeFunction(name='u', grid=model.grid, save=None, time_order=2, space_order=space_order)
    U = TimeFunction(name='U', grid=model.grid, save=None, time_order=2, space_order=space_order)
    dm = Function(name='dm', grid=model.grid, space_order=0)
    s = model.grid.stepping_dim.spacing
    eqn1 = iso_stencil(u, model, kernel)
    eqn2 = iso_stencil(U, model, kernel, q=-dm * u.dt2)
    source = src.inject(field=u.forward, expr=src * s ** 2 / m)
    receivers = rec.interpolate(expr=U)
    return Operator(eqn1 + source + eqn2 + receivers, subs=model.spacing_map, name='Born', **kwargs)


class AcousticWaveSolver:
    """wavesolver.py:11-230: forward, adjoint, Born (`jacobian`) and gradient (`jacobian_adjoint`, with or without
    checkpointing)."""

    def __init__(self, model, geometry, kernel='OT2', space_order=4, **kwargs):
        self.model = model
        self.model._initialize_bcs(bcs="damp")
        self.geometry = geometry
        self.space_order = space_order
        self.kernel = kernel
        self._kwargs = kwargs

    @property
    def dt(self):
        # the 4th-order scheme is stable with a sqrt(3) = 1.73 larger step (wavesolver.py:39-44)
        if self.kernel == 'OT4':
            return self.model.dtype(1.73 * self.model.critical_dt)
        return self.model.critical_dt

    @memoized_meth
    def op_fwd(self, save=None):
        return ForwardOperator(self.model, save=save, geometry=self.geometry, kernel=self.kernel,
                               space_order=self.space_order, **self._kwargs)

    @memoized_meth
    def op_adj(self):
        return AdjointOperator(self.model, save=None, geometry=self.geometry, kernel=self.kernel,
                               space_order=self.space_order, **self._kwargs)

    def adjoint(self, rec, srca=None, v=None, model=None, **kwargs):
        """wavesolver.py:118-156"""
        srca = srca or self.geometry.new_src(name='srca', src_type=None)
        v = v or TimeFunction(name='v', grid=self.model.grid, time_order=2, space_order=self.space_order)
        model = model or self.model
        kwargs.update(model.physical_params(**kwargs))
        summary = self.op_adj().apply(srca=srca, rec=rec, v=v, dt=kwargs.pop('dt', self.dt), **kwargs)
        return srca, v, summary

    @memoized_meth
    def op_grad(self, save=True):
        return GradientOperator(self.model, save=save, geometry=self.geometry, kernel=self.kernel,
                                space_order=self.space_order, **self._kwargs)

    def jacobian_adjoint(self, rec, u=None, src=None, v=None, grad=None, model=None, checkpointing=False,
                         n_checkpoints=None, **kwargs):
        """wavesolver.py:158-230: gradient of the data misfit w.r.t. m. Without `checkpointing`, `u` is the saved
        forward wavefield (`forward(save=True)`). With it, `u` is not needed: one library call recomputes the forward
        field from `n_checkpoints` device checkpoints of two wavefield slots each (binomial checkpointing,
        devito_b200/revolve.py) while it runs the adjoint; `src` drives the forward run (default: the geometry's).
        `n_checkpoints=None` takes as many as fit in 90 % of the free device memory, at most one per time step."""
        if checkpointing:
            return self._jacobian_adjoint_revolve(rec, src=src, v=v, grad=grad, model=model,
                                                  n_checkpoints=n_checkpoints, **kwargs)
        if u is None:
            raise TypeError("jacobian_adjoint() needs the saved forward wavefield `u` (forward(save=True)) unless "
                            "checkpointing=True")
        dt = kwargs.pop('dt', self.dt)
        grad = grad or Function(name='grad', grid=self.model.grid)
        v = v or TimeFunction(name='v', grid=self.model.grid, time_order=2, space_order=self.space_order)
        model = model or self.model
        kwargs.update(model.physical_params(**kwargs))
        summary = self.op_grad().apply(rec=rec, grad=grad, v=v, u=u, dt=dt, **kwargs)
        return grad, summary

    def _revolve_setup(self, rec, src=None, v=None, grad=None, model=None, n_checkpoints=None, **kwargs):
        """The two argument blocks of b2_iso_gradient_revolve (the forward operator's and the Gradient operator's,
        marshalled like their applies; the Gradient's usave, damp and parameter point at the forward block's arrays)
        and its action list. Refuses what the entry point does not run before touching the device."""
        if n_checkpoints is not None and int(n_checkpoints) < 1:
            raise ValueError(f"n_checkpoints must be at least 1, got {n_checkpoints}")
        op_g = self.op_grad(save=True)          # OT4: the Gradient operator's NotImplementedError
        if self.model.grid.distributor.is_parallel:
            raise InvalidArgument("the checkpointed gradient does not run on a decomposed grid in this version")
        op_f = self.op_fwd(save=False)
        for op in (op_f, op_g):
            if op.backend != 'cuda-sm90a':
                raise InvalidArgument(f"operator `{op.name}` is not on the CUDA path: {op._why_not}")
        dt = kwargs.pop('dt', self.dt)
        u = TimeFunction(name='u', grid=self.model.grid, time_order=2, space_order=self.space_order)
        grad = grad or Function(name='grad', grid=self.model.grid)
        v = v or TimeFunction(name='v', grid=self.model.grid, time_order=2, space_order=self.space_order)
        model = model or self.model
        kwargs.update(model.physical_params(**kwargs))
        hold = []
        af, args_f, dev, post_f = op_f._marshal_wave(dict(kwargs, src=src or self.geometry.src, u=u, dt=dt), hold)
        ag, args_g, _, post_g = op_g._marshal_wave(dict(kwargs, rec=rec, v=v, grad=grad, dt=dt), hold,
                                                   omit=('usave',))
        af.rec = None                           # the forward run records nothing
        ag.usave, ag.damp, ag.param = af.u, af.damp, af.param
        # schedule step i <-> forward state at time tf + i (levels tf + i, tf + i - 1) and adjoint time tg + i
        tf, tg = args_f['time_m'], args_g['time_m']
        nsteps = args_g['time_M'] - tg + 1
        if tf - tg not in (0, 1):
            raise InvalidArgument(f"the forward loop starts at time {tf}, the adjoint one at {tg}: the adjoint step at "
                                  "time t needs u[t] among the two levels of forward state t")
        if n_checkpoints is None and nsteps < 1:
            n_checkpoints = 1                   # nothing to reverse: the call returns without device work
        if n_checkpoints is None:
            import torch
            free = torch.cuda.mem_get_info(dev)[0]
            # what the call itself copies in (host-staged arrays) is not free for checkpoints
            free -= sum(o.contents.nbytes for o in (af.u, af.damp, af.param, ag.u, ag.grad)
                        if o and not o.contents.dmap)
            slot = int(np.prod(u.storage.shape[1:])) * np.dtype(np.float32).itemsize
            n_checkpoints = default_n_checkpoints(nsteps, free, slot)
            if n_checkpoints < 1:
                raise InvalidArgument("no device memory is left for a checkpoint (two wavefield slots)")
        n_checkpoints = int(n_checkpoints)
        sched = schedule(nsteps, n_checkpoints)
        flat = []
        for act in sched:
            kind = L_.REVOLVE_ACTIONS[act[0]]
            if act[0] == 'advance':
                flat += [kind, tf + act[1], tf + act[2]]
            elif act[0] == 'takeshot':
                flat += [kind, act[1], tf + act[2]]
            elif act[0] == 'restore':
                flat += [kind, act[1], 0]
            else:
                flat += [kind, tg + act[1], 0]
        actions = (ctypes.c_int * max(len(flat), 1))(*flat)
        return SimpleNamespace(op=op_g, fwd=af, grad=ag, args=args_g, dev=dev, post=post_f + args_f['post'] + post_g + args_g['post'],
                               actions=actions, nactions=len(sched), n_checkpoints=n_checkpoints, schedule=sched,
                               nsteps=nsteps, hold=hold, grad_fn=grad)

    def _jacobian_adjoint_revolve(self, rec, **kwargs):
        return self._revolve_run(self._revolve_setup(rec, **kwargs))

    def _revolve_run(self, c):
        """One call of b2_iso_gradient_revolve with what `_revolve_setup` built: (grad, summary)."""
        L = L_.lib()
        c.fwd.deviceid = c.grad.deviceid = c.dev
        timers = L_.Profiler()
        c.grad.timers = ctypes.pointer(timers)
        t0 = _time.perf_counter()
        rc = L.b2_iso_gradient_revolve(ctypes.byref(c.fwd), ctypes.byref(c.grad), c.actions, c.nactions,
                                       c.n_checkpoints)
        t_wall = _time.perf_counter() - t0
        for fn in c.post:
            fn()
        summary = c.op._finish(rc, L, timers, c.args, t_wall)
        return c.grad_fn, summary

    jacobian_adjoint.__name__ = 'jacobian_adjoint'
    gradient = jacobian_adjoint

    @memoized_meth
    def op_born(self):
        return BornOperator(self.model, save=None, geometry=self.geometry, kernel=self.kernel,
                            space_order=self.space_order, **self._kwargs)

    def jacobian(self, dmin, src=None, rec=None, u=None, U=None, model=None, **kwargs):
        """wavesolver.py:216-254: linearised (Born) modelling for the model perturbation `dmin`
        (a Function, or an array of the grid's shape)."""
        src = src or self.geometry.src
        rec = rec or self.geometry.rec
        mk = lambda n: TimeFunction(name=n, grid=self.model.grid, time_order=2, space_order=self.space_order)
        u = u or mk('u')
        U = U or mk('U')
        model = model or self.model
        kwargs.update(model.physical_params(**kwargs))
        summary = self.op_born().apply(dm=dmin, u=u, U=U, src=src, rec=rec, dt=kwargs.pop('dt', self.dt),
                                       **kwargs)
        return rec, u, U, summary

    born = jacobian

    def forward(self, src=None, rec=None, u=None, model=None, save=None, **kwargs):
        src = src or self.geometry.src
        rec = rec or self.geometry.rec
        u = u or TimeFunction(name='u', grid=self.model.grid, save=self.geometry.nt if save else None,
                              time_order=2, space_order=self.space_order)
        model = model or self.model
        kwargs.update(model.physical_params(**kwargs))
        summary = self.op_fwd(save).apply(src=src, rec=rec, u=u, dt=kwargs.pop('dt', self.dt), **kwargs)
        return rec, u, summary
