"""Host side of `b2_system_forward` (include/b200stencil.h): an explicit linear SYSTEM of updates on a
(staggered) grid described by tap tables — the form the reference's first-order schemes take once their
equations are evaluated: elastic (examples/seismic/elastic/operators.py:26-65), staggered TTI
(examples/seismic/tti/operators.py:280-428) ...

    stage:  out_field[t + out_tshift][p] = sum_k coef_k * C[cfield_k][p] * field_k[t + tshift_k][p + off_k]

`LinearSystem` only marshals; who builds the tables (devito_b200/refplugin.py from the reference's own
evaluated equations) also tabulates the coefficient arrays `C` (averaged material parameters x damping at
the output's staggered position)."""
import ctypes
import time as _time

import numpy as np

from . import _lib as L_
from .exceptions import InvalidArgument

__all__ = ['LinearSystem', 'Stage', 'Tap']


class Tap:
    __slots__ = ('field', 'tshift', 'off', 'coef', 'cfield')

    def __init__(self, field, tshift, off, coef, cfield=-1):
        self.field, self.tshift, self.off, self.coef, self.cfield = int(field), int(tshift), tuple(off), float(coef), int(cfield)


class Stage:
    def __init__(self, out_field, out_tshift, taps, ext=0):
        """ext: the box widened by `ext` cells per side on every space axis (a scratch field that receivers sample
        next to the domain's faces; such a stage may not use coefficient arrays)."""
        self.out_field, self.out_tshift, self.ext = int(out_field), int(out_tshift), int(ext)
        self.taps = sorted(taps, key=lambda t: (t.cfield, t.field, t.tshift, t.off))     # the kernel caches C by run
        if not 1 <= len(self.taps) <= L_.SYS_MAX_TAPS:
            raise InvalidArgument(f"a stage has {len(self.taps)} taps (1..{L_.SYS_MAX_TAPS} supported)")


class LinearSystem:
    def __init__(self, ndim, halo, nfields, stages, injections=(), interpolations=()):
        """injections: (sparse, [field ids], tshift, scale, param_kind, param dataobj | None);
        interpolations: (sparse, field id, tshift)."""
        if nfields > L_.SYS_MAX_FIELDS:
            raise InvalidArgument(f"{nfields} fields (at most {L_.SYS_MAX_FIELDS})")
        self.ndim, self.halo, self.nfields = int(ndim), int(halo), int(nfields)
        self.stages = list(stages)
        self.injections = list(injections)
        self.interpolations = list(interpolations)

    def points_per_step(self, lo, hi):
        return float(np.prod([h - l + 1 for l, h in zip(lo, hi)])) * len(self.stages)

    def apply(self, fields, coefs, lo, hi, time_m, time_M, deviceid=0):
        """fields: list of `_lib.ForeignDataobj` / DataobjHolder (host-staged or resident); coefs: list of float32
        arrays of the grid's shape; injections/interpolations hold `_lib.ForeignSparse`. Returns the timers."""
        L = L_.lib()
        a, timers, hold = self.arguments(fields, coefs, lo, hi, time_m, time_M, deviceid)
        t0 = _time.perf_counter()
        rc = L.b2_system_forward(ctypes.byref(a))
        wall = _time.perf_counter() - t0
        if rc != 0:
            from .exceptions import ExecutionError
            raise ExecutionError(f"b2_system_forward failed with code {rc}: {L.b2_last_error().decode()}")
        return timers, wall

    def arguments(self, fields, coefs, lo, hi, time_m, time_M, deviceid=0):
        """The `struct b2_system_args` of a call, its timers, and what must stay alive while it is in use."""
        nd = self.ndim
        hold = []
        a = L_.SystemArgs()
        a.ndim, a.halo, a.nfields = nd, self.halo, len(fields)
        farr = (ctypes.POINTER(L_.Dataobj) * len(fields))(*[f.ptr for f in fields])
        a.fields = farr
        if len(coefs) > L_.SYS_MAX_COEFS:
            raise InvalidArgument(f"{len(coefs)} coefficient arrays (at most {L_.SYS_MAX_COEFS})")
        # a coefficient array is a float32 ndarray (host-staged by the library) or a ready `struct dataobj` holder
        # (e.g. device-resident: the plugin keeps the tabulated arrays on the GPU across applies)
        cobjs = [c if hasattr(c, 'ptr') else L_.make_dataobj(host=np.ascontiguousarray(c, dtype=np.float32))
                 for c in coefs]
        hold.append(cobjs)
        carr = (ctypes.POINTER(L_.Dataobj) * max(1, len(cobjs)))(*[c.ptr for c in cobjs])
        a.ncoefs, a.coefs = len(cobjs), carr
        st = (L_.SysStage * len(self.stages))()
        for i, s in enumerate(self.stages):
            taps = (L_.SysTap * len(s.taps))()
            for j, t in enumerate(s.taps):
                taps[j].field, taps[j].tshift, taps[j].coef, taps[j].cfield = t.field, t.tshift, t.coef, t.cfield
                for d in range(nd):
                    taps[j].off[d] = int(t.off[d])
            hold.append(taps)
            st[i].out_field, st[i].out_tshift, st[i].ntaps, st[i].taps = s.out_field, s.out_tshift, len(s.taps), taps
            st[i].ext = s.ext
        a.nstages, a.stages = len(self.stages), st

        def sparse(sf):
            s = L_.Sparse()
            s.data, s.gp = sf.data.ptr, sf.gp.ptr
            for i, wo in enumerate(sf.ws):
                s.w[i] = wo.ptr
            s.p_m, s.p_M, s.r = sf.p_m, sf.p_M, sf.r
            hold.append(s)
            return ctypes.pointer(s)
        inj = (L_.SysInject * max(1, len(self.injections)))()
        for i, (sf, fids, tshift, scale, pkind, pobj) in enumerate(self.injections):
            inj[i].s, inj[i].nfields, inj[i].tshift, inj[i].scale = sparse(sf), len(fids), int(tshift), float(scale)
            inj[i].param_kind = int(pkind)
            inj[i].param = pobj.ptr if pobj is not None else None
            for j, f in enumerate(fids):
                inj[i].fields[j] = int(f)
        itp = (L_.SysInterp * max(1, len(self.interpolations)))()
        for i, (sf, fid, tshift) in enumerate(self.interpolations):
            itp[i].s, itp[i].field, itp[i].tshift = sparse(sf), int(fid), int(tshift)
        a.ninject, a.ninterp, a.inject, a.interp = len(self.injections), len(self.interpolations), inj, itp
        lo3, hi3 = list(lo) + [0] * (3 - nd), list(hi) + [0] * (3 - nd)
        a.x_m, a.x_M, a.y_m, a.y_M, a.z_m, a.z_M = lo3[0], hi3[0], lo3[1], hi3[1], lo3[2], hi3[2]
        a.time_m, a.time_M, a.deviceid = int(time_m), int(time_M), int(deviceid)
        timers = L_.Profiler()
        a.timers = ctypes.pointer(timers)
        return a, timers, hold
