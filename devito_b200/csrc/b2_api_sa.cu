// C-ABI entry point b2_sa_forward: the time loop of the reference's generated `IsoFwdOperator` / `IsoAdjOperator`
// (examples/seismic/self_adjoint/operators.py:68-160):
//
//   forward, time = time_m .. time_M:   u[t+1] = iso_stencil(u[t], u[t-1]); u[t+1] += inject(src, dt^2 vp^2/b);
//                                       rec[time] = interpolate(u[t])
//   adjoint, time = time_M .. time_m:   u[t-1] = iso_stencil(u[t], u[t+1]); u[t-1] += inject(rec data, dt^2 vp^2/b);
//                                       srca[time] = interpolate(u[t])
//
// The scale of the injection is the C table the sweep uses, taken at the cell (launch_inject, B2_SCALE_TABLE).
#include "b2_sa.cuh"
#include "b2_sparse.cuh"

using namespace b2;

static int sa_forward_body(const b2_sa_args *a, Staging &st) {
    const int nd = a->ndim;
    const int so = a->space_order;
    int rc = B2_OK;

    if (a->halo) {
        set_error("b2_sa_forward: the self-adjoint update is not combined with halo exchange in this version");
        return B2_ERR_INVALID;
    }
    if (a->free_surface) {
        set_error("b2_sa_forward: the self-adjoint update has no free surface in this version");
        return B2_ERR_INVALID;
    }
    DevArray *u, *b = nullptr, *vp = nullptr, *damp = nullptr;
    SparseDev src, rec;
    if ((rc = st.array(a->u, nd + 1, true, u))) return rc;
    if (a->b && (rc = st.array(a->b, nd, false, b))) return rc;
    if (a->vp && (rc = st.array(a->vp, nd, false, vp))) return rc;
    if (a->damp && (rc = st.array(a->damp, nd, false, damp))) return rc;
    for (DevArray *x : {b, vp, damp})
        if (x)
            for (int d = 0; d < nd; ++d)
                if (x->size[d] != u->size[d + 1]) {
                    set_error("b2_sa_forward: b, vp and damp must have the allocated space layout of u");
                    return B2_ERR_INVALID;
                }
    if ((rc = sparse_stage_in(st, a->src, nd, false, src))) return rc;
    if ((rc = sparse_stage_in(st, a->rec, nd, true, rec))) return rc;
    // devito/operations/interpolators.py:28-37 `check_radius`
    if ((src.present && src.r > so) || (rec.present && rec.r > so)) {
        set_error("b2_sa_forward: sparse radius %d exceeds the halo (space_order %d)",
                  src.present && src.r > so ? src.r : rec.r, so);
        return B2_ERR_INVALID;
    }

    // ---- geometry in the internal 3-dim convention ----
    SaPlan p;
    const int lo_in[3] = {a->x_m, a->y_m, a->z_m};
    const int hi_in[3] = {a->x_M, a->y_M, a->z_M};
    p.tsize = u->size[0];
    p.so = so;
    for (int d = 0; d < 3; ++d) {
        const int di = d - (3 - nd);          // the grid's dim, or < 0 for the dummy leading dim of a 2-D grid
        if (di < 0) {
            p.a[d] = 1; p.n[d] = 1; p.o[d] = 0; p.radius[d] = 0;
            continue;
        }
        p.a[d] = u->size[di + 1];
        p.n[d] = hi_in[di] - lo_in[di] + 1;
        p.o[d] = lo_in[di] + so;
        p.radius[d] = a->radius;
        if (!a->c[di]) { set_error("b2_sa_forward: weights for dim %d missing", di); return B2_ERR_INVALID; }
        for (int i = 0; i < a->radius; ++i) p.c[d][i] = a->c[di][i];
    }
    for (int d = 0; d < 3; ++d) {
        if (p.n[d] <= 0) return B2_OK;
        // the nested stencil reaches 2R-1 points; b is read over [p-R, p+R-1]
        const int rd = p.radius[d] ? 2 * p.radius[d] - 1 : 0;
        if (p.o[d] - rd < 0 || p.o[d] + p.n[d] - 1 + rd >= p.a[d]) {
            set_error("b2_sa_forward: iteration range + radius %d leaves the allocated array (extent %d) on dim %d",
                      rd, p.a[d], d - (3 - nd));
            return B2_ERR_INVALID;
        }
    }
    p.sy = p.a[2];
    p.sx = (long long)p.a[1] * p.a[2];
    p.slot_elems = (size_t)p.a[0] * p.a[1] * p.a[2];
    p.u = (float *)u->d;
    p.b_arr = b ? (const float *)b->d : nullptr;
    p.vp_arr = vp ? (const float *)vp->d : nullptr;
    p.w = damp ? (const float *)damp->d : nullptr;
    p.b_value = a->b_value;
    p.vp_value = a->vp_value;
    p.dt = a->dt;
    p.adjoint = a->adjoint != 0;
    if (!b && !(a->b_value > 0.f)) {
        set_error("b2_sa_forward: scalar buoyancy %g must be positive", (double)a->b_value);
        return B2_ERR_INVALID;
    }
    if ((rc = sa_plan_init(p, a->kernel))) return rc;

    FieldGeom g;
    g.sx = p.sx;
    g.sy = p.sy;
    g.slot_elems = p.slot_elems;
    g.so = so;
    g.ndim = nd;
    for (int d = 0; d < nd; ++d) { g.lo[d] = lo_in[d]; g.hi[d] = hi_in[d]; }

    const int T = p.tsize;
    static cudaEvent_t e0 = nullptr, e1 = nullptr;      // created once (the process is bound to one device)
    if (a->timers) {
        if (!e0 && (cudaEventCreate(&e0) != cudaSuccess || cudaEventCreate(&e1) != cudaSuccess)) {
            e0 = e1 = nullptr;
            set_error("b2_sa_forward: cannot create timing events");
            return B2_ERR_DEVICE;
        }
        cudaEventRecord(e0, stream());
    }
    const bool adj = p.adjoint;
    const int dir = adj ? -1 : 1;
    for (int time = adj ? a->time_M : a->time_m; adj ? time >= a->time_m : time <= a->time_M; time += dir) {
        const int t0 = slot(time, T);
        const int t1 = slot(time + dir, T);     // written
        const int t2 = slot(time - dir, T);     // the other level read
        if ((rc = sa_step(p, t0, t2, t1))) return rc;
        float *f1 = p.u + (size_t)t1 * p.slot_elems;
        if ((rc = launch_inject(src, g, f1, nullptr, time, B2_SCALE_TABLE, p.C, 0.f, 0.f))) return rc;
        if ((rc = launch_interp(rec, g, p.u + (size_t)(a->rec_toff ? t1 : t0) * p.slot_elems, nullptr, time)))
            return rc;
        if (a->errctl && ((time - a->time_m) % 100 == 99 || time == (adj ? a->time_m : a->time_M))) {
            bool bad = false;
            if ((rc = check_finite(f1, p.slot_elems, bad))) return rc;
            if (bad) { set_error("NaN/Inf detected in u at time=%d", time); return B2_ERR_NAN; }
        }
    }
    if (a->timers) cudaEventRecord(e1, stream());
    cudaError_t e = cudaStreamSynchronize(stream());
    if (e != cudaSuccess) {
        set_error("b2_sa_forward: device error: %s", cudaGetErrorString(e));
        return B2_ERR_LAUNCH;
    }
    if (a->timers) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, e0, e1);
        a->timers->section0 += ms * 1e-3;
    }
    return B2_OK;
}

extern "C" int b2_sa_forward(const struct b2_sa_args *a) {
    if (!a || !a->u) { set_error("b2_sa_forward: NULL args"); return B2_ERR_INVALID; }
    if (a->ndim != 2 && a->ndim != 3) { set_error("b2_sa_forward: ndim must be 2 or 3"); return B2_ERR_INVALID; }
    if (a->radius < 1 || a->radius > B2_MAX_RADIUS || 2 * a->radius > a->space_order) {
        set_error("b2_sa_forward: unsupported radius %d (space_order %d)", a->radius, a->space_order);
        return B2_ERR_INVALID;
    }
    if (a->time_M < a->time_m) return B2_OK;
    std::lock_guard<std::mutex> api_lock(api_mutex());
    if (int rc0 = use_device(a->deviceid)) return rc0;
    note_sweep_kernel("");
    Staging st;
    return st.finish(sa_forward_body(a, st));
}
