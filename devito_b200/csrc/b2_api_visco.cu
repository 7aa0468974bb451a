// C-ABI entry point b2_visco_forward: the time loop of the reference's generated SLS `ForwardOperator` /
// `AdjointOperator` at time_order=2 (examples/seismic/viscoacoustic/operators.py:124-192, :482-569):
//
//   forward, time = time_m .. time_M:   r[t+1], p[t+1] = sls(p[t], p[t-1], r[t], r[t-1]);
//                                       p[t+1] += inject(src, dt^2 vp^2); rec[time] = interpolate(p[t])
//   adjoint, time = time_M .. time_m:   r[t-1], s = mix(p[t], r[t], r[t+1]); p[t-1] = sls_adj(s, p[t], p[t+1]);
//                                       p[t-1] += inject(rec data, dt^2 vp^2); srca[time] = interpolate(p[t])
#include "b2_visco.cuh"
#include "b2_sparse.cuh"

using namespace b2;

static int visco_forward_body(const b2_visco_args *a, Staging &st) {
    const int nd = a->ndim;
    const int so = a->space_order;
    int rc = B2_OK;

    if (a->halo) {
        set_error("b2_visco_forward: the viscoacoustic update is not combined with halo exchange in this version");
        return B2_ERR_INVALID;
    }
    if (a->free_surface) {
        set_error("b2_visco_forward: the viscoacoustic update has no free surface in this version");
        return B2_ERR_INVALID;
    }
    DevArray *u, *r, *b = nullptr, *vp = nullptr, *qp = nullptr, *damp = nullptr;
    SparseDev src, rec;
    if ((rc = st.array(a->u, nd + 1, true, u))) return rc;
    if (!a->r) { set_error("b2_visco_forward: the memory variable r is missing"); return B2_ERR_INVALID; }
    if ((rc = st.array(a->r, nd + 1, true, r))) return rc;
    for (int d = 0; d <= nd; ++d)
        if (r->size[d] != u->size[d]) {
            set_error("b2_visco_forward: r must have the allocated layout and time slots of p");
            return B2_ERR_INVALID;
        }
    if (a->b && (rc = st.array(a->b, nd, false, b))) return rc;
    if (a->vp && (rc = st.array(a->vp, nd, false, vp))) return rc;
    if (a->qp && (rc = st.array(a->qp, nd, false, qp))) return rc;
    if (a->damp && (rc = st.array(a->damp, nd, false, damp))) return rc;
    for (DevArray *x : {b, vp, qp, damp})
        if (x)
            for (int d = 0; d < nd; ++d)
                if (x->size[d] != u->size[d + 1]) {
                    set_error("b2_visco_forward: b, vp, qp and damp must have the allocated space layout of p");
                    return B2_ERR_INVALID;
                }
    if ((rc = sparse_stage_pair("b2_visco_forward", st, a->src, a->rec, nd, so, src, rec))) return rc;

    ViscoPlan p;
    static_cast<Box &>(p) = make_box(a, nd, u->size, so);
    for (int di = 0; di < nd; ++di) {
        const int d = 3 - nd + di;
        p.radius[d] = a->radius;
        if (!a->c[di]) { set_error("b2_visco_forward: weights for dim %d missing", di); return B2_ERR_INVALID; }
        for (int i = 0; i < a->radius; ++i) p.c[d][i] = a->c[di][i];
    }
    // the nested stencil reaches 2R-1 points; b is read over [p-R, p+R-1]
    bool empty;
    if ((rc = check_reach("b2_visco_forward", p, nd, 2 * a->radius - 1, empty)) || empty) return rc;
    if (!b && !(a->b_value > 0.f)) {
        set_error("b2_visco_forward: scalar buoyancy %g must be positive", (double)a->b_value);
        return B2_ERR_INVALID;
    }
    if (!(a->f0 > 0.f) || !(a->dt > 0.f)) {
        set_error("b2_visco_forward: f0 (%g) and dt (%g) must be positive", (double)a->f0, (double)a->dt);
        return B2_ERR_INVALID;
    }
    p.p = (float *)u->d;
    p.r = (float *)r->d;
    p.b_arr = b ? (const float *)b->d : nullptr;
    p.vp_arr = vp ? (const float *)vp->d : nullptr;
    p.qp_arr = qp ? (const float *)qp->d : nullptr;
    p.damp = damp ? (const float *)damp->d : nullptr;
    p.b_value = a->b_value;
    p.vp_value = a->vp_value;
    p.qp_value = a->qp_value;
    p.dt = a->dt;
    p.f0 = a->f0;
    p.adjoint = a->adjoint != 0;
    if ((rc = visco_plan_init(p, a->kernel))) return rc;

    const FieldGeom g = field_geom(p, nd);
    const int T = p.tsize;
    const float dt2 = p.dt * p.dt;
    const int pk = p.vp_arr ? B2_PARAM_VP : B2_PARAM_SCALAR;
    const float sscale = dt2 * p.vp_value * p.vp_value;
    if ((rc = loop_timer_start(a->timers))) return rc;
    const bool adj = p.adjoint;
    const int dir = adj ? -1 : 1;
    for (int time = adj ? a->time_M : a->time_m; adj ? time >= a->time_m : time <= a->time_M; time += dir) {
        const int t0 = slot(time, T);
        const int t1 = slot(time + dir, T);     // written
        const int t2 = slot(time - dir, T);     // the other level read
        if ((rc = visco_step(p, t0, t2, t1))) return rc;
        float *f1 = p.p + (size_t)t1 * p.slot_elems;
        if ((rc = launch_inject(src, g, f1, nullptr, time, pk, p.vp_arr, sscale, dt2))) return rc;
        if ((rc = launch_interp(rec, g, p.p + (size_t)(a->rec_toff ? t1 : t0) * p.slot_elems, nullptr, time)))
            return rc;
        if (a->errctl && errctl_due(time, a->time_m, adj ? a->time_m : a->time_M) &&
            ((rc = check_finite(f1, p.slot_elems, "p", time)) ||
             (rc = check_finite(p.r + (size_t)t1 * p.slot_elems, p.slot_elems, "r", time))))
            return rc;
    }
    return loop_finish("b2_visco_forward", a->timers);
}

extern "C" int b2_visco_forward(const struct b2_visco_args *a) {
    if (!a || !a->u) { set_error("b2_visco_forward: NULL args"); return B2_ERR_INVALID; }
    if (a->ndim != 2 && a->ndim != 3) { set_error("b2_visco_forward: ndim must be 2 or 3"); return B2_ERR_INVALID; }
    if (a->radius < 1 || a->radius > B2_MAX_RADIUS || 2 * a->radius > a->space_order) {
        set_error("b2_visco_forward: unsupported radius %d (space_order %d)", a->radius, a->space_order);
        return B2_ERR_INVALID;
    }
    if (a->time_M < a->time_m) return B2_OK;
    std::lock_guard<std::mutex> api_lock(api_mutex());
    if (int rc0 = use_device(a->deviceid)) return rc0;
    note_sweep_kernel("");
    Staging st;
    return st.finish(visco_forward_body(a, st));
}
