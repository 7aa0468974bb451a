// C-ABI entry points of the updates that apply the nested operator L (b2_nested.cuh):
//
// b2_sa_forward, the time loop of the reference's generated self-adjoint `IsoFwdOperator` / `IsoAdjOperator`
// (examples/seismic/self_adjoint/operators.py:68-160):
//
//   forward, time = time_m .. time_M:   u[t+1] = iso_stencil(u[t], u[t-1]); u[t+1] += inject(src, dt^2 vp^2/b);
//                                       rec[time] = interpolate(u[t])
//   adjoint, time = time_M .. time_m:   u[t-1] = iso_stencil(u[t], u[t+1]); u[t-1] += inject(rec data, dt^2 vp^2/b);
//                                       srca[time] = interpolate(u[t])
//
// The scale of the injection is the C table the sweep uses, taken at the cell (launch_inject, B2_SCALE_TABLE).
//
// b2_visco_forward, the time loop of the reference's generated SLS `ForwardOperator` / `AdjointOperator` at
// time_order=2 (examples/seismic/viscoacoustic/operators.py:124-192, :482-569):
//
//   forward, time = time_m .. time_M:   r[t+1], p[t+1] = sls(p[t], p[t-1], r[t], r[t-1]);
//                                       p[t+1] += inject(src, dt^2 vp^2); rec[time] = interpolate(p[t])
//   adjoint, time = time_M .. time_m:   r[t-1], s = mix(p[t], r[t], r[t+1]); p[t-1] = sls_adj(s, p[t], p[t+1]);
//                                       p[t-1] += inject(rec data, dt^2 vp^2); srca[time] = interpolate(p[t])
//
// Both run in nested_entry and start with nested_prologue: the argument checks, the staging of the wavefield u (p), b,
// vp, damp and the sparse pair, the box, the weights and the reach. Each then stages and checks its own operands and
// runs its own time loop, whose injection scale and errctl fields differ.
#include "b2_sa.cuh"
#include "b2_visco.cuh"
#include "b2_sparse.cuh"

using namespace b2;

// x is null (a scalar) or has the allocated space layout of the wavefield u
static bool same_space(const DevArray *x, const DevArray *u, int nd) {
    for (int d = 0; x && d < nd; ++d)
        if (x->size[d] != u->size[d + 1]) return false;
    return true;
}

// The part of an entry point that b2_sa_args and b2_visco_args (A) share: refuses halo exchange and a free surface,
// stages u (written), b, vp and damp, which must have u's space layout, and the sparse pair, and sets p's box, radius,
// weights, dt, direction and b, vp. The nested stencil reaches 2R-1 points (b is read over [p-R, p+R-1]): a box that
// this reach takes out of the allocation is refused; an empty box sets `empty` and returns before the check that a
// scalar b is positive.
template <class A>
static int nested_prologue(const char *who, const A *a, Staging &st, NestedPlan &p, DevArray *&u, DevArray *&damp,
                           SparseDev &src, SparseDev &rec, bool &empty) {
    const int nd = a->ndim;
    const int so = a->space_order;
    int rc;
    if (a->halo) {
        set_error("%s: this update is not combined with halo exchange in this version", who);
        return B2_ERR_INVALID;
    }
    if (a->free_surface) {
        set_error("%s: this update has no free surface in this version", who);
        return B2_ERR_INVALID;
    }
    DevArray *b = nullptr, *vp = nullptr;
    damp = nullptr;
    if ((rc = st.array(a->u, nd + 1, true, u))) return rc;
    if (a->b && (rc = st.array(a->b, nd, false, b))) return rc;
    if (a->vp && (rc = st.array(a->vp, nd, false, vp))) return rc;
    if (a->damp && (rc = st.array(a->damp, nd, false, damp))) return rc;
    if (!same_space(b, u, nd) || !same_space(vp, u, nd) || !same_space(damp, u, nd)) {
        set_error("%s: b, vp and damp must have the allocated space layout of the wavefield", who);
        return B2_ERR_INVALID;
    }
    if ((rc = sparse_stage_pair(who, st, a->src, a->rec, nd, so, src, rec))) return rc;

    static_cast<Box &>(p) = make_box(a, nd, u->size, so);
    for (int di = 0; di < nd; ++di) {
        const int d = 3 - nd + di;
        p.radius[d] = a->radius;
        if (!a->c[di]) { set_error("%s: weights for dim %d missing", who, di); return B2_ERR_INVALID; }
        for (int i = 0; i < a->radius; ++i) p.c[d][i] = a->c[di][i];
    }
    if ((rc = check_reach(who, p, nd, 2 * a->radius - 1, empty)) || empty) return rc;
    if (!b && !(a->b_value > 0.f)) {
        set_error("%s: scalar buoyancy %g must be positive", who, (double)a->b_value);
        return B2_ERR_INVALID;
    }
    p.b_arr = b ? (const float *)b->d : nullptr;
    p.vp_arr = vp ? (const float *)vp->d : nullptr;
    p.b_value = a->b_value;
    p.vp_value = a->vp_value;
    p.dt = a->dt;
    p.adjoint = a->adjoint != 0;
    return B2_OK;
}

// The C entry point around `body`: the checks that need no device, the API lock, the device, and one staging scope
// that releases every staged array on return.
template <class A>
static int nested_entry(const char *who, const A *a, int (*body)(const A *, Staging &)) {
    if (!a || !a->u) { set_error("%s: NULL args", who); return B2_ERR_INVALID; }
    if (a->ndim != 2 && a->ndim != 3) { set_error("%s: ndim must be 2 or 3", who); return B2_ERR_INVALID; }
    if (a->radius < 1 || a->radius > B2_MAX_RADIUS || 2 * a->radius > a->space_order) {
        set_error("%s: unsupported radius %d (space_order %d)", who, a->radius, a->space_order);
        return B2_ERR_INVALID;
    }
    if (a->time_M < a->time_m) return B2_OK;
    std::lock_guard<std::mutex> api_lock(api_mutex());
    if (int rc0 = use_device(a->deviceid)) return rc0;
    note_sweep_kernel("");
    Staging st;
    return st.finish(body(a, st));
}

static int sa_forward_body(const b2_sa_args *a, Staging &st) {
    SaPlan p;
    DevArray *u, *damp;
    SparseDev src, rec;
    bool empty;
    int rc;
    if ((rc = nested_prologue("b2_sa_forward", a, st, p, u, damp, src, rec, empty)) || empty) return rc;
    p.u = (float *)u->d;
    p.w = damp ? (const float *)damp->d : nullptr;
    if ((rc = sa_plan_init(p, a->kernel))) return rc;

    const FieldGeom g = field_geom(p, a->ndim);
    const int T = p.tsize;
    if ((rc = loop_timer_start(a->timers))) return rc;
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
        if (a->errctl && errctl_due(time, a->time_m, adj ? a->time_m : a->time_M) &&
            (rc = check_finite(f1, p.slot_elems, "u", time)))
            return rc;
    }
    return loop_finish("b2_sa_forward", a->timers);
}

static int visco_forward_body(const b2_visco_args *a, Staging &st) {
    const int nd = a->ndim;
    ViscoPlan p;
    DevArray *u, *damp, *r, *qp = nullptr;
    SparseDev src, rec;
    bool empty;
    int rc;
    if ((rc = nested_prologue("b2_visco_forward", a, st, p, u, damp, src, rec, empty))) return rc;
    if (!a->r) { set_error("b2_visco_forward: the memory variable r is missing"); return B2_ERR_INVALID; }
    if ((rc = st.array(a->r, nd + 1, true, r))) return rc;
    for (int d = 0; d <= nd; ++d)
        if (r->size[d] != u->size[d]) {
            set_error("b2_visco_forward: r must have the allocated layout and time slots of p");
            return B2_ERR_INVALID;
        }
    if (a->qp && (rc = st.array(a->qp, nd, false, qp))) return rc;
    if (!same_space(qp, u, nd)) {
        set_error("b2_visco_forward: qp must have the allocated space layout of the wavefield");
        return B2_ERR_INVALID;
    }
    if (empty) return B2_OK;
    if (!(a->f0 > 0.f) || !(a->dt > 0.f)) {
        set_error("b2_visco_forward: f0 (%g) and dt (%g) must be positive", (double)a->f0, (double)a->dt);
        return B2_ERR_INVALID;
    }
    p.p = (float *)u->d;
    p.r = (float *)r->d;
    p.qp_arr = qp ? (const float *)qp->d : nullptr;
    p.damp = damp ? (const float *)damp->d : nullptr;
    p.qp_value = a->qp_value;
    p.f0 = a->f0;
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

extern "C" int b2_sa_forward(const struct b2_sa_args *a) { return nested_entry("b2_sa_forward", a, sa_forward_body); }

extern "C" int b2_visco_forward(const struct b2_visco_args *a) {
    return nested_entry("b2_visco_forward", a, visco_forward_body);
}
