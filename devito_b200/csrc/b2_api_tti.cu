// C-ABI entry point b2_tti_forward: time loop of the reference's generated `ForwardTTI`
// (examples/seismic/tti/operators.py:431-480): coupled u, v update, injection of the same
// source into both fields (:475-476), receivers sample u+v (:477); halo exchange of both
// fields in one call (tests/test_mpi.py:3690-3694). With born_du / born_dv / born_dm the loop is that of the
// reference's `BornTTI` (tti/operators.py:532-586): the background pair is stepped and the source injected into it,
// then the linearised pair is stepped with the same sweep and driven by -dm * u0.dt2 / -dm * v0.dt2, and the
// receivers sample du + dv. With `adjoint` the loop is that of the reference's `AdjointTTI` (time reversed, the
// mixes e2 p + sd r / sd p + r formed by k_tti_adj_mix and swept with the forward kernels' adjoint variants), and
// with grad / usave / vsave that of `GradientTTI` (the imaging condition after each step and its injection).
#include "b2_tti.cuh"
#include "b2_sparse.cuh"
#include "b2_halo.cuh"

using namespace b2;

static int tti_forward_body(const b2_tti_args *a, Staging &st) {
    const int so = a->space_order;
    const int nd = a->ndim == 2 ? 2 : 3;
    int rc = B2_OK;
    if (nd == 2 && (a->phi != 0.f || a->phi_arr || a->halo)) {
        set_error("b2_tti_forward: a 2-D call takes no azimuth (phi = 0, phi_arr NULL) and no halo exchange");
        return B2_ERR_INVALID;
    }

    DevArray *u, *v, *damp = nullptr, *parr[5] = {}, *bdu = nullptr, *bdv = nullptr, *bdm = nullptr, *grad = nullptr,
             *usave = nullptr, *vsave = nullptr;
    SparseDev src, rec;
    TtiPlan p, pd, pa;

    if ((rc = st.array(a->u, nd + 1, true, u))) return rc;
    if ((rc = st.array(a->v, nd + 1, true, v))) return rc;
    if (a->damp && (rc = st.array(a->damp, nd, false, damp))) return rc;
    {
        const b2_dataobj *pa[5] = {a->vp_arr, a->epsilon_arr, a->delta_arr, a->theta_arr, a->phi_arr};
        for (int i = 0; i < 5; ++i)
            if (pa[i] && (rc = st.array(pa[i], nd, false, parr[i]))) return rc;
    }
    const bool born = a->born_du || a->born_dv || a->born_dm;
    int dmh = 0;
    if (born) {
        if (!a->born_du || !a->born_dv || !a->born_dm) {
            set_error("b2_tti_forward: Born modelling needs born_du, born_dv and born_dm together");
            return B2_ERR_INVALID;
        }
        if (a->halo) {
            set_error("b2_tti_forward: Born modelling is not combined with halo exchange in this version");
            return B2_ERR_INVALID;
        }
        if ((rc = st.array(a->born_du, nd + 1, true, bdu))) return rc;
        if ((rc = st.array(a->born_dv, nd + 1, true, bdv))) return rc;
        if ((rc = st.array(a->born_dm, nd, false, bdm))) return rc;
        for (int d = 0; d <= nd; ++d)
            if (bdu->size[d] != u->size[d] || bdv->size[d] != u->size[d]) {
                set_error("b2_tti_forward: born_du and born_dv must have the layout of u");
                return B2_ERR_INVALID;
            }
        if ((dmh = grid_halo("b2_tti_forward", "born_dm", a->born_dm, *bdm, 0, *u, nd, so)) < 0) return B2_ERR_INVALID;
    }
    const bool adj = a->adjoint != 0;
    int gh = 0;
    if (adj && a->halo) {
        set_error("b2_tti_forward: the adjoint is not combined with halo exchange in this version");
        return B2_ERR_INVALID;
    }
    if (adj && born) {
        set_error("b2_tti_forward: the adjoint is not combined with Born modelling");
        return B2_ERR_INVALID;
    }
    if (a->grad || a->usave || a->vsave) {
        if (!a->grad || !a->usave || !a->vsave) {
            set_error("b2_tti_forward: the imaging condition needs grad, usave and vsave together");
            return B2_ERR_INVALID;
        }
        if (!adj) {
            set_error("b2_tti_forward: the imaging condition runs with the adjoint only");
            return B2_ERR_INVALID;
        }
        if ((rc = st.array(a->grad, nd, true, grad))) return rc;
        if ((rc = st.array(a->usave, nd + 1, false, usave))) return rc;
        if ((rc = st.array(a->vsave, nd + 1, false, vsave))) return rc;
        if (grid_halo("b2_tti_forward", "usave", a->usave, *usave, 1, *u, nd, so, so) < 0 ||
            grid_halo("b2_tti_forward", "vsave", a->vsave, *vsave, 1, *u, nd, so, so) < 0 ||
            (gh = grid_halo("b2_tti_forward", "grad", a->grad, *grad, 0, *u, nd, so)) < 0)
            return B2_ERR_INVALID;
    }
    if ((rc = sparse_stage_pair("b2_tti_forward", st, a->src, a->rec, nd, so, src, rec))) return rc;

    static_cast<Box &>(p) = make_box(a, nd, u->size, so);
    bool empty;
    if ((rc = check_reach("b2_tti_forward", p, nd, a->radius, empty)) || empty) return rc;
    for (int d = 1; d <= nd; ++d)
        if (v->size[d] != u->size[d]) { set_error("b2_tti_forward: u and v shapes differ"); return B2_ERR_INVALID; }
    p.ndim = nd;
    p.R = a->radius;
    p.u = (float *)u->d;
    p.v = (float *)v->d;
    p.damp = damp ? (const float *)damp->d : nullptr;
    p.vp = a->vp;
    p.dt = a->dt;
    p.epsilon = a->epsilon;
    p.delta = a->delta;
    p.theta = a->theta;
    p.phi = a->phi;
    const float *pv[5];
    for (int i = 0; i < 5; ++i) pv[i] = parr[i] ? (const float *)parr[i]->d : nullptr;
    p.vp_a = pv[0]; p.eps_a = pv[1]; p.delta_a = pv[2]; p.theta_a = pv[3]; p.phi_a = pv[4];
    for (int di = 0; di < nd; ++di) {       // a 2-D plan's dummy dim keeps zero weights
        const int d = di + 3 - nd;
        if (!a->w2[di] || !a->w1[di]) { set_error("b2_tti_forward: weights missing"); return B2_ERR_INVALID; }
        for (int i = 0; i <= a->radius; ++i) p.w2[d][i] = a->w2[di][i];
        for (int i = 0; i < a->radius; ++i) p.w1[d][i] = a->w1[di][i];
    }
    {
        // both pairs run one sweep variant: a linearised pair that cannot take the fused kernel sends both to the
        // two-pass kernel (a forced fused kernel fails in tti_plan_retarget instead)
        int kernel = a->kernel;
        if (born && kernel != 2 && ((uintptr_t)bdu->d % 16 != 0 || (uintptr_t)bdv->d % 16 != 0)) kernel = 1;
        if ((rc = tti_plan_init(p, kernel))) return rc;
        if (born && (rc = tti_plan_retarget(p, (float *)bdu->d, (float *)bdv->d, pd))) return rc;
        if (adj && (rc = tti_plan_adjoint(p, pa))) return rc;
    }

    const FieldGeom g = field_geom(p, nd, a->halo);
    DevArray grad3;                             // grad with the plan's (dummy, x, z) extents on a 2-D grid
    if (grad) {
        grad3 = *grad;
        if (nd == 2) { grad3.size[0] = 1; grad3.size[1] = grad->size[0]; grad3.size[2] = grad->size[1]; }
    }

    const float dt2 = a->dt * a->dt;
    const float scalar_scale = dt2 * a->vp * a->vp;
    const int T = p.tsize;
    if ((rc = loop_timer_start(a->timers))) return rc;
    const bool p2p = a->halo && halo_p2p_active(a->halo, p.u) && halo_p2p_active(a->halo, p.v);
    if (a->halo) a->halo->reset_primed();
    const int dir = adj ? -1 : 1;
    for (int time = adj ? a->time_M : a->time_m; adj ? time >= a->time_m : time <= a->time_M; time += dir) {
        const int t0 = slot(time, T);
        const int t1 = slot(time + dir, T);     // written
        const int t2 = slot(time - dir, T);     // the other level read
        if (adj) {
            if ((rc = tti_adj_mix(pa, t0))) return rc;
            if ((rc = tti_step(pa, t0, t2, t1, 0, p.n[0]))) return rc;
        } else if (a->halo) {
            if ((rc = halo_exchange_and_step_tti(a->halo, p, t0, t2, t1))) return rc;
        } else {
            if ((rc = tti_step(p, t0, t2, t1, 0, p.n[0]))) return rc;
        }
        float *fu = p.u + (size_t)t1 * p.slot_elems;
        float *fv = p.v + (size_t)t1 * p.slot_elems;
        if ((rc = launch_inject(src, g, fu, fv, time, p.vp_a ? B2_PARAM_VP : B2_PARAM_SCALAR, p.vp_a,
                                scalar_scale, dt2)))
            return rc;
        if (p2p) {
            if ((rc = halo_p2p_publish(a->halo, p.u, p.v, p.slot_elems, t1, (size_t)p.sx, p.o[0], p.n[0], p.R)))
                return rc;
            a->halo->set_primed(p.u);
            a->halo->set_primed(p.v);
            // receivers that sample the just-written time level may touch halo cells: those
            // arrive with the neighbours' stores of this same step
            if (a->rec_toff && rec.present && (rc = halo_p2p_wait(a->halo))) return rc;
        }
        if (born) {
            if ((rc = tti_step(pd, t0, t2, t1, 0, p.n[0]))) return rc;
            if ((rc = tti_born_source(p, pd, t0, t2, t1, (const float *)bdm->d,
                                      nd == 3 ? (long long)bdm->size[1] * bdm->size[2] : 0, bdm->size[nd - 1], dmh)))
                return rc;
        }
        const size_t ro = (size_t)(a->rec_toff ? t1 : t0) * p.slot_elems;
        const TtiPlan &pr = born ? pd : p;
        if ((rc = launch_interp(rec, g, pr.u + ro, pr.v + ro, time))) return rc;
        if (grad) {
            if (time < 0 || time >= usave->size[0] || time >= vsave->size[0]) {
                set_error("b2_tti_forward: time=%d outside the saved wavefields (nt=%d, %d)", time, usave->size[0],
                          vsave->size[0]);
                return B2_ERR_INVALID;
            }
            if ((rc = launch_imaging(p, grad3, gh, (const float *)usave->d + (size_t)time * p.slot_elems, p.u,
                                     (const float *)vsave->d + (size_t)time * p.slot_elems, p.v, t0, t1, t2)))
                return rc;
        }
        if (a->errctl && errctl_due(time, a->time_m, adj ? a->time_m : a->time_M)) {
            if ((rc = check_finite(fu, p.slot_elems, "u", time))) return rc;
            if (born && (rc = check_finite(pd.u + (size_t)t1 * p.slot_elems, p.slot_elems, "du", time))) return rc;
        }
    }
    if (a->halo && (rc = halo_p2p_drain(a->halo))) return rc;
    return loop_finish("b2_tti_forward", a->timers);
}

extern "C" int b2_tti_forward(const struct b2_tti_args *a) {
    if (!a || !a->u || !a->v) { set_error("b2_tti_forward: NULL args"); return B2_ERR_INVALID; }
    if (a->ndim != 0 && a->ndim != 2 && a->ndim != 3) {
        set_error("b2_tti_forward: ndim must be 2 or 3 (0: 3)");
        return B2_ERR_INVALID;
    }
    if (a->time_M < a->time_m) return B2_OK;
    std::lock_guard<std::mutex> api_lock(api_mutex());
    if (int rc0 = use_device(a->deviceid)) return rc0;
    note_sweep_kernel("");
    Staging st;
    return st.finish(tti_forward_body(a, st));
}
