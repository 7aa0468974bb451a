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

namespace b2 {
int check_finite(const float *f, size_t n, bool &bad);
}

extern "C" int b2_tti_forward(const struct b2_tti_args *a) {
    if (!a || !a->u || !a->v) { set_error("b2_tti_forward: NULL args"); return B2_ERR_INVALID; }
    if (a->time_M < a->time_m) return B2_OK;
    std::lock_guard<std::mutex> api_lock(api_mutex());
    if (int rc0 = use_device(a->deviceid)) return rc0;
    note_sweep_kernel("");
    const int so = a->space_order;
    int rc = B2_OK;

    DevArray u, v, damp, parr[5], bdu, bdv, bdm, grad, usave, vsave;
    bool sparr[5] = {false, false, false, false, false};
    SparseDev src, rec;
    TtiPlan p, pd, pa;
    FieldGeom g;
    bool su = false, sv = false, sd = false, sdu = false, sdv = false, sdm = false, sg = false, sus = false,
         svs = false;

    auto cleanup = [&](int code) {
        const bool back = code == B2_OK || code == B2_ERR_NAN;
        int r1 = su ? stage_out(u, back) : B2_OK;
        int r2 = sv ? stage_out(v, back) : B2_OK;
        const int r4 = sdu ? stage_out(bdu, back) : B2_OK;
        const int r5 = sdv ? stage_out(bdv, back) : B2_OK;
        if (sdm) stage_out(bdm, false);
        if (sus) stage_out(usave, false);
        if (svs) stage_out(vsave, false);
        const int r6 = sg ? stage_out(grad, back) : B2_OK;
        if (sd) stage_out(damp, false);
        for (int i = 0; i < 5; ++i) if (sparr[i]) stage_out(parr[i], false);
        sparse_stage_out(src, false);
        int r3 = sparse_stage_out(rec, back);
        tti_plan_free(p);
        if (code != B2_OK) return code;
        return r1 ? r1 : (r2 ? r2 : (r3 ? r3 : (r4 ? r4 : (r5 ? r5 : r6))));
    };

    if ((rc = stage_in(a->u, 4, u, true))) return cleanup(rc);
    su = true;
    if ((rc = stage_in(a->v, 4, v, true))) return cleanup(rc);
    sv = true;
    if (a->damp) {
        if ((rc = stage_in(a->damp, 3, damp, true))) return cleanup(rc);
        sd = true;
    }
    {
        const b2_dataobj *pa[5] = {a->vp_arr, a->epsilon_arr, a->delta_arr, a->theta_arr, a->phi_arr};
        for (int i = 0; i < 5; ++i)
            if (pa[i]) {
                if ((rc = stage_in(pa[i], 3, parr[i], true))) return cleanup(rc);
                sparr[i] = true;
            }
    }
    const bool born = a->born_du || a->born_dv || a->born_dm;
    int dmh = 0;
    if (born) {
        if (!a->born_du || !a->born_dv || !a->born_dm) {
            set_error("b2_tti_forward: Born modelling needs born_du, born_dv and born_dm together");
            return cleanup(B2_ERR_INVALID);
        }
        if (a->halo) {
            set_error("b2_tti_forward: Born modelling is not combined with halo exchange in this version");
            return cleanup(B2_ERR_INVALID);
        }
        if ((rc = stage_in(a->born_du, 4, bdu, true))) return cleanup(rc);
        sdu = true;
        if ((rc = stage_in(a->born_dv, 4, bdv, true))) return cleanup(rc);
        sdv = true;
        if ((rc = stage_in(a->born_dm, 3, bdm, true))) return cleanup(rc);
        sdm = true;
        for (int d = 0; d < 4; ++d)
            if (bdu.size[d] != u.size[d] || bdv.size[d] != u.size[d]) {
                set_error("b2_tti_forward: born_du and born_dv must have the layout of u");
                return cleanup(B2_ERR_INVALID);
            }
        dmh = a->born_dm->hsize ? a->born_dm->hsize[0] : (bdm.size[0] - (u.size[1] - 2 * so)) / 2;
        for (int d = 0; d < 3; ++d)
            if (dmh < 0 || bdm.size[d] != u.size[d + 1] - 2 * so + 2 * dmh) {
                set_error("b2_tti_forward: born_dm extent %d on dim %d does not match the grid", bdm.size[d], d);
                return cleanup(B2_ERR_INVALID);
            }
    }
    const bool adj = a->adjoint != 0;
    int gh = 0;
    if (adj && a->halo) {
        set_error("b2_tti_forward: the adjoint is not combined with halo exchange in this version");
        return cleanup(B2_ERR_INVALID);
    }
    if (adj && born) {
        set_error("b2_tti_forward: the adjoint is not combined with Born modelling");
        return cleanup(B2_ERR_INVALID);
    }
    if (a->grad || a->usave || a->vsave) {
        if (!a->grad || !a->usave || !a->vsave) {
            set_error("b2_tti_forward: the imaging condition needs grad, usave and vsave together");
            return cleanup(B2_ERR_INVALID);
        }
        if (!adj) {
            set_error("b2_tti_forward: the imaging condition runs with the adjoint only");
            return cleanup(B2_ERR_INVALID);
        }
        if ((rc = stage_in(a->grad, 3, grad, true))) return cleanup(rc);
        sg = true;
        if ((rc = stage_in(a->usave, 4, usave, true))) return cleanup(rc);
        sus = true;
        if ((rc = stage_in(a->vsave, 4, vsave, true))) return cleanup(rc);
        svs = true;
        for (int d = 1; d < 4; ++d)
            if (usave.size[d] != u.size[d] || vsave.size[d] != u.size[d]) {
                set_error("b2_tti_forward: usave and vsave must have the space layout of u");
                return cleanup(B2_ERR_INVALID);
            }
        gh = a->grad->hsize ? a->grad->hsize[0] : (grad.size[0] - (u.size[1] - 2 * so)) / 2;
        for (int d = 0; d < 3; ++d)
            if (gh < 0 || grad.size[d] != u.size[d + 1] - 2 * so + 2 * gh) {
                set_error("b2_tti_forward: grad extent %d on dim %d does not match the grid", grad.size[d], d);
                return cleanup(B2_ERR_INVALID);
            }
    }
    if ((rc = sparse_stage_in(a->src, 3, src, true))) return cleanup(rc);
    if ((rc = sparse_stage_in(a->rec, 3, rec, true))) return cleanup(rc);
    // devito/operations/interpolators.py:28-37 `check_radius`
    if ((src.present && src.r > so) || (rec.present && rec.r > so)) {
        set_error("b2_tti_forward: sparse radius %d exceeds the halo (space_order %d)",
                  src.present && src.r > so ? src.r : rec.r, so);
        return cleanup(B2_ERR_INVALID);
    }

    const int lo_in[3] = {a->x_m, a->y_m, a->z_m};
    const int hi_in[3] = {a->x_M, a->y_M, a->z_M};
    p.R = a->radius;
    p.so = so;
    p.tsize = u.size[0];
    for (int d = 0; d < 3; ++d) {
        p.a[d] = u.size[d + 1];
        p.n[d] = hi_in[d] - lo_in[d] + 1;
        p.o[d] = lo_in[d] + so;
        if (p.n[d] <= 0) return cleanup(B2_OK);
        if (v.size[d + 1] != p.a[d]) { set_error("b2_tti_forward: u and v shapes differ"); return cleanup(B2_ERR_INVALID); }
        if (p.o[d] - p.R < 0 || p.o[d] + p.n[d] - 1 + p.R >= p.a[d]) {
            set_error("b2_tti_forward: iteration range + radius leaves the allocated array on dim %d", d);
            return cleanup(B2_ERR_INVALID);
        }
    }
    p.sy = p.a[2];
    p.sx = (long long)p.a[1] * p.a[2];
    p.slot_elems = (size_t)p.a[0] * p.a[1] * p.a[2];
    p.u = (float *)u.d;
    p.v = (float *)v.d;
    p.damp = a->damp ? (const float *)damp.d : nullptr;
    p.vp = a->vp;
    p.dt = a->dt;
    p.epsilon = a->epsilon;
    p.delta = a->delta;
    p.theta = a->theta;
    p.phi = a->phi;
    p.vp_a = sparr[0] ? (const float *)parr[0].d : nullptr;
    p.eps_a = sparr[1] ? (const float *)parr[1].d : nullptr;
    p.delta_a = sparr[2] ? (const float *)parr[2].d : nullptr;
    p.theta_a = sparr[3] ? (const float *)parr[3].d : nullptr;
    p.phi_a = sparr[4] ? (const float *)parr[4].d : nullptr;
    for (int d = 0; d < 3; ++d) {
        if (!a->w2[d] || !a->w1[d]) { set_error("b2_tti_forward: weights missing"); return cleanup(B2_ERR_INVALID); }
        for (int i = 0; i <= a->radius; ++i) p.w2[d][i] = a->w2[d][i];
        for (int i = 0; i < a->radius; ++i) p.w1[d][i] = a->w1[d][i];
    }
    {
        // both pairs run one sweep variant: a linearised pair that cannot take the fused kernel sends both to the
        // two-pass kernel (a forced fused kernel fails in tti_plan_retarget instead)
        int kernel = a->kernel;
        if (born && kernel != 2 && ((uintptr_t)bdu.d % 16 != 0 || (uintptr_t)bdv.d % 16 != 0)) kernel = 1;
        if ((rc = tti_plan_init(p, kernel))) return cleanup(rc);
        if (born && (rc = tti_plan_retarget(p, (float *)bdu.d, (float *)bdv.d, pd))) return cleanup(rc);
        if (adj && (rc = tti_plan_adjoint(p, pa))) return cleanup(rc);
    }

    g.sx = p.sx;
    g.sy = p.sy;
    g.slot_elems = p.slot_elems;
    g.so = so;
    g.ndim = 3;
    for (int d = 0; d < 3; ++d) { g.lo[d] = lo_in[d]; g.hi[d] = hi_in[d]; }
    if (a->halo) { g.nb_lo = a->halo->rank > 0; g.nb_hi = a->halo->rank < a->halo->nranks - 1; }

    const float dt2 = a->dt * a->dt;
    const float scalar_scale = dt2 * a->vp * a->vp;
    const int T = p.tsize;
    static cudaEvent_t e0 = nullptr, e1 = nullptr;      // created once (the process is bound to one device)
    if (a->timers) {
        if (!e0 && (cudaEventCreate(&e0) != cudaSuccess || cudaEventCreate(&e1) != cudaSuccess)) {
            e0 = e1 = nullptr;
            set_error("b2_tti_forward: cannot create timing events");
            return cleanup(B2_ERR_DEVICE);
        }
        cudaEventRecord(e0, stream());
    }
    const bool p2p = a->halo && halo_p2p_active(a->halo, p.u) && halo_p2p_active(a->halo, p.v);
    if (a->halo) a->halo->reset_primed();
    const int dir = adj ? -1 : 1;
    for (int time = adj ? a->time_M : a->time_m; adj ? time >= a->time_m : time <= a->time_M; time += dir) {
        const int t0 = ((time % T) + T) % T;
        const int t1 = (((time + dir) % T) + T) % T;     // written
        const int t2 = (((time - dir) % T) + T) % T;     // the other level read
        if (adj) {
            if ((rc = tti_adj_mix(pa, t0))) return cleanup(rc);
            if ((rc = tti_step(pa, t0, t2, t1, 0, p.n[0]))) return cleanup(rc);
        } else if (a->halo) {
            if ((rc = halo_exchange_and_step_tti(a->halo, p, t0, t2, t1))) return cleanup(rc);
        } else {
            if ((rc = tti_step(p, t0, t2, t1, 0, p.n[0]))) return cleanup(rc);
        }
        float *fu = p.u + (size_t)t1 * p.slot_elems;
        float *fv = p.v + (size_t)t1 * p.slot_elems;
        if ((rc = launch_inject(src, g, fu, fv, time, p.vp_a ? B2_PARAM_VP : B2_PARAM_SCALAR, p.vp_a,
                                scalar_scale, dt2)))
            return cleanup(rc);
        if (p2p) {
            if ((rc = halo_p2p_publish(a->halo, p.u, p.v, p.slot_elems, t1, (size_t)p.sx, p.o[0], p.n[0], p.R)))
                return cleanup(rc);
            a->halo->set_primed(p.u);
            a->halo->set_primed(p.v);
            // receivers that sample the just-written time level may touch halo cells: those
            // arrive with the neighbours' stores of this same step
            if (a->rec_toff && rec.present && (rc = halo_p2p_wait(a->halo))) return cleanup(rc);
        }
        if (born) {
            if ((rc = tti_step(pd, t0, t2, t1, 0, p.n[0]))) return cleanup(rc);
            if ((rc = tti_born_source(p, pd, t0, t2, t1, (const float *)bdm.d, (long long)bdm.size[1] * bdm.size[2],
                                      bdm.size[2], dmh)))
                return cleanup(rc);
        }
        const size_t ro = (size_t)(a->rec_toff ? t1 : t0) * p.slot_elems;
        const TtiPlan &pr = born ? pd : p;
        if ((rc = launch_interp(rec, g, pr.u + ro, pr.v + ro, time))) return cleanup(rc);
        if (sg) {
            if (time < 0 || time >= usave.size[0] || time >= vsave.size[0]) {
                set_error("b2_tti_forward: time=%d outside the saved wavefields (nt=%d, %d)", time, usave.size[0],
                          vsave.size[0]);
                return cleanup(B2_ERR_INVALID);
            }
            ImgK ik;
            ik.grad = (float *)grad.d;
            ik.us = (const float *)usave.d + (size_t)time * p.slot_elems;
            ik.v0 = p.u + (size_t)t0 * p.slot_elems;
            ik.v1 = p.u + (size_t)t1 * p.slot_elems;
            ik.v2 = p.u + (size_t)t2 * p.slot_elems;
            ik.us2 = (const float *)vsave.d + (size_t)time * p.slot_elems;
            ik.w0 = p.v + (size_t)t0 * p.slot_elems;
            ik.w1 = p.v + (size_t)t1 * p.slot_elems;
            ik.w2 = p.v + (size_t)t2 * p.slot_elems;
            ik.sx = p.sx; ik.sy = p.sy;
            ik.gsy = grad.size[2];
            ik.gsx = (long long)grad.size[1] * grad.size[2];
            ik.n0 = p.n[0]; ik.n1 = p.n[1]; ik.n2 = p.n[2];
            ik.o0 = p.o[0]; ik.o1 = p.o[1]; ik.o2 = p.o[2];
            ik.g0 = a->x_m + gh; ik.g1 = a->y_m + gh; ik.g2 = a->z_m + gh;
            ik.inv_dt2 = 1.0f / (a->dt * a->dt);
            if ((rc = launch_imaging(ik))) return cleanup(rc);
        }
        if (a->errctl && ((time - a->time_m) % 100 == 99 || time == (adj ? a->time_m : a->time_M))) {
            bool bad = false;
            if ((rc = check_finite(fu, p.slot_elems, bad))) return cleanup(rc);
            if (bad) { set_error("NaN/Inf detected in u at time=%d", time); return cleanup(B2_ERR_NAN); }
            if (born) {
                if ((rc = check_finite(pd.u + (size_t)t1 * p.slot_elems, p.slot_elems, bad))) return cleanup(rc);
                if (bad) { set_error("NaN/Inf detected in du at time=%d", time); return cleanup(B2_ERR_NAN); }
            }
        }
    }
    if (a->halo && (rc = halo_p2p_drain(a->halo))) return cleanup(rc);
    if (a->timers) cudaEventRecord(e1, stream());
    cudaError_t e = cudaStreamSynchronize(stream());
    if (e != cudaSuccess) {
        set_error("b2_tti_forward: device error: %s", cudaGetErrorString(e));
        return cleanup(B2_ERR_LAUNCH);
    }
    if (a->timers) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, e0, e1);
        a->timers->section0 += ms * 1e-3;
    }
    return cleanup(B2_OK);
}
