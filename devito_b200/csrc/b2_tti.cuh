// TTI (tilted transverse isotropy) centred-kernel stencils — internal interface.
#pragma once
#include "b2_common.cuh"

namespace b2 {

// A 2-D grid (x, z) is planned as (1, x, z): extent 1 and no stencil taps on the leading dim, rotation factors
// (0, sin theta, cos theta). Its sweeps march along the grid's x, the plan's dim 1.
struct TtiPlan : Box {
    int ndim = 3;                // 2 or 3
    int R = 4;                   // radius = space_order/2 (even)
    float *u = nullptr, *v = nullptr;
    const float *damp = nullptr;
    float vp = 1.f, dt = 1.f, epsilon = 0.f, delta = 0.f, theta = 0.f, phi = 0.f;
    float w2[3][B2_MAX_RADIUS + 1] = {};
    float w1[3][B2_MAX_RADIUS] = {};
    // scratch (two-pass kernel): Gz(u), Gz(v)
    float *gzu = nullptr, *gzv = nullptr;
    int kernel = 0;
    // fused single-pass kernel
    bool use_fused = false;
    bool arr_fused = false;      // fused kernel with per-point parameter tables (k_tti_fused<.., ARR = true>)
    CUtensorMap tm_u, tm_v;
    CUtensorMap tm_cx, tm_cy, tm_cz;   // factor tables (arr_fused)
    float *coefA = nullptr;
    // array-valued parameters (device pointers, nullptr -> scalar)
    const float *vp_a = nullptr, *eps_a = nullptr, *delta_a = nullptr, *theta_a = nullptr, *phi_a = nullptr;
    // tabulated per-point coefficients (library scratch) when any parameter is an array
    float *tCx = nullptr, *tCy = nullptr, *tCz = nullptr, *tE2 = nullptr, *tSD = nullptr, *tMD = nullptr;
    bool has_arrays = false;
    int tm_rows = 0;             // rows of the u / v tensor-map boxes (fused plans)
    bool use_2d = false;         // 2-D single-pass sweep k_tti2d (tm_u / tm_v: row boxes; ARR: tm_cy / tm_cz)
    // adjoint plan (tti_plan_adjoint): the sweep's stencil inputs are the one-slot mixes ma = e2 p + sd r and
    // mb = sd p + r (library scratch, tm_u / tm_v cover them), combined with (1, 0); u / v stay p / r, whose level
    // slot0 gives the centre of the update, slotm the previous level and slot1 the level written
    bool adj = false;
    float *ma = nullptr, *mb = nullptr;
};

int tti_plan_init(TtiPlan &p, int kernel);
// A plan for a second field pair (u, v) of the same layout that shares p's tables, scratch and sweep variant: only the
// tensor maps are rebuilt for the new pointers. Fails (210) when p is fused and the new pointers do not qualify.
int tti_plan_retarget(const TtiPlan &p, float *u, float *v, TtiPlan &out);
// one time step over x in [xlo, xlo+xcount)
int tti_step(const TtiPlan &p, int slot0, int slotm, int slot1, int xlo, int xcount);
// Born source term (b2_tti_point.cuh) over the whole box after the linearised pair `pd` was stepped with the same
// sweep as the background pair `p`: adds -dm * f.dt2 / (m/dt^2 + damp/dt) of p's u / v to pd's u / v at slot1.
// `dm` has strides dsx, dsy and its own halo width dmh. Appends "+born_v4" / "+born_s" to the sweep-kernel name.
int tti_born_source(const TtiPlan &p, const TtiPlan &pd, int slot0, int slotm, int slot1, const float *dm,
                    long long dsx, long long dsy, int dmh);
// The adjoint plan of p (same sweep variant, tables and A): a copy of p whose tensor maps cover two one-slot scratch
// buffers, the mixes written by tti_adj_mix.
int tti_plan_adjoint(const TtiPlan &p, TtiPlan &out);
// k_tti_adj_mix: the adjoint plan's scratch slots from level slot0 of p / r, over the whole allocated slot (the
// sweep reads them up to R outside the box). 16 B/point with scalar parameters, 24 with the e2 / sd tables.
int tti_adj_mix(const TtiPlan &pa, int slot0);

}  // namespace b2
