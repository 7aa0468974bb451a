// Second-order SLS viscoacoustic update (internal interface of b2_visco.cu). Scheme: b2_visco_point.cuh.
#pragma once
#include "b2_common.cuh"
#include "b2_visco_point.cuh"

namespace b2 {

// The box: a 2-D grid is (1, x, y) with radius 0 on dim 0.
struct ViscoPlan : Box {
    int radius[3] = {0, 0, 0};
    float *p = nullptr, *r = nullptr;
    float c[3][B2_MAX_RADIUS] = {};
    float dt = 0.f, f0 = 0.f;
    // parameters: an array in p's space layout, or the scalar next to it; damp null = 1 (no absorbing layer)
    const float *b_arr = nullptr, *vp_arr = nullptr, *qp_arr = nullptr, *damp = nullptr;
    float b_value = 1.f, vp_value = 1.f, qp_value = 1.f;
    // library scratch: the tables VK_*, b expanded when it is a scalar, and s (adjoint)
    float *K[VK_NTAB] = {};
    float *b = nullptr, *s = nullptr;
    bool adjoint = false;
    // visco_tma<R> (3-D, R in {2, 4}, z rows and the box start 16-byte aligned): tensor maps of the haloed plane of
    // the field L is applied to (p, every slot, the slot a coordinate; or s) and of the haloed b plane
    bool use_tma = false;
    CUtensorMap tm_f, tm_b;
};

// Checks the layout, allocates the scratch and tabulates the tables (and b) over the whole allocated slot.
// kernel: 0 auto (visco_tma<R> when the layout qualifies, else k_visco_generic), 1 generic, 2 TMA (210 with a
// message when the layout does not qualify).
int visco_plan_init(ViscoPlan &p, int kernel);

// One time step: p and r at slot t1 from slots t0 and t2 (forward: t1 = t+1, t2 = t-1; adjoint: t1 = t-1, t2 = t+1).
int visco_step(const ViscoPlan &p, int t0, int t2, int t1);

}  // namespace b2
