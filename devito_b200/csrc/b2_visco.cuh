// Second-order SLS viscoacoustic update (internal interface of b2_visco.cu). Scheme: b2_visco_point.cuh.
#pragma once
#include "b2_common.cuh"
#include "b2_nested.cuh"
#include "b2_visco_point.cuh"

namespace b2 {

// The plan of NestedPlan's nested operator applied to p (forward) or s (adjoint): the TMA sweep's maps are of that
// field (p: every slot; s: its one slot) and b.
struct ViscoPlan : NestedPlan {
    float *p = nullptr, *r = nullptr;
    float f0 = 0.f;
    // an array in p's space layout, or the scalar next to it; damp null = 1 (no absorbing layer)
    const float *qp_arr = nullptr, *damp = nullptr;
    float qp_value = 1.f;
    // library scratch: the tables VK_*, and s (adjoint)
    float *K[VK_NTAB] = {};
    float *s = nullptr;
};

// Checks the layout, allocates the scratch and tabulates the tables (and b) over the whole allocated slot.
// kernel: 0 auto (visco_tma<R> when the layout qualifies, else k_visco_generic), 1 generic, 2 TMA (210 with a
// message when the layout does not qualify).
int visco_plan_init(ViscoPlan &p, int kernel);

// One time step: p and r at slot t1 from slots t0 and t2 (forward: t1 = t+1, t2 = t-1; adjoint: t1 = t-1, t2 = t+1).
int visco_step(const ViscoPlan &p, int t0, int t2, int t1);

}  // namespace b2
