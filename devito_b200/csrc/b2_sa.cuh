// Self-adjoint variable-density visco-acoustic update (internal interface of b2_sa.cu). Scheme: b2_sa_point.cuh.
#pragma once
#include "b2_common.cuh"
#include "b2_nested.cuh"

namespace b2 {

// The plan of NestedPlan's nested operator applied to u: the TMA sweep's maps are of u (every slot) and b.
struct SaPlan : NestedPlan {
    float *u = nullptr;
    const float *w = nullptr;        // w/Q in u's space layout, or null (no attenuation)
    float *C = nullptr;              // library scratch: C = dt^2 vp^2 / b
};

// Checks the layout, allocates the scratch and tabulates C (and b) over the whole allocated slot.
// kernel: 0 auto (sa_tma<R> when the layout qualifies, else k_sa_generic), 1 generic, 2 TMA (210 with a message
// when the layout does not qualify).
int sa_plan_init(SaPlan &p, int kernel);

// One time step: level slot1 from slot0 (centre and taps) and slotm (the other level read).
int sa_step(const SaPlan &p, int slot0, int slotm, int slot1);

}  // namespace b2
