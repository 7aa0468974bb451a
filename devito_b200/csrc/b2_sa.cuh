// Self-adjoint variable-density visco-acoustic update (internal interface of b2_sa.cu). Scheme: b2_sa_point.cuh.
#pragma once
#include "b2_common.cuh"

namespace b2 {

// The box: a 2-D grid is (1, x, y) with radius 0 on dim 0.
struct SaPlan : Box {
    int radius[3] = {0, 0, 0};
    float *u = nullptr;
    float c[3][B2_MAX_RADIUS] = {};
    float dt = 0.f;
    // parameters: an array in u's space layout, or the scalar next to it
    const float *b_arr = nullptr, *vp_arr = nullptr, *w = nullptr;
    float b_value = 1.f, vp_value = 1.f;
    // library scratch: C = dt^2 vp^2 / b, and b expanded when it is a scalar
    float *C = nullptr, *b = nullptr;
    bool adjoint = false;
    // sa_tma<R> (3-D, R in {2, 4}, z rows and the box start 16-byte aligned): tensor maps of the haloed u[t] plane
    // (all slots; the slot is a coordinate) and of the haloed b plane
    bool use_tma = false;
    CUtensorMap tm_u, tm_b;
};

// Checks the layout, allocates the scratch and tabulates C (and b) over the whole allocated slot.
// kernel: 0 auto (sa_tma<R> when the layout qualifies, else k_sa_generic), 1 generic, 2 TMA (210 with a message
// when the layout does not qualify).
int sa_plan_init(SaPlan &p, int kernel);

// One time step: level slot1 from slot0 (centre and taps) and slotm (the other level read).
int sa_step(const SaPlan &p, int slot0, int slotm, int slot1);

}  // namespace b2
