// One-point form of the self-adjoint variable-density visco-acoustic update (b2_sa_forward).
//
// `__host__ __device__`, like b2_iso_point.cuh, so that tests/support/emu_sa.cu can loop the same code on the CPU and
// compare it with the float64 restatement without a GPU. The scheme (the reference's `iso_stencil`,
// examples/seismic/self_adjoint/operators.py:4-65, at fd_order = space_order) with R = so/2, c_k = the weights of
// `fd_weights(1, range(-R+1, R+1), 1/2)` at offset +k divided by h_d, and L the nested operator of
// b2_nested_point.cuh applied to u[t]:
//
//   u_new(p)   = C(p) * L(u)(p) + (2 - dt w(p)) u(p) + (dt w(p) - 1) u_old(p),   C = dt^2 vp^2 / b
//
// C and w are sampled at the output point. Forward in time u_new = u[t+1], u_old = u[t-1]; the adjoint writes u[t-1]
// from u[t] and u[t+1] with the same formula.
#pragma once
#include "b2_nested_point.cuh"

namespace b2 {

struct SaK {
    const float *__restrict__ u0;    // u[t]
    const float *__restrict__ um;    // u[t - dir]
    float *__restrict__ u1;          // u[t + dir], written
    const float *__restrict__ b;     // buoyancy, u's space layout (a scalar b is expanded into scratch)
    const float *__restrict__ C;     // dt^2 vp^2 / b, u's space layout (k_sa_coef)
    const float *__restrict__ w;     // w/Q, u's space layout, or null (no attenuation)
    long long sx, sy;
    int n0, n1, n2;                  // extents of this launch
    int o0, o1, o2;                  // array index of the first point
    int r[3];                        // radius per internal dim (0 on the dummy dim of a 2-D grid)
    float c[3][B2_MAX_RADIUS];       // c[d][k-1] = c_k / h_d
    float dt;
};

#define B2_SA_HD __host__ __device__ __forceinline__

B2_SA_HD long long sa_index(const SaK &k, int x, int y, int z) {
    return (long long)(k.o0 + x) * k.sx + (long long)(k.o1 + y) * k.sy + (k.o2 + z);
}

B2_SA_HD void sa_point(const SaK &k, int x, int y, int z) {
    const long long idx = sa_index(k, x, y, z);
    const float dw = k.w ? k.dt * k.w[idx] : 0.f;
    k.u1[idx] = k.C[idx] * nested_div(k.u0, k.b, k.sx, k.sy, k.r, k.c, idx) + (2.f - dw) * k.u0[idx] + (dw - 1.f) * k.um[idx];
}

}  // namespace b2
