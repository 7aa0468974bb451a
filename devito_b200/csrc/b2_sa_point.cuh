// One-point form of the self-adjoint variable-density visco-acoustic update (b2_sa_forward).
//
// `__host__ __device__`, like b2_iso_point.cuh, so that tests/support/emu_sa.cu can loop the same code on the CPU and
// compare it with the float64 restatement without a GPU. The scheme (the reference's `iso_stencil`,
// examples/seismic/self_adjoint/operators.py:4-65, at fd_order = space_order) with R = so/2 and c_k = the weights of
// `fd_weights(1, range(-R+1, R+1), 1/2)` at offset +k, divided by h_d (the weight at offset -k+1 is -c_k):
//
//   F_d(q)     = b(q) * sum_k c_k [u(q + k e_d) - u(q - (k-1) e_d)]          (inner derivative, at q + h/2)
//   (D-F_d)(p) = sum_k c_k [F_d(p + (k-1) e_d) - F_d(p - k e_d)]            (outer derivative, at p)
//   u_new(p)   = C(p) * sum_d (D-F_d)(p) + (2 - dt w(p)) u(p) + (dt w(p) - 1) u_old(p),   C = dt^2 vp^2 / b
//
// b is sampled at the grid nodes q (no interpolation), C and w at the output point. Forward in time u_new = u[t+1],
// u_old = u[t-1]; the adjoint writes u[t-1] from u[t] and u[t+1] with the same formula.
#pragma once
#include "b2_common.cuh"

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

// F_d at node q along stride s
B2_SA_HD float sa_flux(const SaK &k, const float *__restrict__ c, int R, long long q, long long s) {
    float acc = 0.f;
    for (int i = 1; i <= R; ++i) acc += c[i - 1] * (k.u0[q + i * s] - k.u0[q - (i - 1) * s]);
    return k.b[q] * acc;
}

// sum_d (D-F_d)(p)
B2_SA_HD float sa_div(const SaK &k, long long idx) {
    float acc = 0.f;
    const long long st[3] = {k.sx, k.sy, 1};
    for (int d = 0; d < 3; ++d) {
        const int R = k.r[d];
        const long long s = st[d];
        for (int i = 1; i <= R; ++i)
            acc += k.c[d][i - 1] * (sa_flux(k, k.c[d], R, idx + (i - 1) * s, s) - sa_flux(k, k.c[d], R, idx - i * s, s));
    }
    return acc;
}

B2_SA_HD void sa_point(const SaK &k, int x, int y, int z) {
    const long long idx = sa_index(k, x, y, z);
    const float dw = k.w ? k.dt * k.w[idx] : 0.f;
    k.u1[idx] = k.C[idx] * sa_div(k, idx) + (2.f - dw) * k.u0[idx] + (dw - 1.f) * k.um[idx];
}

}  // namespace b2
