// One-point form of the nested operator of the self-adjoint (b2_sa_point.cuh) and SLS viscoacoustic
// (b2_visco_point.cuh) updates, with R = so/2 and c_k the half-node first-derivative weights at offset +k divided by h_d
// (the weight at offset -k+1 is -c_k):
//
//   F_d(q) = b(q) * sum_k c_k [f(q + k e_d) - f(q - (k-1) e_d)]                  (inner derivative, at q + h/2)
//   L(f)(p) = sum_d sum_k c_k [F_d(p + (k-1) e_d) - F_d(p - k e_d)]              (outer derivative, at p)
//
// b is sampled at the grid nodes q (no interpolation). `__host__ __device__`, so that the emulators of tests/support run
// the same code on the CPU. The 2.5-D TMA form of L is k_nested_tma (b2_nested.cuh); this header stays free of it so
// that it compiles for any architecture.
#pragma once
#include "b2_common.cuh"

namespace b2 {

#define B2_NESTED_HD __host__ __device__ __forceinline__

// The pointers are not __restrict__: with it k_sa_generic and k_visco_generic spill (40 registers instead of 48).

// F_d at node q along stride s, radius R, weights c
B2_NESTED_HD float nested_flux(const float *f, const float *b, const float *c, int R, long long q, long long s) {
    float acc = 0.f;
    for (int i = 1; i <= R; ++i) acc += c[i - 1] * (f[q + i * s] - f[q - (i - 1) * s]);
    return b[q] * acc;
}

// L(f) at idx: strides (sx, sy, 1), r[d] the radius and c[d][k-1] = c_k / h_d on dim d (radius 0: no term)
B2_NESTED_HD float nested_div(const float *f, const float *b, long long sx, long long sy, const int *r,
                              const float (*c)[B2_MAX_RADIUS], long long idx) {
    float acc = 0.f;
    const long long st[3] = {sx, sy, 1};
    for (int d = 0; d < 3; ++d) {
        const int R = r[d];
        const long long s = st[d];
        for (int i = 1; i <= R; ++i)
            acc += c[d][i - 1] * (nested_flux(f, b, c[d], R, idx + (i - 1) * s, s) -
                                  nested_flux(f, b, c[d], R, idx - i * s, s));
    }
    return acc;
}

}  // namespace b2
