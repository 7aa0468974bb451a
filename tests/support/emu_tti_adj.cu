// CPU emulation of the centred-TTI adjoint's field mix -- TEST INFRASTRUCTURE ONLY.
//
// devito_b200/csrc/b2_tti_point.cuh holds the body of k_tti_adj_mix as a __host__ __device__ function. This file
// loops it over a whole slot on the CPU (compiled by nvcc as host code, no GPU needed), with the argument set-up of
// b2::tti_adj_mix (b2_tti.cu): e2 / sd from per-point tables when given, else from the scalar epsilon / delta.
#include "b2_tti_point.cuh"
#include <cmath>

using namespace b2;

extern "C" int emu_tti_adj_mix(const float *p, const float *r, float *a, float *b, const float *tE2,
                               const float *tSD, float epsilon, float delta, long long n) {
    const float e2 = 1.0f + 2.0f * epsilon;
    const float sd = sqrtf(1.0f + 2.0f * delta);
    for (long long i = 0; i < n; ++i)
        tti_adj_mix_point(tE2 ? tE2[i] : e2, tSD ? tSD[i] : sd, p[i], r[i], a[i], b[i]);
    return 0;
}
