// CPU emulation of the self-adjoint update's point body -- TEST INFRASTRUCTURE ONLY.
//
// devito_b200/csrc/b2_sa_point.cuh holds the body of k_sa_generic as a __host__ __device__ function. This file loops
// it over the iteration box on the CPU (compiled by nvcc as host code, no GPU needed), with the argument set-up of
// b2::sa_step (b2_sa.cu) in the internal 3-dim convention: a 2-D grid is (1, x, y) with radius 0 on dim 0.
#include "b2_sa_point.cuh"

using namespace b2;

// a[3]: allocated extents, lo / n: first domain index and extent of the box, C: dt^2 vp^2 / b, w may be null
extern "C" int emu_sa_step(const float *u0, const float *um, float *u1, const float *b, const float *C,
                           const float *w, const int *a, const int *lo, const int *n, const int *radius,
                           const float *c, int so, float dt) {
    SaK k;
    k.u0 = u0; k.um = um; k.u1 = u1; k.b = b; k.C = C; k.w = w;
    k.sy = a[2];
    k.sx = (long long)a[1] * a[2];
    k.n0 = n[0]; k.n1 = n[1]; k.n2 = n[2];
    k.o0 = radius[0] ? lo[0] + so : 0;
    k.o1 = lo[1] + so;
    k.o2 = lo[2] + so;
    for (int d = 0; d < 3; ++d) {
        k.r[d] = radius[d];
        for (int i = 0; i < B2_MAX_RADIUS; ++i) k.c[d][i] = i < radius[d] ? c[d * B2_MAX_RADIUS + i] : 0.f;
    }
    k.dt = dt;
    for (int x = 0; x < k.n0; ++x)
        for (int y = 0; y < k.n1; ++y)
            for (int z = 0; z < k.n2; ++z) sa_point(k, x, y, z);
    return 0;
}
