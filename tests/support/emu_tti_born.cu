// CPU emulation of the centred-TTI Born source term -- TEST INFRASTRUCTURE ONLY.
//
// devito_b200/csrc/b2_tti_point.cuh holds the body of k_tti_born_src's one-point path as a __host__ __device__
// function. This file loops it over the box on the CPU (compiled by nvcc as host code, no GPU needed), with the
// argument set-up of b2::tti_born_source (b2_tti.cu), so that tests/test_zz_tti_born.py can compare the very code the
// GPU runs with float64.
#include "b2_tti_point.cuh"

using namespace b2;

// Centred-TTI Born source term (b2::tti_born_source, b2_tti.cu) over the box, one point at a time: du, dv at slot t1
// get -dm * f.dt2 of u, v divided by the denominator (A != NULL: times the tabulated A; else m/dt^2 from md or the
// scalar vp, plus damp/dt). `dm` has its own allocation and halo width.
extern "C" int emu_tti_born_source(const float *u, const float *v, float *du, float *dv, const float *dm,
                                   const int *dmalloc, int dmh, const int *alloc, int so, const float *A,
                                   const float *md, const float *damp, float vp, float dt, const int *lo,
                                   const int *hi, int t0, int t2, int t1) {
    TtiBK k;
    const size_t slot = (size_t)alloc[0] * alloc[1] * alloc[2];
    k.u1 = u + (size_t)t1 * slot; k.u0 = u + (size_t)t0 * slot; k.um = u + (size_t)t2 * slot;
    k.v1 = v + (size_t)t1 * slot; k.v0 = v + (size_t)t0 * slot; k.vm = v + (size_t)t2 * slot;
    k.du1 = du + (size_t)t1 * slot;
    k.dv1 = dv + (size_t)t1 * slot;
    k.A = A;
    k.tMD = md;
    k.damp = damp;
    k.dm = dm;
    k.sy = alloc[2];
    k.sx = (long long)alloc[1] * alloc[2];
    k.dsy = dmalloc[2];
    k.dsx = (long long)dmalloc[1] * dmalloc[2];
    k.n0 = hi[0] - lo[0] + 1; k.n1 = hi[1] - lo[1] + 1; k.n2 = hi[2] - lo[2] + 1;
    k.o0 = lo[0] + so; k.o1 = lo[1] + so; k.o2 = lo[2] + so;
    k.dg0 = lo[0] + dmh; k.dg1 = lo[1] + dmh; k.dg2 = lo[2] + dmh;
    k.inv_dt = 1.0f / dt;
    k.inv_dt2 = 1.0f / (dt * dt);
    k.m_dt2 = (1.0f / (vp * vp)) * k.inv_dt2;
    for (int x = 0; x < k.n0; ++x)
        for (int y = 0; y < k.n1; ++y)
            for (int z = 0; z < k.n2; ++z) tti_born_point(k, x, y, z);
    return 0;
}
