// CPU emulation of the SLS viscoacoustic update -- TEST INFRASTRUCTURE ONLY.
//
// devito_b200/csrc/b2_visco_point.cuh holds the table formula of k_visco_coef, the adjoint's mix (k_visco_adj_mix)
// and the point body of k_visco_generic as __host__ __device__ functions. This file runs them on the CPU (compiled by
// nvcc as host code, no GPU needed) for one time step, with the argument set-up of b2::visco_plan_init and
// b2::visco_step (b2_visco.cu) in the internal 3-dim convention: a 2-D grid is (1, x, y) with radius 0 on dim 0.
#include "b2_visco_point.cuh"

#include <vector>

using namespace b2;

// a[3]: allocated extents, lo / n: first domain index and extent of the box. vp, qp, damp: arrays of the slot (damp
// may be null). p0 = p[t], pm = p[t - dir], p1 = p[t + dir]; r0 = r[t], r1 = r[t + dir]. Forward writes p1 and r1 in
// the box; adjoint writes r1 in the box and p1 in the box from s = ((1 + tt) p[t] + r[t-1]) / b over the slot.
extern "C" int emu_visco_step(const float *p0, const float *pm, float *p1, const float *r0, float *r1, const float *b,
                              const float *vp, const float *qp, const float *damp, const int *a, const int *lo,
                              const int *n, const int *radius, const float *c, int so, float dt, float f0,
                              int adjoint) {
    const size_t elems = (size_t)a[0] * a[1] * a[2];
    std::vector<float> tab[VK_NTAB], s;
    ViscoCoefK ck;
    for (int i = 0; i < VK_NTAB; ++i) {
        tab[i].resize(elems);
        ck.K[i] = tab[i].data();
    }
    ck.bx = nullptr;
    ck.vp = vp; ck.qp = qp; ck.damp = damp;
    ck.vp_value = ck.qp_value = ck.b_value = 1.f;
    ck.f0 = f0; ck.dt = dt;
    ck.n = elems;
    for (size_t i = 0; i < elems; ++i) visco_coef_point(ck, i);

    ViscoK k;
    k.p0 = p0; k.pm = pm; k.p1 = p1; k.f = p0;
    k.r0 = adjoint ? nullptr : r0;
    k.r1 = adjoint ? nullptr : r1;
    k.b = b;
    for (int i = 0; i < VK_NTAB; ++i) k.K[i] = tab[i].data();
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
    k.adjoint = adjoint;
    if (adjoint) {
        s.resize(elems);
        ViscoMixK mk;
        for (int i = 0; i < VK_NTAB; ++i) mk.K[i] = tab[i].data();
        mk.b = b; mk.p0 = p0; mk.r0 = r0; mk.rw = r1; mk.s = s.data();
        mk.sx = k.sx; mk.sy = k.sy;
        mk.o0 = k.o0; mk.o1 = k.o1; mk.o2 = k.o2;
        mk.n0 = k.n0; mk.n1 = k.n1; mk.n2 = k.n2;
        mk.n = elems;
        for (size_t i = 0; i < elems; ++i) visco_mix_at(mk, i);
        k.f = s.data();
    }
    for (int x = 0; x < k.n0; ++x)
        for (int y = 0; y < k.n1; ++y)
            for (int z = 0; z < k.n2; ++z) visco_point(k, x, y, z);
    return 0;
}
