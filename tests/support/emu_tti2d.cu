// CPU emulation of one step of the 2-D centred-TTI sweep -- TEST INFRASTRUCTURE ONLY.
//
// devito_b200/csrc/b2_tti_point.cuh holds the point forms k_tti2d (b2_tti.cu) calls: the Gz combination, the forward
// and adjoint time updates, and the adjoint's mix. This file applies them one point at a time on the CPU (compiled by
// nvcc as host code, no GPU needed) with the sweep's derivative sums, so that tests/test_zz_tti2d.py can compare the
// very point code the GPU runs with the float64 restatement (tests/tti2d_ref.py).
#include <vector>

#include "b2_tti_point.cuh"

using namespace b2;

// One step over the box [lo, hi] (grid indices) of fields laid out (slots, nx + 2 so, nz + 2 so): slot t1 of u, v
// is written from slots t0 (centre) and t2 (the other level). Per-point tables over the whole slot: s, c = sin / cos
// of theta, e2 = 1+2 eps, sd = sqrt(1+2 delta), md = m/dt^2, A = 1/(md + damp/dt). `adj` != 0: the adjoint step,
// whose stencil inputs are the mixes e2 p + sd r, sd p + r.
extern "C" int emu_tti2d_step(float *u, float *v, const int *alloc, int so, const float *w2x, const float *w2z,
                              const float *w1x, const float *w1z, const float *s, const float *c, const float *e2,
                              const float *sd, const float *md, const float *A, const int *lo, const int *hi, int t0,
                              int t2, int t1, int adj) {
    const int R = so / 2, H = R / 2;
    const long long sr = alloc[1], slot = (long long)alloc[0] * alloc[1];
    const float *u0 = u + t0 * slot, *v0 = v + t0 * slot, *um = u + t2 * slot, *vm = v + t2 * slot;
    float *u1 = u + t1 * slot, *v1 = v + t1 * slot;
    std::vector<float> fa(slot), fb(slot), gu(slot, 0.f), gv(slot, 0.f);
    for (long long i = 0; i < slot; ++i) {
        if (adj) tti_adj_mix_point(e2[i], sd[i], u0[i], v0[i], fa[i], fb[i]);
        else { fa[i] = u0[i]; fb[i] = v0[i]; }
    }
    auto at = [&](int x, int z) { return (long long)(x + so) * sr + (z + so); };
    // Gz on the box grown by [-H, H-1]
    for (int x = lo[0] - H; x <= hi[0] + H - 1; ++x)
        for (int z = lo[1] - H; z <= hi[1] + H - 1; ++z) {
            const long long i = at(x, z);
            float dxa = 0.f, dza = 0.f, dxb = 0.f, dzb = 0.f;
            for (int j = 0; j < R; ++j) {
                const int o = j - H + 1;
                dxa = fmaf(w1x[j], fa[i + o * sr], dxa); dza = fmaf(w1z[j], fa[i + o], dza);
                dxb = fmaf(w1x[j], fb[i + o * sr], dxb); dzb = fmaf(w1z[j], fb[i + o], dzb);
            }
            gu[i] = tti2d_gz_point(s[i], c[i], dxa, dza);
            gv[i] = tti2d_gz_point(s[i], c[i], dxb, dzb);
        }
    for (int x = lo[0]; x <= hi[0]; ++x)
        for (int z = lo[1]; z <= hi[1]; ++z) {
            const long long i = at(x, z);
            float lap = (w2x[0] + w2z[0]) * fa[i];
            for (int k = 1; k <= R; ++k) {
                lap = fmaf(w2z[k], fa[i - k] + fa[i + k], lap);
                lap = fmaf(w2x[k], fa[i - k * sr] + fa[i + k * sr], lap);
            }
            float za = 0.f, zb = 0.f;
            for (int j = 0; j < R; ++j) {
                const long long ix = i + (j - H) * sr, iz = i + (j - H);
                za = fmaf(s[ix] * w1x[j], gu[ix], za); zb = fmaf(s[ix] * w1x[j], gv[ix], zb);
                za = fmaf(c[iz] * w1z[j], gu[iz], za); zb = fmaf(c[iz] * w1z[j], gv[iz], zb);
            }
            if (adj) tti_update_adj_point(lap, za, zb, u0[i], v0[i], um[i], vm[i], A[i], md[i], u1[i], v1[i]);
            else tti_update_point(lap, za, zb, u0[i], v0[i], um[i], vm[i], A[i], md[i], e2[i], sd[i], u1[i], v1[i]);
        }
    return 0;
}
