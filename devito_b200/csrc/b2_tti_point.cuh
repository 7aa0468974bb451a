// One-point forms of the centred-TTI Born source term (k_tti_born_src, b2_tti.cu), of the adjoint's field mix
// (k_tti_adj_mix) and of the 2-D sweep's Gz and time update (k_tti2d).
//
// `__host__ __device__` like b2_iso_point.cuh, so that tests/support/emu_points.cu can loop the SAME body on the
// CPU and compare it with the float64 reference without a GPU.
#pragma once
#include "b2_common.cuh"

#ifndef B2_HD
#define B2_HD __host__ __device__ __forceinline__
#endif

namespace b2 {

// The reference's `BornTTI` (examples/seismic/tti/operators.py:532-586): the linearised pair (du, dv) is the plain
// centred-TTI update with qu = -dm * u0.dt2 (qv = -dm * v0.dt2) added to the numerator, which is divided by
// m/dt^2 + damp/dt; u0.dt2 = (u0[t+1] - 2 u0[t] + u0[t-1]) / dt^2 is taken after the source was injected into
// u0[t+1]. The plain update of (du, dv) has already run, so this adds q / (m/dt^2 + damp/dt) to du[t+1], dv[t+1].
struct TtiBK {
    const float *__restrict__ u1;      // background levels t+1 (after the injection), t, t-1
    const float *__restrict__ u0;
    const float *__restrict__ um;
    const float *__restrict__ v1;
    const float *__restrict__ v0;
    const float *__restrict__ vm;
    float *__restrict__ du1;           // linearised pair, level t+1 (read and written)
    float *__restrict__ dv1;
    // A = 1/(m/dt^2 + damp/dt) tabulated by the fused plans; nullptr -> the denominator is computed from
    // tMD (m/dt^2 per point, array parameters) or m_dt2, and damp
    const float *__restrict__ A;
    const float *__restrict__ tMD;
    const float *__restrict__ damp;
    const float *__restrict__ dm;      // own strides and halo width
    long long sx, sy, dsx, dsy;
    int n0, n1, n2;                    // extents of the iteration box
    int o0, o1, o2;                    // array index of its first point
    int dg0, dg1, dg2;                 // index in dm of the first point (grid index + dm's halo width)
    float m_dt2, inv_dt, inv_dt2;
};

B2_HD float tti_born_q(float dmv, float f1, float f0, float fm, float inv_dt2) {
    return -dmv * ((f1 - 2.f * f0 + fm) * inv_dt2);
}

// denominator m/dt^2 + damp/dt at idx (two-pass plans, no A table)
B2_HD float tti_born_den(const TtiBK &k, long long idx) {
    const float md = k.tMD ? k.tMD[idx] : k.m_dt2;
    return md + (k.damp ? k.damp[idx] * k.inv_dt : 0.f);
}

B2_HD void tti_born_point(const TtiBK &k, int x, int y, int z) {
    const long long idx = (long long)(k.o0 + x) * k.sx + (long long)(k.o1 + y) * k.sy + (k.o2 + z);
    const long long j = (long long)(k.dg0 + x) * k.dsx + (long long)(k.dg1 + y) * k.dsy + (k.dg2 + z);
    const float dmv = k.dm[j];
    const float qu = tti_born_q(dmv, k.u1[idx], k.u0[idx], k.um[idx], k.inv_dt2);
    const float qv = tti_born_q(dmv, k.v1[idx], k.v0[idx], k.vm[idx], k.inv_dt2);
    if (k.A) {
        const float a = k.A[idx];
        k.du1[idx] += qu * a;
        k.dv1[idx] += qv * a;
    } else {
        const float den = tti_born_den(k, idx);
        k.du1[idx] += qu / den;
        k.dv1[idx] += qv / den;
    }
}

// The reference's adjoint (tti/operators.py `kernel_centered(..., forward=False)`) takes H0 = Gh(e2 p + sd r) and
// Hz = Gzz(sd p + r) with e2 = 1+2eps and sd = sqrt(1+2delta) sampled at every tap point. k_tti_adj_mix forms the
// two mixes over the whole slot (halo included), so that the forward sweep with the combination (1, 0) computes
// H0 and Hz from them.
B2_HD void tti_adj_mix_point(float e2, float sd, float p, float r, float &a, float &b) {
    a = fmaf(e2, p, sd * r);
    b = fmaf(sd, p, r);
}

// The 2-D sweep k_tti2d (b2_tti.cu), one point at a time. With D+x f, D+z f the half-node first derivatives at the Gz
// point and s, c = sin(theta), cos(theta) there, Gz = s D+x f + c D+z f (`Gzz_centered_2d`).
B2_HD float tti2d_gz_point(float s, float c, float dxf, float dzf) { return fmaf(c, dzf, s * dxf); }

// The time update of the forward pair from lap(u), Gzz(u), Gzz(v) at the point, the centre u, v at t, the level t-1
// (um, vm), A = 1/(m/dt^2 + damp/dt) and md = m/dt^2: H0 = e2 (lap - Gzz u) + sd Gzz v, Hz = sd (lap - Gzz u) + Gzz v,
// f[t+1] = f + A (md (f - f[t-1]) + H) -- the reference's (md (2 f - f[t-1]) + damp/dt f + H) / (md + damp/dt).
B2_HD void tti_update_point(float lap, float gzzu, float gzzv, float uc, float vc, float um, float vm, float A,
                            float md, float e2, float sd, float &ou, float &ov) {
    const float gh = lap - gzzu;
    const float H0 = fmaf(e2, gh, sd * gzzv);
    const float Hz = fmaf(sd, gh, gzzv);
    ou = fmaf(A, fmaf(md, uc - um, H0), uc);
    ov = fmaf(A, fmaf(md, vc - vm, Hz), vc);
}

// The adjoint pair: lap / gzza of the mix a = e2 p + sd r, gzzb of b = sd p + r (tti_adj_mix_point), the centre p, r at
// t and the level t+1 (pm, rm): H0 = lap(a) - Gzz(a), Hz = Gzz(b), f[t-1] = f + A (md (f - f[t+1]) + H).
B2_HD void tti_update_adj_point(float lapa, float gzza, float gzzb, float pc, float rc, float pm, float rm, float A,
                                float md, float &op, float &orr) {
    op = fmaf(A, fmaf(md, pc - pm, lapa - gzza), pc);
    orr = fmaf(A, fmaf(md, rc - rm, gzzb), rc);
}

}  // namespace b2
