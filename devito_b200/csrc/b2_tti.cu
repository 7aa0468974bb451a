// TTI centred forward kernels for sm_90a, scalar Thomsen parameters.
//
// Numerical spec (reference: examples/seismic/tti/operators.py:65-104 `Gzz_centered`,
// :146-183 `Gh_centered`, :186-247 `kernel_centered`, :12-39 `second_order_stencil`; the
// operation order below follows the code the reference generates for `ForwardTTI`):
//
//   D+_d f (p) = sum_j w1_d[j] f(p + (j - R/2 + 1) e_d)     half-node derivative at p + h/2
//   D-_d g (p) = sum_j w1_d[j] g(p + (j - R/2)     e_d)     half-node derivative at p - h/2
//   Gz(f)  = sin(th)cos(ph) D+_x f + sin(th)sin(ph) D+_y f + cos(th) D+_z f
//   Gzz(f) = D-_z(cos(th) Gz f) + D-_x(sin(th)cos(ph) Gz f) + D-_y(sin(th)sin(ph) Gz f)
//   H0 = (1+2 eps) (lap(u) - Gzz(u)) + sqrt(1+2 delta) Gzz(v)
//   Hz = sqrt(1+2 delta) (lap(u) - Gzz(u)) + Gzz(v)
//   u+ = ( m/dt^2 (2u - u-) + damp/dt u + H0 ) / ( m/dt^2 + damp/dt ),  v+ likewise with Hz
//
// Kernel 1 (two-pass, any even radius): pass A writes Gz(u), Gz(v) to scratch, pass B
// applies the outer derivatives + Laplacian + time update.
#include "b2_tti.cuh"
#include "b2_tti_point.cuh"
#include "b2_ptx.cuh"
#include <algorithm>
#include <cstdlib>

namespace b2 {

struct TtiK {
    const float *__restrict__ u0;
    const float *__restrict__ v0;
    const float *__restrict__ um;
    const float *__restrict__ vm;
    float *__restrict__ u1;
    float *__restrict__ v1;
    const float *__restrict__ damp;
    float *__restrict__ gzu;
    float *__restrict__ gzv;
    long long sx, sy;
    int n0, n1, n2;
    int o0, o1, o2;
    int R;
    int rx;                    // taps on dim 0: R, or 0 on the dummy dim of a 2-D plan
    float m_dt2, inv_dt;
    float cx, cy, cz;          // sin(th)cos(ph), sin(th)sin(ph), cos(th); 2-D: 0, sin(th), cos(th)
    float e2, sd;              // 1+2eps, sqrt(1+2delta)
    float w2[3][B2_MAX_RADIUS + 1];
    float w1[3][B2_MAX_RADIUS];
    // per-point coefficient tables (nullptr -> the scalars above)
    const float *__restrict__ tCx;
    const float *__restrict__ tCy;
    const float *__restrict__ tCz;
    const float *__restrict__ tE2;
    const float *__restrict__ tSD;
    const float *__restrict__ tMD;
    // ADJ: the centre of the update, p[t] / r[t] (u0 / v0 then hold the mixes of the adjoint plan)
    const float *__restrict__ pc;
    const float *__restrict__ rc;
};

// time-invariant tables for array-valued parameters (the reference hoists the same quantities:
// r2..r5 of the generated ForwardTTI for `layers-tti`)
__global__ void __launch_bounds__(256)
k_tti_tables(const float *__restrict__ vp, const float *__restrict__ eps, const float *__restrict__ delta,
             const float *__restrict__ theta, const float *__restrict__ phi, float vp_s, float eps_s,
             float delta_s, float theta_s, float phi_s, float inv_dt2, float *Cx, float *Cy, float *Cz,
             float *E2, float *SD, float *MD, size_t n, int two_d) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        const float th = theta ? theta[i] : theta_s, ph = phi ? phi[i] : phi_s;
        const float st = sinf(th), ct = cosf(th);
        // 2-D (1, x, z): `Gzz_centered_2d`'s rotation (sin th, cos th) on the plan's dims 1, 2; no Cx
        if (!two_d) Cx[i] = st * cosf(ph);
        Cy[i] = two_d ? st : st * sinf(ph);
        Cz[i] = ct;
        E2[i] = 2.0f * (eps ? eps[i] : eps_s) + 1.0f;
        SD[i] = sqrtf(2.0f * (delta ? delta[i] : delta_s) + 1.0f);
        const float v = vp ? vp[i] : vp_s;
        MD[i] = inv_dt2 / (v * v);
    }
}

// pass A: Gz over the box extended by [-R/2, R/2-1]
__global__ void __launch_bounds__(256) k_tti_gz(TtiK k) {
    const int h = k.R / 2, hx = k.rx / 2;
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (z >= k.n2 + k.R || y >= k.n1 + k.R) return;
    for (int x = blockIdx.z; x < k.n0 + k.rx; x += gridDim.z) {
        const long long idx = (long long)(k.o0 + x - hx) * k.sx + (long long)(k.o1 + y - h) * k.sy + (k.o2 + z - h);
        float dxu = 0.f, dyu = 0.f, dzu = 0.f, dxv = 0.f, dyv = 0.f, dzv = 0.f;
        for (int j = 0; j < k.R; ++j) {
            const int off = j - h + 1;
            if (k.rx) dxu = fmaf(k.w1[0][j], k.u0[idx + off * k.sx], dxu);
            dyu = fmaf(k.w1[1][j], k.u0[idx + off * k.sy], dyu);
            dzu = fmaf(k.w1[2][j], k.u0[idx + off], dzu);
            if (k.rx) dxv = fmaf(k.w1[0][j], k.v0[idx + off * k.sx], dxv);
            dyv = fmaf(k.w1[1][j], k.v0[idx + off * k.sy], dyv);
            dzv = fmaf(k.w1[2][j], k.v0[idx + off], dzv);
        }
        const float cx = k.tCx ? k.tCx[idx] : k.cx, cy = k.tCy ? k.tCy[idx] : k.cy,
                    cz = k.tCz ? k.tCz[idx] : k.cz;
        k.gzu[idx] = cx * dxu + cy * dyu + cz * dzu;
        k.gzv[idx] = cx * dxv + cy * dyv + cz * dzv;
    }
}

// ADJ: the adjoint step -- stencil inputs are the mixes a, b (combined with e2 = 1, sd = 0), the centre of the
// time update comes from p[t], r[t]
template <bool ADJ>
__global__ void __launch_bounds__(256) k_tti_update(TtiK k) {
    const int h = k.R / 2;
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (z >= k.n2 || y >= k.n1) return;
    for (int x = blockIdx.z; x < k.n0; x += gridDim.z) {
        const long long idx = (long long)(k.o0 + x) * k.sx + (long long)(k.o1 + y) * k.sy + (k.o2 + z);
        const float uc = k.u0[idx], vc = k.v0[idx];
        float lap = (k.w2[0][0] + k.w2[1][0] + k.w2[2][0]) * uc;
        for (int i = 1; i <= k.R; ++i) {
            if (k.rx) lap = fmaf(k.w2[0][i], k.u0[idx - i * k.sx] + k.u0[idx + i * k.sx], lap);
            lap = fmaf(k.w2[1][i], k.u0[idx - i * k.sy] + k.u0[idx + i * k.sy], lap);
            lap = fmaf(k.w2[2][i], k.u0[idx - i] + k.u0[idx + i], lap);
        }
        float gu = 0.f, gv = 0.f;
        for (int j = 0; j < k.R; ++j) {
            const int off = j - h;
            const long long ix = idx + off * k.sx, iy = idx + off * k.sy, iz = idx + off;
            const float cx = !k.rx ? 0.f : k.tCx ? k.tCx[ix] : k.cx, cy = k.tCy ? k.tCy[iy] : k.cy,
                        cz = k.tCz ? k.tCz[iz] : k.cz;
            if (k.rx) gu = fmaf(cx * k.w1[0][j], k.gzu[ix], gu);
            gu = fmaf(cy * k.w1[1][j], k.gzu[iy], gu);
            gu = fmaf(cz * k.w1[2][j], k.gzu[iz], gu);
            if (k.rx) gv = fmaf(cx * k.w1[0][j], k.gzv[ix], gv);
            gv = fmaf(cy * k.w1[1][j], k.gzv[iy], gv);
            gv = fmaf(cz * k.w1[2][j], k.gzv[iz], gv);
        }
        const float gh = lap - gu;                  // Gxx + Gyy applied to u
        const float md = k.tMD ? k.tMD[idx] : k.m_dt2;
        float H0, Hz, fu = uc, fv = vc;
        if constexpr (ADJ) {
            H0 = gh;
            Hz = gv;
            fu = k.pc[idx];
            fv = k.rc[idx];
        } else {
            const float e2 = k.tE2 ? k.tE2[idx] : k.e2, sd = k.tSD ? k.tSD[idx] : k.sd;
            H0 = e2 * gh + sd * gv;
            Hz = sd * gh + gv;
        }
        const float d = k.damp ? k.damp[idx] * k.inv_dt : 0.f;
        const float den = md + d;
        k.u1[idx] = (md * (2.f * fu - k.um[idx]) + d * fu + H0) / den;
        k.v1[idx] = (md * (2.f * fv - k.vm[idx]) + d * fv + Hz) / den;
    }
}

// ------------------------------------------------------------------------------------------
// Kernel 2 (fused, radius 2 or 4): one pass over HBM — 28 B/point (u,v: t r, t-1 r, t+1 w; A r).
// ------------------------------------------------------------------------------------------
// A CTA owns a (TY x 64) yz-tile and marches along x. Per x-iteration (output plane x):
//   producer warp : TMA-loads the haloed planes u[t](x+R) and v[t](x+R-1) into shared rings;
//   stage A       : all consumer threads evaluate Gz(u), Gz(v) at plane x+1 on the tile extended
//                   by [-R/2, R/2-1] in y and z (inputs from the shared u/v planes x..x+3) and
//                   store them in a 4-plane shared ring — the reference materialises these
//                   intermediates in HBM/scratch arrays (CIRE temporaries r12..r17);
//   stage B       : each thread owns 4 consecutive z points: Laplacian (x-taps from a register
//                   queue, y/z taps from the shared plane), the outer half-node derivatives of
//                   Gz from the shared Gz ring, the coupled update, 16-byte stores.
// The update uses the tabulated A = 1/(m/dt^2 + damp/dt): f+ = f + A (m/dt^2 (f - f-) + H).
__device__ __forceinline__ void f4fma_(float4 &acc, float w, const float4 &v) {
    acc.x = fmaf(w, v.x, acc.x);
    acc.y = fmaf(w, v.y, acc.y);
    acc.z = fmaf(w, v.z, acc.z);
    acc.w = fmaf(w, v.w, acc.w);
}

struct TtiFK {
    float *__restrict__ u1;
    float *__restrict__ v1;
    const float *__restrict__ um;
    const float *__restrict__ vm;
    const float *__restrict__ A;
    long long sx, sy;
    int ny, nz;
    int ox, oy, oz;
    int xlo, xcount, lx;
    int ntz, nty;
    int slot0;
    float m_dt2;
    float cx, cy, cz;          // sin(th)cos(ph), sin(th)sin(ph), cos(th)
    float e2, sd;              // 1+2eps, sqrt(1+2delta)
    float w2x[5], w2y[5], w2z[5];
    float w1x[4], w1y[4], w1z[4];      // already multiplied by cx, cy, cz
    // {w, w} pairs for the fp32 pair arithmetic of k_tti_ws (b2_ptx.cuh)
    float2 p_w2x[5], p_w2y[5], p_w1x[4], p_w1y[4];
    float2 p_wc, p_e2, p_sd, p_mdt2;
    // array-valued parameters (k_tti_fused<.., ARR = true>): per-point tables; w1x/w1y/w1z then hold the RAW weights
    const float *__restrict__ tCx;
    const float *__restrict__ tCy;
    const float *__restrict__ tCz;
    const float *__restrict__ tE2;
    const float *__restrict__ tSD;
    const float *__restrict__ tMD;
    int hint;                  // != 0: once-per-CTA table reads bypass L1 allocation
    // ADJ: the centre of the update, p[t] / r[t]; the tensor maps then cover the mixes of the adjoint plan
    const float *__restrict__ pc;
    const float *__restrict__ rc;
};

// ARR: the array-parameter sweep, which stages the rotation-factor tiles through shared memory by TMA (a ring of
// three tables per plane, paid for with one batch less of u / v prefetch)
template <int R, int TY, bool ARR = false>
struct TtiCfg {
    static constexpr int D = ARR ? 2 : 3;            // batches the producer may run ahead of the slowest consumer
    static constexpr int H = R / 2;
    static constexpr int TZ4 = 16, TZ = 64, RZ = 4;
    static constexpr int PR = TY + 2 * R;            // rows of a u/v plane box
    static constexpr int BZ = TZ + 2 * RZ;           // 72
    static constexpr int GR = TY + R;                // rows of a Gz plane: [-H, TY+H-1] (+pad)
    static constexpr int NUU = R + D;                // u planes x..x+R, + (D-1) in flight
    static constexpr int NUV = R + D - 1;            // v planes x..x+R-1, + (D-1) in flight
    static constexpr int NG = R + 1;                 // Gz planes x-H..x+H-1, +1 so that stage A of the
                                                     // next iteration never overwrites a plane still read
    static constexpr int NB = 4;                     // barrier ring
    static constexpr int PLANE = ((PR * BZ + 31) / 32) * 32;
    static constexpr int GPLANE = ((GR * BZ + 31) / 32) * 32;
    static constexpr int NCT = TY * TZ4;             // consumer threads
    static constexpr int NCW = NCT / 32;
    static constexpr int GGROUPS = (TY + R - 1) * (BZ / 4);   // float4 groups of the extended tile
    // factor-tile ring: stage A's plane x+H-1 and the planes down to x for stage B (H live planes + the one in flight)
    static constexpr int NCT_PLANES = ARR ? H + 1 : 0;
    static constexpr size_t SMEM = (size_t)((NUU + NUV) * PLANE + (2 * NG + 3 * NCT_PLANES) * GPLANE) * 4 + 2 * NB * 8 + 128;
};

// ARR = true: array-valued vp / epsilon / delta / theta / phi (`layers-tti`). The rotation factors are sampled where
// the reference samples them — at the Gz point inside Gz, at the shifted point in the outer derivative — from the
// per-point tables of k_tti_tables. cx, cy, cz of stage A's plane arrive by TMA with the u / v batch (boxes of the
// extended tile, zero-filled outside the array) in a ring of R/2 + 1 planes, so stage A has no global loads at all;
// stage B keeps cx of its own column in a register queue along x and reads cy of the R rows / cz of the z segment
// around its four points from the ring's plane x. (1+2eps), sqrt(1+2delta), m/dt^2 and A come with u[t-1], v[t-1]
// at the top of the iteration. 52 B/point instead of 28.
// ADJ: the adjoint step. The tensor maps cover the mixes a = e2 p + sd r, b = sd p + r, combined with e2 = 1, sd = 0;
// the centre of the time update is loaded from p[t], r[t] (with ARR in place of the e2 / sd tables, so the array
// kernel moves the same bytes as the forward one).
template <int R, int TY, bool ARR, bool ADJ = false>
__global__ void __launch_bounds__(TY * 16 + 32, 1)
k_tti_fused(const __grid_constant__ CUtensorMap tm_u, const __grid_constant__ CUtensorMap tm_v,
            const __grid_constant__ CUtensorMap tm_cx, const __grid_constant__ CUtensorMap tm_cy,
            const __grid_constant__ CUtensorMap tm_cz, const TtiFK k) {
    using C = TtiCfg<R, TY, ARR>;
    constexpr int D = C::D;
    constexpr int NCP = ARR ? C::NCT_PLANES : 1;    // planes of the factor-tile ring
    constexpr int H = C::H, TZ = C::TZ, RZ = C::RZ, BZ = C::BZ, PR = C::PR, GR = C::GR;
    constexpr int NUU = C::NUU, NUV = C::NUV, NG = C::NG, NB = C::NB;
    constexpr int PLANE = C::PLANE, GPLANE = C::GPLANE, NCT = C::NCT, NCW = C::NCW;
    constexpr int PRE = 2 * R;                      // priming iterations before the first output

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *s_u = reinterpret_cast<float *>(smem_raw);
    float *s_v = s_u + NUU * PLANE;
    float *s_gu = s_v + NUV * PLANE;
    float *s_gv = s_gu + NG * GPLANE;
    float *s_c = s_gv + NG * GPLANE;                // ARR: [plane mod NCP][cx, cy, cz][GPLANE]
    uint64_t *full = reinterpret_cast<uint64_t *>(s_c + 3 * C::NCT_PLANES * GPLANE);
    uint64_t *empty = full + NB;

    int b = blockIdx.x;
    const int iz = b % k.ntz;
    b /= k.ntz;
    const int iy = b % k.nty;
    const int ix = b / k.nty;
    const int z0 = iz * TZ, y0 = iy * TY;
    const int xs = k.xlo + ix * k.lx;
    const int xe = min(xs + k.lx, k.xlo + k.xcount);
    const int NIT = (xe - xs) + PRE;                // iterations: x = xs - PRE + it

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;

    if (tid == 0) {
        for (int i = 0; i < NB; ++i) {
            b2ptx::mbar_init(&full[i], 1);
            b2ptx::mbar_init(&empty[i], NCW);
        }
        b2ptx::fence_mbar_init();
    }
    __syncthreads();

    if (warp == NCW) {
        if (lane == 0) {
            b2ptx::tma_prefetch_desc(&tm_u);
            b2ptx::tma_prefetch_desc(&tm_v);
            // batch `it` carries u plane (x+R) and v plane (x+R-1) of iteration x = xs-PRE+it.
            // Its slots were last read in iteration it-3 (u plane x-3+R... see DESIGN.md §3.3).
            if constexpr (ARR) {
                b2ptx::tma_prefetch_desc(&tm_cx);
                b2ptx::tma_prefetch_desc(&tm_cy);
                b2ptx::tma_prefetch_desc(&tm_cz);
            }
            for (int it = 0; it < NIT; ++it) {
                const int x = xs - PRE + it;
                if (it >= D) {
                    const int w = it - D;
                    b2ptx::mbar_wait(&empty[w % NB], (w / NB) & 1);
                }
                const int pu = x + R;                    // u plane index (relative to origin)
                const int pv = x + R - 1;
                const bool hv = pv >= xs - (R - 1);      // v planes below xs-R+1 are never used
                // ARR: factor tiles of stage A's plane x+H-1; their slot held plane x+H-1-NCP, last read (by stage B) in
                // iteration it-2
                const bool hc = ARR && (x + H - 1 >= xs - H);
                b2ptx::mbar_arrive_expect_tx(&full[it % NB], (uint32_t)(PR * BZ * 4) * (hv ? 2u : 1u) +
                                                                 (hc ? (uint32_t)(3 * C::GR * BZ * 4) : 0u));
                b2ptx::tma_load_4d(s_u + ((pu % NUU + NUU) % NUU) * PLANE, &tm_u, &full[it % NB],
                                   k.oz + z0 - RZ, k.oy + y0 - R, k.ox + pu, k.slot0);
                if (hv)
                    b2ptx::tma_load_4d(s_v + ((pv % NUV + NUV) % NUV) * PLANE, &tm_v, &full[it % NB],
                                       k.oz + z0 - RZ, k.oy + y0 - R, k.ox + pv, k.slot0);
                if constexpr (ARR) {
                    if (hc) {
                        float *dst = s_c + (((x + H - 1) % NCP + NCP) % NCP) * 3 * GPLANE;
                        b2ptx::tma_load_4d(dst, &tm_cx, &full[it % NB], k.oz + z0 - RZ, k.oy + y0 - H, k.ox + x + H - 1, 0);
                        b2ptx::tma_load_4d(dst + GPLANE, &tm_cy, &full[it % NB], k.oz + z0 - RZ, k.oy + y0 - H, k.ox + x + H - 1, 0);
                        b2ptx::tma_load_4d(dst + 2 * GPLANE, &tm_cz, &full[it % NB], k.oz + z0 - RZ, k.oy + y0 - H, k.ox + x + H - 1, 0);
                    }
                }
            }
        }
        return;
    }

    // ---------------- consumers ----------------
    const int ty = tid / 16, tz4 = tid % 16;
    const int gy = y0 + ty, gz = z0 + 4 * tz4;
    const bool yok = gy < k.ny;
    const int zcnt = yok ? min(max(k.nz - gz, 0), 4) : 0;
    const int my_off = (ty + R) * BZ + RZ + 4 * tz4;          // own column in a u/v plane box
    const int my_goff = (ty + H) * BZ + RZ + 4 * tz4;         // own column in a Gz plane
    const long long gidx0 = (long long)(k.oy + gy) * k.sy + (k.oz + gz);

    float4 uq[2 * R + 1];
#pragma unroll
    for (int i = 0; i <= 2 * R; ++i) uq[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    const float wc = k.w2x[0] + k.w2y[0] + k.w2z[0];

    // stage-A work items of this thread: (field, float4-group) pairs of the tile extended by
    // [-H, H-1], dealt round-robin; packed as poff | fv<<16 | has_left<<17 | has_right<<18 | valid<<19
    constexpr int NTASK = (2 * C::GGROUPS + NCT - 1) / NCT;
    int tdesc[NTASK];
#pragma unroll
    for (int t = 0; t < NTASK; ++t) {
        const int task = tid + t * NCT;
        const bool valid = task < 2 * C::GGROUPS;
        const bool fv = task >= C::GGROUPS;
        const int grp = fv ? task - C::GGROUPS : task;
        const int gr = grp / (BZ / 4), gc = grp - gr * (BZ / 4);
        const int poff = (gr + R - H) * BZ + 4 * gc;
        tdesc[t] = poff | (fv ? 1 << 16 : 0) | (gc > 0 ? 1 << 17 : 0) | (gc < BZ / 4 - 1 ? 1 << 18 : 0) |
                   (valid ? 1 << 19 : 0);
    }
    float4 cxq[ARR ? R : 1];           // ARR: cx of the own column at planes x-H .. x+H-1
    if constexpr (ARR) {
#pragma unroll
        for (int i = 0; i < R; ++i) cxq[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    long long gi = (long long)(k.ox + xs - PRE) * k.sx + gidx0;

    // ring positions of plane x (updated incrementally; x starts at xs - PRE)
    int iu = ((xs - PRE) % NUU + NUU) % NUU, iv = ((xs - PRE) % NUV + NUV) % NUV,
        ig = ((xs - PRE) % NG + NG) % NG;
    int ic = ((xs - PRE) % NCP + NCP) % NCP;        // ARR: ring slot of factor plane x
    auto wrap = [](int v, int n) { return v >= n ? v - n : v; };
    // per-point tables read once per CTA: optionally kept out of L1
    const bool stream_hint = ARR && k.hint != 0;
    auto ldt = [&](const float *q) -> float4 {
        float4 r;
        if (stream_hint)
            asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
                         : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(q));
        else
            r = __ldg(reinterpret_cast<const float4 *>(q));
        return r;
    };

    for (int it = 0; it < NIT; ++it) {
        const int x = xs - PRE + it;
        // u[t-1], v[t-1], A of the output plane: issued first so that stage A and most of stage B
        // hide their latency (loads issued one statement before use stall the consumers)
        float4 pu = make_float4(0, 0, 0, 0), pv = pu, pa = pu;
        if (x >= xs && zcnt > 0) {
            if (zcnt == 4) {
                if constexpr (ARR) {
                    pu = ldt(k.um + gi); pv = ldt(k.vm + gi); pa = ldt(k.A + gi);
                } else {
                    pu = *reinterpret_cast<const float4 *>(k.um + gi);
                    pv = *reinterpret_cast<const float4 *>(k.vm + gi);
                    pa = *reinterpret_cast<const float4 *>(k.A + gi);
                }
            } else {
                float t[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
                for (int i = 0; i < zcnt; ++i) { t[i] = k.um[gi + i]; t[4 + i] = k.vm[gi + i]; t[8 + i] = k.A[gi + i]; }
                pu = make_float4(t[0], t[1], t[2], t[3]);
                pv = make_float4(t[4], t[5], t[6], t[7]);
                pa = make_float4(t[8], t[9], t[10], t[11]);
            }
        }
        float4 pcn = make_float4(0, 0, 0, 0), rcn = pcn;      // ADJ: p[t], r[t] at the four points
        if constexpr (ADJ && !ARR) {
            if (x >= xs && zcnt > 0) {
                if (zcnt == 4) {
                    pcn = *reinterpret_cast<const float4 *>(k.pc + gi);
                    rcn = *reinterpret_cast<const float4 *>(k.rc + gi);
                } else {
                    float t[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                    for (int i = 0; i < zcnt; ++i) { t[i] = k.pc[gi + i]; t[4 + i] = k.rc[gi + i]; }
                    pcn = make_float4(t[0], t[1], t[2], t[3]);
                    rcn = make_float4(t[4], t[5], t[6], t[7]);
                }
            }
        }
        float4 pe2 = pu, psd = pu, pmd = pu;
        if constexpr (ARR) {
            // the 16-byte table reads stay inside the array for every gz < nz (az % 4 == 0, >= 4 cells of halo)
            if (x >= xs && zcnt > 0) {
                if constexpr (!ADJ) {
                    pe2 = ldt(k.tE2 + gi);
                    psd = ldt(k.tSD + gi);
                }
                pmd = ldt(k.tMD + gi);
            }
#pragma unroll
            for (int i = 0; i < R - 1; ++i) cxq[i] = cxq[i + 1];
        }
        b2ptx::mbar_wait(&full[it % NB], (it / NB) & 1);
        if constexpr (ARR) {                         // own column of the cx tile that just landed (plane x+H-1)
            if (x + H - 1 >= xs - H)
                cxq[R - 1] = b2ptx::lds128(s_c + wrap(ic + H - 1, NCP) * 3 * GPLANE + my_goff);
        }

        // queue: uq[i] = u plane x - R + i   (newest = x + R)
#pragma unroll
        for (int i = 0; i < 2 * R; ++i) uq[i] = uq[i + 1];
        uq[2 * R] = b2ptx::lds128(s_u + wrap(iu + R, NUU) * PLANE + my_off);

        // ---- stage A: Gz(u), Gz(v) at plane g = x + H - 1 (needs f planes x .. x+R-1) ----
        // Work items are (field, float4-group) pairs of the tile extended by [-H, H-1], dealt
        // round-robin so that no thread gets more than one item above the average.
        if (x + H - 1 >= xs - H) {
            const float *up[R], *vp[R];
#pragma unroll
            for (int j = 0; j < R; ++j) {
                up[j] = s_u + wrap(iu + j, NUU) * PLANE;
                vp[j] = s_v + wrap(iv + j, NUV) * PLANE;
            }
            const int sgz = wrap(ig + H - 1, NG) * GPLANE;
#pragma unroll
            for (int t = 0; t < NTASK; ++t) {
                const int d = tdesc[t];
                if (!(d & (1 << 19))) continue;
                const bool fv = d & (1 << 16);
                const int poff = d & 0xffff;
                float4 rr = make_float4(0, 0, 0, 0);
                float4 c4x = rr, c4y = rr, c4z = rr, ry = rr, rz = rr;   // ARR: factors at the Gz point; D+y, D+z kept apart
                if constexpr (ARR) {
                    const float *cs = s_c + wrap(ic + H - 1, NCP) * 3 * GPLANE + poff - (R - H) * BZ;
                    c4x = b2ptx::lds128(cs);
                    c4y = b2ptx::lds128(cs + GPLANE);
                    c4z = b2ptx::lds128(cs + 2 * GPLANE);
                }
#pragma unroll
                for (int j = 0; j < R; ++j) {                // x taps
                    const float4 a = b2ptx::lds128((fv ? vp[j] : up[j]) + poff);
                    f4fma_(rr, k.w1x[j], a);
                }
                const float *fc = (fv ? vp[H - 1] : up[H - 1]) + poff;     // plane g, this point
#pragma unroll
                for (int j = 0; j < R; ++j) {                // y taps
                    const float4 a = b2ptx::lds128(fc + (j - H + 1) * BZ);
                    f4fma_(ARR ? ry : rr, k.w1y[j], a);
                }
                {                                            // z taps: segment [-4, 8) around the group
                    const float4 l = (d & (1 << 17)) ? b2ptx::lds128(fc - 4) : make_float4(0, 0, 0, 0);
                    const float4 c = b2ptx::lds128(fc);
                    const float4 r = (d & (1 << 18)) ? b2ptx::lds128(fc + 4) : make_float4(0, 0, 0, 0);
                    const float zz[12] = {l.x, l.y, l.z, l.w, c.x, c.y, c.z, c.w, r.x, r.y, r.z, r.w};
                    float4 &az_ = ARR ? rz : rr;
#pragma unroll
                    for (int j = 0; j < R; ++j) {
                        const int o = 4 + j - H + 1;
                        az_.x = fmaf(k.w1z[j], zz[o + 0], az_.x); az_.y = fmaf(k.w1z[j], zz[o + 1], az_.y);
                        az_.z = fmaf(k.w1z[j], zz[o + 2], az_.z); az_.w = fmaf(k.w1z[j], zz[o + 3], az_.w);
                    }
                }
                if constexpr (ARR) {                         // Gz = cx D+x + cy D+y + cz D+z with the factors of this point
                    rr.x = fmaf(c4z.x, rz.x, fmaf(c4y.x, ry.x, c4x.x * rr.x));
                    rr.y = fmaf(c4z.y, rz.y, fmaf(c4y.y, ry.y, c4x.y * rr.y));
                    rr.z = fmaf(c4z.z, rz.z, fmaf(c4y.z, ry.z, c4x.z * rr.z));
                    rr.w = fmaf(c4z.w, rz.w, fmaf(c4y.w, ry.w, c4x.w * rr.w));
                }
                *reinterpret_cast<float4 *>((fv ? s_gv : s_gu) + sgz + poff - (R - H) * BZ) = rr;
            }
        }
        // Gz written by all threads must be visible before its y/z neighbours are read; one barrier
        // per iteration among the consumer warps (the Gz ring has R+1 planes so that the next
        // iteration's stage A never overwrites a plane that stage B of this one still reads).
        asm volatile("bar.sync 1, %0;" ::"n"(NCT) : "memory");

        // ---- stage B: output plane x ----
        if (x >= xs) {
            if constexpr (ADJ && ARR) {              // in place of the e2 / sd tables; issued here, where registers are free
                if (zcnt > 0) {
                    pcn = ldt(k.pc + gi);
                    rcn = ldt(k.rc + gi);
                }
            }
            // ARR: cy at the R rows and cz on the z segment around the four points, issued ahead of their use
            float4 cyq[ARR ? R : 1];
            float czr[ARR ? 12 : 1];
            if constexpr (ARR) {                   // plane x of the factor ring: rows y-H+j of cy, z segment of cz
                const float *cb = s_c + ic * 3 * GPLANE + my_goff;
#pragma unroll
                for (int j = 0; j < R; ++j) cyq[j] = b2ptx::lds128(cb + GPLANE + (j - H) * BZ);
                const float4 l = b2ptx::lds128(cb + 2 * GPLANE - 4), cc = b2ptx::lds128(cb + 2 * GPLANE),
                             r = b2ptx::lds128(cb + 2 * GPLANE + 4);
                czr[0] = l.x; czr[1] = l.y; czr[2] = l.z; czr[3] = l.w; czr[4] = cc.x; czr[5] = cc.y; czr[6] = cc.z;
                czr[7] = cc.w; czr[8] = r.x; czr[9] = r.y; czr[10] = r.z; czr[11] = r.w;
            }
            const float *cpl = s_u + iu * PLANE + my_off;   // u plane x, own column
            const float4 c = uq[R];
            const float4 vcn = b2ptx::lds128(s_v + iv * PLANE + my_off);
            // Laplacian of u
            float4 lap = make_float4(wc * c.x, wc * c.y, wc * c.z, wc * c.w);
            {
                const float4 l = b2ptx::lds128(cpl - 4), r = b2ptx::lds128(cpl + 4);
                float zr[12] = {l.x, l.y, l.z, l.w, c.x, c.y, c.z, c.w, r.x, r.y, r.z, r.w};
#pragma unroll
                for (int i = 1; i <= R; ++i) {
                    lap.x = fmaf(k.w2z[i], zr[4 - i] + zr[4 + i], lap.x);
                    lap.y = fmaf(k.w2z[i], zr[5 - i] + zr[5 + i], lap.y);
                    lap.z = fmaf(k.w2z[i], zr[6 - i] + zr[6 + i], lap.z);
                    lap.w = fmaf(k.w2z[i], zr[7 - i] + zr[7 + i], lap.w);
                }
            }
#pragma unroll
            for (int i = 1; i <= R; ++i) {
                const float4 a = b2ptx::lds128(cpl - i * BZ), bb = b2ptx::lds128(cpl + i * BZ);
                lap.x = fmaf(k.w2y[i], a.x + bb.x, lap.x); lap.y = fmaf(k.w2y[i], a.y + bb.y, lap.y);
                lap.z = fmaf(k.w2y[i], a.z + bb.z, lap.z); lap.w = fmaf(k.w2y[i], a.w + bb.w, lap.w);
            }
#pragma unroll
            for (int i = 1; i <= R; ++i) {
                const float4 a = uq[R - i], bb = uq[R + i];
                lap.x = fmaf(k.w2x[i], a.x + bb.x, lap.x); lap.y = fmaf(k.w2x[i], a.y + bb.y, lap.y);
                lap.z = fmaf(k.w2x[i], a.z + bb.z, lap.z); lap.w = fmaf(k.w2x[i], a.w + bb.w, lap.w);
            }
            // Gzz(u), Gzz(v): outer half-node derivatives of Gz at offsets -H..H-1
            float4 zu4 = make_float4(0, 0, 0, 0), zv4 = zu4;
#pragma unroll
            for (int j = 0; j < R; ++j) {                       // x direction: planes x-H+j
                int sl_ = ig - H + j;
                sl_ = sl_ < 0 ? sl_ + NG : (sl_ >= NG ? sl_ - NG : sl_);
                const int so_ = sl_ * GPLANE + my_goff;
                const float4 a = b2ptx::lds128(s_gu + so_), bb = b2ptx::lds128(s_gv + so_);
                const float w = k.w1x[j];
                if constexpr (ARR) {
                    const float4 q = cxq[j];
                    const float wx = q.x * w, wy = q.y * w, wz = q.z * w, ww = q.w * w;
                    zu4.x = fmaf(wx, a.x, zu4.x); zu4.y = fmaf(wy, a.y, zu4.y); zu4.z = fmaf(wz, a.z, zu4.z); zu4.w = fmaf(ww, a.w, zu4.w);
                    zv4.x = fmaf(wx, bb.x, zv4.x); zv4.y = fmaf(wy, bb.y, zv4.y); zv4.z = fmaf(wz, bb.z, zv4.z); zv4.w = fmaf(ww, bb.w, zv4.w);
                } else {
                    zu4.x = fmaf(w, a.x, zu4.x); zu4.y = fmaf(w, a.y, zu4.y); zu4.z = fmaf(w, a.z, zu4.z); zu4.w = fmaf(w, a.w, zu4.w);
                    zv4.x = fmaf(w, bb.x, zv4.x); zv4.y = fmaf(w, bb.y, zv4.y); zv4.z = fmaf(w, bb.z, zv4.z); zv4.w = fmaf(w, bb.w, zv4.w);
                }
            }
            const float *gpu_ = s_gu + ig * GPLANE + my_goff;
            const float *gpv_ = s_gv + ig * GPLANE + my_goff;
#pragma unroll
            for (int j = 0; j < R; ++j) {                       // y direction: rows y-H+j
                const float4 a = b2ptx::lds128(gpu_ + (j - H) * BZ), bb = b2ptx::lds128(gpv_ + (j - H) * BZ);
                const float w = k.w1y[j];
                if constexpr (ARR) {
                    const float4 q = cyq[j];
                    const float wx = q.x * w, wy = q.y * w, wz = q.z * w, ww = q.w * w;
                    zu4.x = fmaf(wx, a.x, zu4.x); zu4.y = fmaf(wy, a.y, zu4.y); zu4.z = fmaf(wz, a.z, zu4.z); zu4.w = fmaf(ww, a.w, zu4.w);
                    zv4.x = fmaf(wx, bb.x, zv4.x); zv4.y = fmaf(wy, bb.y, zv4.y); zv4.z = fmaf(wz, bb.z, zv4.z); zv4.w = fmaf(ww, bb.w, zv4.w);
                } else {
                    zu4.x = fmaf(w, a.x, zu4.x); zu4.y = fmaf(w, a.y, zu4.y); zu4.z = fmaf(w, a.z, zu4.z); zu4.w = fmaf(w, a.w, zu4.w);
                    zv4.x = fmaf(w, bb.x, zv4.x); zv4.y = fmaf(w, bb.y, zv4.y); zv4.z = fmaf(w, bb.z, zv4.z); zv4.w = fmaf(w, bb.w, zv4.w);
                }
            }
            {
                const float4 lu = b2ptx::lds128(gpu_ - 4), cu = b2ptx::lds128(gpu_), ru_ = b2ptx::lds128(gpu_ + 4);
                const float4 lv = b2ptx::lds128(gpv_ - 4), cv = b2ptx::lds128(gpv_), rv_ = b2ptx::lds128(gpv_ + 4);
                float au[12] = {lu.x, lu.y, lu.z, lu.w, cu.x, cu.y, cu.z, cu.w, ru_.x, ru_.y, ru_.z, ru_.w};
                float av[12] = {lv.x, lv.y, lv.z, lv.w, cv.x, cv.y, cv.z, cv.w, rv_.x, rv_.y, rv_.z, rv_.w};
#pragma unroll
                for (int j = 0; j < R; ++j) {                   // z direction: offsets j-H
                    const float w = k.w1z[j];
                    const int o = 4 + j - H;
                    if constexpr (ARR) {
                        zu4.x = fmaf(czr[o + 0] * w, au[o + 0], zu4.x); zu4.y = fmaf(czr[o + 1] * w, au[o + 1], zu4.y);
                        zu4.z = fmaf(czr[o + 2] * w, au[o + 2], zu4.z); zu4.w = fmaf(czr[o + 3] * w, au[o + 3], zu4.w);
                        zv4.x = fmaf(czr[o + 0] * w, av[o + 0], zv4.x); zv4.y = fmaf(czr[o + 1] * w, av[o + 1], zv4.y);
                        zv4.z = fmaf(czr[o + 2] * w, av[o + 2], zv4.z); zv4.w = fmaf(czr[o + 3] * w, av[o + 3], zv4.w);
                    } else {
                        zu4.x = fmaf(w, au[o + 0], zu4.x); zu4.y = fmaf(w, au[o + 1], zu4.y);
                        zu4.z = fmaf(w, au[o + 2], zu4.z); zu4.w = fmaf(w, au[o + 3], zu4.w);
                        zv4.x = fmaf(w, av[o + 0], zv4.x); zv4.y = fmaf(w, av[o + 1], zv4.y);
                        zv4.z = fmaf(w, av[o + 2], zv4.z); zv4.w = fmaf(w, av[o + 3], zv4.w);
                    }
                }
            }
            float4 ou, ov;
#define B2_TTI_UPD(F)                                                              \
            {                                                                      \
                const float gh = lap.F - zu4.F;                                    \
                const float md_ = ARR ? pmd.F : k.m_dt2;                           \
                if constexpr (ADJ) {                                               \
                    ou.F = fmaf(pa.F, fmaf(md_, pcn.F - pu.F, gh), pcn.F);         \
                    ov.F = fmaf(pa.F, fmaf(md_, rcn.F - pv.F, zv4.F), rcn.F);      \
                } else {                                                           \
                const float e2_ = ARR ? pe2.F : k.e2, sd_ = ARR ? psd.F : k.sd;    \
                const float H0 = fmaf(e2_, gh, sd_ * zv4.F);                       \
                const float Hz = fmaf(sd_, gh, zv4.F);                             \
                ou.F = fmaf(pa.F, fmaf(md_, c.F - pu.F, H0), c.F);                 \
                ov.F = fmaf(pa.F, fmaf(md_, vcn.F - pv.F, Hz), vcn.F);             \
                }                                                                  \
            }
            B2_TTI_UPD(x) B2_TTI_UPD(y) B2_TTI_UPD(z) B2_TTI_UPD(w)
#undef B2_TTI_UPD
            if (zcnt == 4) {
                *reinterpret_cast<float4 *>(k.u1 + gi) = ou;
                *reinterpret_cast<float4 *>(k.v1 + gi) = ov;
            } else if (zcnt > 0) {
                const float tu[4] = {ou.x, ou.y, ou.z, ou.w}, tv[4] = {ov.x, ov.y, ov.z, ov.w};
                for (int i = 0; i < zcnt; ++i) { k.u1[gi + i] = tu[i]; k.v1[gi + i] = tv[i]; }
            }
        }
        __syncwarp();
        if (lane == 0) b2ptx::mbar_arrive(&empty[it % NB]);
        ic = wrap(ic + 1, NCP);
        iu = wrap(iu + 1, NUU);
        iv = wrap(iv + 1, NUV);
        ig = wrap(ig + 1, NG);
        gi += k.sx;
    }
}

// ------------------------------------------------------------------------------------------
// Kernel 3 (fused, warp-specialised, radius 4): same data flow as k_tti_fused, reorganised so that
// every x-direction tap comes from registers and the extended-tile (halo) part of Gz is produced
// by helper warps instead of unbalancing the main warps.
//   warpgroups 0-2 (384 threads): one float4 column each (24 x 64 tile). Register queues hold the
//       x-history of u (9 planes), v (4 planes) and of the thread's own Gz(u), Gz(v) (4 planes):
//       D+x, the x-taps of the Laplacian and D-x cost no shared-memory traffic at all.
//   warpgroup 3: warp 0 = TMA producer; warps 1-3 = helpers computing Gz on the 102 halo groups of
//       the extended tile (rows -2,-1,+TY and the float4 columns left/right of the tile).
// 512 threads x 128 registers; the main path fits in 128 registers (ptxas: a few bytes spilled), so no
// `setmaxnreg` rebalancing is needed.
// ------------------------------------------------------------------------------------------
template <int TY>
struct TtiWsCfg {
    static constexpr int R = 4, H = 2, TZ = 64, RZ = 4;
    static constexpr int PR = TY + 2 * R, BZ = TZ + 2 * RZ, GR = TY + R;
    static constexpr int NUU = R + 3, NUV = R + 3, NG = 4, NB = 4;
    static constexpr int PLANE = ((PR * BZ + 31) / 32) * 32;
    static constexpr int GPLANE = ((GR * BZ + 31) / 32) * 32;
    static constexpr int NMAIN = TY * 16;               // 384 for TY = 24
    static constexpr int NHELP = 96;
    static constexpr int NHALO = 3 * (BZ / 4) + 2 * TY; // 54 + 48
    static constexpr size_t SMEM = (size_t)((NUU + NUV) * PLANE + 2 * NG * GPLANE) * 4 + 2 * NB * 8 + 128;
};

template <int TY>
__global__ void __launch_bounds__(TY * 16 + 128, 1)
k_tti_ws(const __grid_constant__ CUtensorMap tm_u, const __grid_constant__ CUtensorMap tm_v, const TtiFK k) {
    using C = TtiWsCfg<TY>;
    constexpr int R = 4, H = 2, TZ = C::TZ, RZ = C::RZ, BZ = C::BZ, PR = C::PR;
    constexpr int NUU = C::NUU, NUV = C::NUV, NG = C::NG, NB = C::NB;
    constexpr int PLANE = C::PLANE, GPLANE = C::GPLANE, NMAIN = C::NMAIN;
    constexpr int PRE = 2 * R;
    constexpr int NSYNC = NMAIN + C::NHELP;            // threads in the per-iteration barrier
    constexpr int NARR = NMAIN / 32 + C::NHELP / 32;   // warps releasing a stage

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *s_u = reinterpret_cast<float *>(smem_raw);
    float *s_v = s_u + NUU * PLANE;
    float *s_gu = s_v + NUV * PLANE;
    float *s_gv = s_gu + NG * GPLANE;
    uint64_t *full = reinterpret_cast<uint64_t *>(s_gv + NG * GPLANE);
    uint64_t *empty = full + NB;

    int b = blockIdx.x;
    const int iz = b % k.ntz;
    b /= k.ntz;
    const int iy = b % k.nty;
    const int ix = b / k.nty;
    const int z0 = iz * TZ, y0 = iy * TY;
    const int xs = k.xlo + ix * k.lx;
    const int xe = min(xs + k.lx, k.xlo + k.xcount);
    const int NIT = (xe - xs) + PRE;

    const int tid = threadIdx.x;
    const int lane = tid & 31;

    if (tid == 0) {
        for (int i = 0; i < NB; ++i) {
            b2ptx::mbar_init(&full[i], 1);
            b2ptx::mbar_init(&empty[i], NARR);
        }
        b2ptx::fence_mbar_init();
    }
    __syncthreads();
    auto wrap = [](int v, int n) { return v >= n ? v - n : v; };

    if (tid >= NMAIN) {
        // =================== warpgroup 3: producer + helpers ===================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
        const int wtid = tid - NMAIN;
        if (wtid < 32) {
            if (lane == 0) {
                b2ptx::tma_prefetch_desc(&tm_u);
                b2ptx::tma_prefetch_desc(&tm_v);
                for (int it = 0; it < NIT; ++it) {
                    const int x = xs - PRE + it;
                    if (it >= 3) {
                        const int w = it - 3;
                        b2ptx::mbar_wait(&empty[w % NB], (w / NB) & 1);
                    }
                    const int pu = x + R, pv = x + R;          // helpers run one plane ahead: v too
                    const bool hv = pv >= xs - (R - 1);
                    b2ptx::mbar_arrive_expect_tx(&full[it % NB], (uint32_t)(PR * BZ * 4) * (hv ? 2u : 1u));
                    b2ptx::tma_load_4d(s_u + ((pu % NUU + NUU) % NUU) * PLANE, &tm_u, &full[it % NB],
                                       k.oz + z0 - RZ, k.oy + y0 - R, k.ox + pu, k.slot0);
                    if (hv)
                        b2ptx::tma_load_4d(s_v + ((pv % NUV + NUV) % NUV) * PLANE, &tm_v, &full[it % NB],
                                           k.oz + z0 - RZ, k.oy + y0 - R, k.ox + pv, k.slot0);
                }
            }
            return;
        }
        // ---- helpers: Gz on the halo groups of the extended tile ----
        const int hid = wtid - 32;
        int hoff[2], hflag[2];
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            const int g = hid + t * C::NHELP;
            int gr, gc;
            if (g < 3 * (BZ / 4)) {
                const int rr = g / (BZ / 4);
                gr = rr < 2 ? rr : TY + 2;
                gc = g - rr * (BZ / 4);
            } else {
                const int kx = g - 3 * (BZ / 4);
                gr = 2 + (kx >> 1);
                gc = (kx & 1) ? BZ / 4 - 1 : 0;
            }
            hoff[t] = (gr + R - H) * BZ + 4 * gc;
            hflag[t] = (g < C::NHALO ? 1 : 0) | (gc > 0 ? 2 : 0) | (gc < BZ / 4 - 1 ? 4 : 0);
        }
        int iu = ((xs - PRE) % NUU + NUU) % NUU, iv = ((xs - PRE) % NUV + NUV) % NUV,
            ig = ((xs - PRE) % NG + NG) % NG;
        // Helpers run ONE PLANE AHEAD of the main warps: in iteration `it` they first join the
        // barrier (which certifies their halo of plane x+1, computed last iteration), then produce
        // the halo of plane x+2 while the main warps do stage B — they never sit on the critical path.
        for (int it = 0; it < NIT; ++it) {
            const int x = xs - PRE + it;
            b2ptx::mbar_wait(&full[it % NB], (it / NB) & 1);
            asm volatile("bar.sync 1, %0;" ::"n"(NSYNC) : "memory");
            if (x + 2 >= xs - H) {
                const int sgz = wrap(ig + 2, NG) * GPLANE;
#pragma unroll
                for (int t = 0; t < 2; ++t) {
                    if (!(hflag[t] & 1)) continue;
                    const int poff = hoff[t];
#pragma unroll
                    for (int f = 0; f < 2; ++f) {
                        const float *ring = f ? s_v : s_u;
                        const int nr = f ? NUV : NUU;
                        const int i0 = f ? iv : iu;
                        float4 rr = make_float4(0, 0, 0, 0);
#pragma unroll
                        for (int j = 0; j < R; ++j)         // planes x+1 .. x+4
                            f4fma_(rr, k.w1x[j], b2ptx::lds128(ring + wrap(i0 + 1 + j, nr) * PLANE + poff));
                        const float *fc = ring + wrap(i0 + 2, nr) * PLANE + poff;     // plane x+2
#pragma unroll
                        for (int j = 0; j < R; ++j)
                            f4fma_(rr, k.w1y[j], b2ptx::lds128(fc + (j - H + 1) * BZ));
                        const float l = (hflag[t] & 2) ? fc[-1] : 0.f;
                        const float4 c = b2ptx::lds128(fc);
                        const float2 r = (hflag[t] & 4) ? *reinterpret_cast<const float2 *>(fc + 4) : make_float2(0.f, 0.f);
                        const float zz[7] = {l, c.x, c.y, c.z, c.w, r.x, r.y};
#pragma unroll
                        for (int j = 0; j < R; ++j) {
                            rr.x = fmaf(k.w1z[j], zz[j + 0], rr.x); rr.y = fmaf(k.w1z[j], zz[j + 1], rr.y);
                            rr.z = fmaf(k.w1z[j], zz[j + 2], rr.z); rr.w = fmaf(k.w1z[j], zz[j + 3], rr.w);
                        }
                        *reinterpret_cast<float4 *>((f ? s_gv : s_gu) + sgz + poff - (R - H) * BZ) = rr;
                    }
                }
            }
            __syncwarp();
            if (lane == 0) b2ptx::mbar_arrive(&empty[it % NB]);
            iu = wrap(iu + 1, NUU);
            iv = wrap(iv + 1, NUV);
            ig = wrap(ig + 1, NG);
        }
        return;
    }

    // =================== main warpgroups ===================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 152;");
    const int ty = tid / 16, tz4 = tid % 16;
    const int gy = y0 + ty, gz = z0 + 4 * tz4;
    const bool yok = gy < k.ny;
    const int zcnt = yok ? min(max(k.nz - gz, 0), 4) : 0;
    const int my_off = (ty + R) * BZ + RZ + 4 * tz4;
    const int my_goff = (ty + H) * BZ + RZ + 4 * tz4;
    const long long gidx0 = (long long)(k.oy + gy) * k.sy + (k.oz + gz);

    using b2ptx::F4;
    // Register queues with STATIC slots: the loop is unrolled 4x, plane x+k of a 4-deep queue lives in slot
    // (p + k) & 3 with p = it & 3, so advancing the sweep by one plane moves no data (the first version
    // shifted 18 float4 per iteration: a fifth of the main warps' instructions). The 9-plane x-history of u is
    // split into fut (planes x+1..x+4), cen (plane x) and pst (planes x-4..x-1): two float4 copies per plane.
    static_assert(R == 4 && NB == 4, "static queue slots assume 4-deep queues");
    F4 fut[4], pst[4], cen = b2ptx::f4zero(), vq[4], gqu[4], gqv[4];
    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        fut[i] = b2ptx::f4zero(); pst[i] = b2ptx::f4zero();
        vq[i] = b2ptx::f4zero(); gqu[i] = b2ptx::f4zero(); gqv[i] = b2ptx::f4zero();
    }
    long long gi = (long long)(k.ox + xs - PRE) * k.sx + gidx0;
    int iu = ((xs - PRE) % NUU + NUU) % NUU, iv = ((xs - PRE) % NUV + NUV) % NUV,
        ig = ((xs - PRE) % NG + NG) % NG;
    float4 nu = zero4, nv = zero4, na = zero4;      // prefetched u[t-1], v[t-1], A of plane x+1

    for (int itb = 0; itb < NIT; itb += 4) {
#pragma unroll
    for (int p = 0; p < 4; ++p) {
        const int it = itb + p;
        if (it >= NIT) break;
        const int x = xs - PRE + it;
        b2ptx::mbar_wait(&full[p], (itb >> 2) & 1);
        // u plane x+k: fut[(p+k)&3] (k = 1..4), cen (k = 0), pst[(p+k)&3] (k = -4..-1);
        // v plane x+k: vq[(p+k)&3] (k = 0..3); Gz plane x+k: gq*[(p+k)&3] (k = -2..1)
        pst[(p + 3) & 3] = cen;
        cen = fut[p];
        fut[p] = b2ptx::f4pack(b2ptx::lds128(s_u + wrap(iu + R, NUU) * PLANE + my_off));
        vq[(p + 3) & 3] = b2ptx::f4pack(b2ptx::lds128(s_v + wrap(iv + R - 1, NUV) * PLANE + my_off));

        // ---- stage A: own-column Gz(u), Gz(v) at plane g = x + 1 ----
        // x and y taps as fp32 pair operations, the z taps — whose operands straddle the pairs — in
        // scalar form
        {
            const float *uc = s_u + wrap(iu + 1, NUU) * PLANE + my_off;
            const float *vc = s_v + wrap(iv + 1, NUV) * PLANE + my_off;
            float4 ru, rv;
            {
                // D+z needs z-1 .. z+5 of the row: one float left, two floats right (4-byte and
                // 8-byte shared loads cost 1 and 2 wavefronts per warp instead of 4)
                const float lu = uc[-1], lv = vc[-1];
                const float2 ru_ = *reinterpret_cast<const float2 *>(uc + 4);
                const float2 rv_ = *reinterpret_cast<const float2 *>(vc + 4);
                const float4 cu = b2ptx::f4unpack(fut[(p + 1) & 3]), cv = b2ptx::f4unpack(vq[(p + 1) & 3]);
                const float zu[7] = {lu, cu.x, cu.y, cu.z, cu.w, ru_.x, ru_.y};
                const float zv[7] = {lv, cv.x, cv.y, cv.z, cv.w, rv_.x, rv_.y};
                ru = make_float4(k.w1z[0] * zu[0], k.w1z[0] * zu[1], k.w1z[0] * zu[2], k.w1z[0] * zu[3]);
                rv = make_float4(k.w1z[0] * zv[0], k.w1z[0] * zv[1], k.w1z[0] * zv[2], k.w1z[0] * zv[3]);
#pragma unroll
                for (int j = 1; j < R; ++j) {          // offsets j-1 relative to each of the 4 points
                    ru.x = fmaf(k.w1z[j], zu[j + 0], ru.x); ru.y = fmaf(k.w1z[j], zu[j + 1], ru.y);
                    ru.z = fmaf(k.w1z[j], zu[j + 2], ru.z); ru.w = fmaf(k.w1z[j], zu[j + 3], ru.w);
                    rv.x = fmaf(k.w1z[j], zv[j + 0], rv.x); rv.y = fmaf(k.w1z[j], zv[j + 1], rv.y);
                    rv.z = fmaf(k.w1z[j], zv[j + 2], rv.z); rv.w = fmaf(k.w1z[j], zv[j + 3], rv.w);
                }
            }
            F4 pu_ = b2ptx::f4pack(ru), pv_ = b2ptx::f4pack(rv);
#pragma unroll
            for (int j = 0; j < R; ++j) {            // x taps: planes x+j, from registers
                b2ptx::f4fma2(pu_, k.p_w1x[j], j == 0 ? cen : fut[(p + j) & 3]);
                b2ptx::f4fma2(pv_, k.p_w1x[j], vq[(p + j) & 3]);
            }
#pragma unroll
            for (int j = 0; j < R; ++j) {            // y taps: rows y-1..y+2 (own row from registers)
                const F4 a = (j == H - 1) ? fut[(p + 1) & 3] : b2ptx::f4pack(b2ptx::lds128(uc + (j - H + 1) * BZ));
                const F4 c = (j == H - 1) ? vq[(p + 1) & 3] : b2ptx::f4pack(b2ptx::lds128(vc + (j - H + 1) * BZ));
                b2ptx::f4fma2(pu_, k.p_w1y[j], a);
                b2ptx::f4fma2(pv_, k.p_w1y[j], c);
            }
            gqu[(p + 1) & 3] = pu_;
            gqv[(p + 1) & 3] = pv_;
            const int sgz = wrap(ig + 1, NG) * GPLANE + my_goff;
            *reinterpret_cast<float4 *>(s_gu + sgz) = b2ptx::f4unpack(pu_);
            *reinterpret_cast<float4 *>(s_gv + sgz) = b2ptx::f4unpack(pv_);
        }
        // u[t-1], v[t-1], A: loaded one full iteration before they are used (the registers are
        // there: the main warpgroups own 152 each after setmaxnreg)
        const float4 pu = nu, pv = nv, pa = na;
        {
            // one plane deep: a second plane would cost 12 registers, and the 4x unrolled body with static
            // queue slots is register-bound
            const long long gn = gi + k.sx;                 // plane x + 1
            if (x + 1 >= xs && x + 1 < xe && zcnt > 0) {
                nu = *reinterpret_cast<const float4 *>(k.um + gn);
                nv = *reinterpret_cast<const float4 *>(k.vm + gn);
                na = *reinterpret_cast<const float4 *>(k.A + gn);
            }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(NSYNC) : "memory");

        // ---- stage B: output plane x ----
        if (x >= xs) {
            const float *cpl = s_u + iu * PLANE + my_off;
            const F4 c = cen;
            const F4 vcn = vq[p];
            const float *gpu_ = s_gu + ig * GPLANE + my_goff;
            const float *gpv_ = s_gv + ig * GPLANE + my_goff;
            // z direction (scalar): Laplacian taps and D-z of Gz
            float4 lapz, zuz, zvz;
            {
                const float4 cc = b2ptx::f4unpack(c);
                const float4 l = b2ptx::lds128(cpl - 4), r = b2ptx::lds128(cpl + 4);
                const float zr[12] = {l.x, l.y, l.z, l.w, cc.x, cc.y, cc.z, cc.w, r.x, r.y, r.z, r.w};
                lapz.x = k.w2z[1] * (zr[3] + zr[5]); lapz.y = k.w2z[1] * (zr[4] + zr[6]);
                lapz.z = k.w2z[1] * (zr[5] + zr[7]); lapz.w = k.w2z[1] * (zr[6] + zr[8]);
#pragma unroll
                for (int i = 2; i <= R; ++i) {
                    lapz.x = fmaf(k.w2z[i], zr[4 - i] + zr[4 + i], lapz.x);
                    lapz.y = fmaf(k.w2z[i], zr[5 - i] + zr[5 + i], lapz.y);
                    lapz.z = fmaf(k.w2z[i], zr[6 - i] + zr[6 + i], lapz.z);
                    lapz.w = fmaf(k.w2z[i], zr[7 - i] + zr[7 + i], lapz.w);
                }
                // D-z needs z-2 .. z+4: two floats left, one float right
                const float2 lu = *reinterpret_cast<const float2 *>(gpu_ - 2);
                const float2 lv = *reinterpret_cast<const float2 *>(gpv_ - 2);
                const float ru_ = gpu_[4], rv_ = gpv_[4];
                const float4 cu = b2ptx::f4unpack(gqu[p]), cv = b2ptx::f4unpack(gqv[p]);
                const float au[7] = {lu.x, lu.y, cu.x, cu.y, cu.z, cu.w, ru_};
                const float av[7] = {lv.x, lv.y, cv.x, cv.y, cv.z, cv.w, rv_};
                zuz = make_float4(k.w1z[0] * au[0], k.w1z[0] * au[1], k.w1z[0] * au[2], k.w1z[0] * au[3]);
                zvz = make_float4(k.w1z[0] * av[0], k.w1z[0] * av[1], k.w1z[0] * av[2], k.w1z[0] * av[3]);
#pragma unroll
                for (int j = 1; j < R; ++j) {          // offsets j-2
                    zuz.x = fmaf(k.w1z[j], au[j + 0], zuz.x); zuz.y = fmaf(k.w1z[j], au[j + 1], zuz.y);
                    zuz.z = fmaf(k.w1z[j], au[j + 2], zuz.z); zuz.w = fmaf(k.w1z[j], au[j + 3], zuz.w);
                    zvz.x = fmaf(k.w1z[j], av[j + 0], zvz.x); zvz.y = fmaf(k.w1z[j], av[j + 1], zvz.y);
                    zvz.z = fmaf(k.w1z[j], av[j + 2], zvz.z); zvz.w = fmaf(k.w1z[j], av[j + 3], zvz.w);
                }
            }
            // x and y directions, as pairs
            F4 lap = b2ptx::f4pack(lapz);
            b2ptx::f4fma2(lap, k.p_wc, c);
#pragma unroll
            for (int i = 1; i <= R; ++i) {
                const F4 a = b2ptx::f4pack(b2ptx::lds128(cpl - i * BZ)), bb = b2ptx::f4pack(b2ptx::lds128(cpl + i * BZ));
                b2ptx::f4fma2(lap, k.p_w2y[i], b2ptx::f4add2(a, bb));
            }
#pragma unroll
            for (int i = 1; i <= R; ++i) b2ptx::f4fma2(lap, k.p_w2x[i], b2ptx::f4add2(pst[(p + 4 - i) & 3], fut[(p + i) & 3]));
            F4 zu4 = b2ptx::f4pack(zuz), zv4 = b2ptx::f4pack(zvz);
#pragma unroll
            for (int j = 0; j < R; ++j) {            // x direction: own Gz history (registers)
                b2ptx::f4fma2(zu4, k.p_w1x[j], gqu[(p + 2 + j) & 3]);
                b2ptx::f4fma2(zv4, k.p_w1x[j], gqv[(p + 2 + j) & 3]);
            }
#pragma unroll
            for (int j = 0; j < R; ++j) {            // y direction: rows y-2..y+1 (own row from registers)
                const F4 a = (j == H) ? gqu[p] : b2ptx::f4pack(b2ptx::lds128(gpu_ + (j - H) * BZ));
                const F4 bb = (j == H) ? gqv[p] : b2ptx::f4pack(b2ptx::lds128(gpv_ + (j - H) * BZ));
                b2ptx::f4fma2(zu4, k.p_w1y[j], a);
                b2ptx::f4fma2(zv4, k.p_w1y[j], bb);
            }
            // coupled update: f+ = f + A (m/dt^2 (f - f-) + H), H0 = e2 gh + sd Gzz(v), Hz = sd gh + Gzz(v)
            const F4 gh = b2ptx::f4sub2(lap, zu4);
            F4 H0 = b2ptx::f4mul2(k.p_sd, zv4);
            b2ptx::f4fma2(H0, k.p_e2, gh);
            F4 Hz = zv4;
            b2ptx::f4fma2(Hz, k.p_sd, gh);
            const F4 ppa = b2ptx::f4pack(pa);
            b2ptx::f4fma2(H0, k.p_mdt2, b2ptx::f4sub2(c, b2ptx::f4pack(pu)));
            b2ptx::f4fma2(Hz, k.p_mdt2, b2ptx::f4sub2(vcn, b2ptx::f4pack(pv)));
            const F4 ou_ = F4{b2ptx::fma2(ppa.a, H0.a, c.a), b2ptx::fma2(ppa.b, H0.b, c.b)};
            const F4 ov_ = F4{b2ptx::fma2(ppa.a, Hz.a, vcn.a), b2ptx::fma2(ppa.b, Hz.b, vcn.b)};
            const float4 ou = b2ptx::f4unpack(ou_), ov = b2ptx::f4unpack(ov_);
            if (zcnt == 4) {
                *reinterpret_cast<float4 *>(k.u1 + gi) = ou;
                *reinterpret_cast<float4 *>(k.v1 + gi) = ov;
            } else if (zcnt > 0) {
                const float tu[4] = {ou.x, ou.y, ou.z, ou.w}, tv[4] = {ov.x, ov.y, ov.z, ov.w};
                for (int i = 0; i < zcnt; ++i) { k.u1[gi + i] = tu[i]; k.v1[gi + i] = tv[i]; }
            }
        }
        __syncwarp();
        if (lane == 0) b2ptx::mbar_arrive(&empty[p]);
        iu = wrap(iu + 1, NUU);
        iv = wrap(iv + 1, NUV);
        ig = wrap(ig + 1, NG);
        gi += k.sx;
    }
    }
}

// ------------------------------------------------------------------------------------------
// 2-D single-pass sweep k_tti2d<R, ARR, ADJ> (radius 2 or 4): the 2-D reduction of k_tti_fused.
// ------------------------------------------------------------------------------------------
// A CTA owns a z-segment of TZ = 512 points (128 consumer threads, four consecutive z points each) and marches
// along x over a chunk of rows. Per iteration (output row x):
//   producer warp : TMA-loads the haloed rows u[t](x+R), v[t](x+R) (ARR: the sin / cos tables of row x+H-1) into
//                   shared rings, D rows ahead of the consumers;
//   stage A       : Gz(u), Gz(v) of row g = x+H-1 once, when its last input row has arrived: own columns from the
//                   register queue of u and the shared v rows, the two halo groups of the segment by one lane of
//                   each consumer warp; stored in a shared ring of H+1 rows and, for the own column, in register
//                   queues of R rows;
//   stage B       : the Laplacian (x-taps from the register queue of u, z-taps from the shared row), the outer
//                   half-node derivatives of Gz (x from the register queues, z from the shared row), the coupled
//                   update with A = 1/(m/dt^2 + damp/dt), 16-byte stores.
// u[t] and v[t] come from HBM once per step apart from the 2R rows that prime each chunk and the halo columns of
// each segment. Bytes per point: 28 with scalar parameters (u, v at t and t-1, A; u, v at t+1 written), 48 with
// arrays (+ sin, cos, 1+2eps, sqrt(1+2delta), m/dt^2); the adjoint reads the two mixes and p, r at t in place of u,
// v at t (and of the eps / delta tables): 36 and 48.
template <int R, bool ARR>
struct Tti2dCfg {
    static constexpr int H = R / 2;
    static constexpr int NC = 128;                   // consumer threads
    static constexpr int TZ = 4 * NC;                // z points of a segment
    static constexpr int RZ = 32;                    // halo columns on either side (128 B: TMA destinations aligned)
    static constexpr int NBOX = 3, BOXZ = 192;       // TMA boxes of a row: <= 256 elements, 128-byte multiples
    static constexpr int BZ = NBOX * BOXZ;           // = TZ + 2 RZ
    static constexpr int D = ARR ? 3 : 4;            // batches the producer may run ahead of the slowest consumer
    static constexpr int NU = R + D;                 // u / v rows x .. x+R, + (D-1) in flight
    static constexpr int NCR = R + D - 1;            // ARR: factor rows x-H .. x+H-1, + (D-1) in flight
    static constexpr int NG = H + 1;                 // Gz rows x .. x+H (stage A of x+1 writes x+H while B reads x)
    static constexpr int NB = 4;                     // barrier ring (>= D)
    static constexpr int MINB = R == 2 ? 3 : 2;      // CTAs per SM the registers must allow (R = 4: no spills)
    static constexpr size_t SMEM = (size_t)(2 * NU + 2 * NG + (ARR ? 2 * NCR : 0)) * BZ * 4 + 2 * NB * 8;
    static_assert(BZ == TZ + 2 * RZ && RZ >= 8 && NB >= D, "2-D TTI sweep layout");
};

struct Tti2dK {
    float *__restrict__ u1;
    float *__restrict__ v1;
    const float *__restrict__ um;
    const float *__restrict__ vm;
    const float *__restrict__ A;
    const float *__restrict__ tE2;     // ARR, forward
    const float *__restrict__ tSD;
    const float *__restrict__ tMD;     // ARR
    const float *__restrict__ pc;      // ADJ: p[t], r[t] (the tensor maps cover the mixes)
    const float *__restrict__ rc;
    long long sr;                      // row stride (the allocated z extent)
    int nx, nz, ox, oz;                // box extents and the array index of its first point
    int lx, ntz, slot0;
    float m_dt2, e2, sd;
    float w2x[5], w2z[5];
    float w1x[4], w1z[4];              // scalar: multiplied by sin(th) / cos(th); ARR: the raw weights
};

template <int N>
__device__ __forceinline__ int ring_(int r) { return (r + 64 * N) % N; }      // rows >= -2R > -64 N

template <int R, bool ARR, bool ADJ>
__global__ void __launch_bounds__(Tti2dCfg<R, ARR>::NC + 32, Tti2dCfg<R, ARR>::MINB)
k_tti2d(const __grid_constant__ CUtensorMap tm_u, const __grid_constant__ CUtensorMap tm_v,
        const __grid_constant__ CUtensorMap tm_s, const __grid_constant__ CUtensorMap tm_c, const Tti2dK k) {
    using C = Tti2dCfg<R, ARR>;
    constexpr int H = C::H, NC = C::NC, TZ = C::TZ, RZ = C::RZ, BZ = C::BZ, D = C::D;
    constexpr int NU = C::NU, NG = C::NG, NB = C::NB, NCW = NC / 32;
    constexpr int NCR = ARR ? C::NCR : 1;
    constexpr int PRE = 2 * R;                      // priming iterations before the first output row
    constexpr uint32_t ROWB = (uint32_t)BZ * 4;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *s_u = reinterpret_cast<float *>(smem_raw);
    float *s_v = s_u + NU * BZ;
    float *s_gu = s_v + NU * BZ;
    float *s_gv = s_gu + NG * BZ;
    float *s_c = s_gv + NG * BZ;                    // ARR: [row mod NCR][sin, cos][BZ]
    uint64_t *full = reinterpret_cast<uint64_t *>(s_c + (ARR ? 2 * NCR * BZ : 0));
    uint64_t *empty = full + NB;

    const int iz = blockIdx.x % k.ntz;
    const int z0 = iz * TZ;
    const int xs = (blockIdx.x / k.ntz) * k.lx;
    const int xe = min(xs + k.lx, k.nx);
    const int NIT = (xe - xs) + PRE;                // iterations: x = xs - PRE + it

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;

    if (tid == 0) {
        for (int i = 0; i < NB; ++i) {
            b2ptx::mbar_init(&full[i], 1);
            b2ptx::mbar_init(&empty[i], NCW);
        }
        b2ptx::fence_mbar_init();
    }
    __syncthreads();

    if (warp == NCW) {
        if (lane == 0) {
            b2ptx::tma_prefetch_desc(&tm_u);
            b2ptx::tma_prefetch_desc(&tm_v);
            if constexpr (ARR) {
                b2ptx::tma_prefetch_desc(&tm_s);
                b2ptx::tma_prefetch_desc(&tm_c);
            }
            for (int it = 0; it < NIT; ++it) {
                const int x = xs - PRE + it;
                if (it >= D) {
                    const int w = it - D;
                    b2ptx::mbar_wait(&empty[w % NB], (w / NB) & 1);
                }
                const int q = x + R;                        // u / v row of this batch
                const bool hv = q >= xs - R + 1;            // v rows below xs-R+1 are never read
                const int qc = x + H - 1;                   // ARR: factor row of stage A
                const bool hc = ARR && qc >= xs - H;
                b2ptx::mbar_arrive_expect_tx(&full[it % NB], ROWB * ((hv ? 2u : 1u) + (hc ? 2u : 0u)));
                float *du = s_u + ring_<NU>(q) * BZ, *dv = s_v + ring_<NU>(q) * BZ;
#pragma unroll
                for (int b = 0; b < C::NBOX; ++b) {
                    const int zc = k.oz + z0 - RZ + b * C::BOXZ;
                    b2ptx::tma_load_4d(du + b * C::BOXZ, &tm_u, &full[it % NB], zc, k.ox + q, 0, k.slot0);
                    if (hv) b2ptx::tma_load_4d(dv + b * C::BOXZ, &tm_v, &full[it % NB], zc, k.ox + q, 0, k.slot0);
                    if constexpr (ARR) {
                        if (hc) {
                            float *dc = s_c + ring_<NCR>(qc) * 2 * BZ + b * C::BOXZ;
                            b2ptx::tma_load_4d(dc, &tm_s, &full[it % NB], zc, k.ox + qc, 0, 0);
                            b2ptx::tma_load_4d(dc + BZ, &tm_c, &full[it % NB], zc, k.ox + qc, 0, 0);
                        }
                    }
                }
            }
        }
        return;
    }

    // ---------------- consumers ----------------
    const int gz = z0 + 4 * tid;
    const int zcnt = min(max(k.nz - gz, 0), 4);
    const int my = RZ + 4 * tid;                    // own column in a row
    // halo group of this warp's lane 0: field (warp & 1: v), side (warp >> 1: right)
    const int hoff = (warp >> 1) ? RZ + TZ : RZ - 4;
    const bool hfv = warp & 1;

    float4 uq[2 * R + 1];                           // u rows x-R .. x+R, own column
    float4 gqu[R], gqv[R];                          // Gz(u), Gz(v) rows x-H .. x+H-1, own column
#pragma unroll
    for (int i = 0; i <= 2 * R; ++i) uq[i] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < R; ++i) gqu[i] = gqv[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    const float wc = k.w2x[0] + k.w2z[0];
    long long gi = (long long)(k.ox + xs - PRE) * k.sr + (k.oz + gz);

    auto zwin = [](const float *c, float (&o)[12]) {      // the z points c-4 .. c+7
        const float4 l = b2ptx::lds128(c - 4), m = b2ptx::lds128(c), r = b2ptx::lds128(c + 4);
        o[0] = l.x; o[1] = l.y; o[2] = l.z; o[3] = l.w; o[4] = m.x; o[5] = m.y;
        o[6] = m.z; o[7] = m.w; o[8] = r.x; o[9] = r.y; o[10] = r.z; o[11] = r.w;
    };
    // Gz of four consecutive points: D+x from `xr` (rows g-H+1 .. g+H), D+z from the row window `zz` of row g,
    // factors `fs` / `fc` at the points (ARR)
    auto gz4 = [&](const float4 (&xr)[R], const float (&zz)[12], float4 fs, float4 fc) -> float4 {
        float4 dx = make_float4(0.f, 0.f, 0.f, 0.f), dz = dx;
#pragma unroll
        for (int j = 0; j < R; ++j) f4fma_(dx, k.w1x[j], xr[j]);
#pragma unroll
        for (int j = 0; j < R; ++j) {
            const int o = 4 + j - H + 1;
            dz.x = fmaf(k.w1z[j], zz[o + 0], dz.x); dz.y = fmaf(k.w1z[j], zz[o + 1], dz.y);
            dz.z = fmaf(k.w1z[j], zz[o + 2], dz.z); dz.w = fmaf(k.w1z[j], zz[o + 3], dz.w);
        }
        if constexpr (ARR)
            return make_float4(tti2d_gz_point(fs.x, fc.x, dx.x, dz.x), tti2d_gz_point(fs.y, fc.y, dx.y, dz.y),
                               tti2d_gz_point(fs.z, fc.z, dx.z, dz.z), tti2d_gz_point(fs.w, fc.w, dx.w, dz.w));
        return make_float4(dx.x + dz.x, dx.y + dz.y, dx.z + dz.z, dx.w + dz.w);   // weights hold sin / cos
    };
    auto ldt = [](const float *q) -> float4 {            // streams read once: no L1 allocation
        float4 r;
        asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
                     : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(q));
        return r;
    };
    auto ld4 = [&](const float *q) -> float4 {
        if (zcnt == 4) return ldt(q + gi);
        float t[4] = {0.f, 0.f, 0.f, 0.f};
        for (int i = 0; i < zcnt; ++i) t[i] = q[gi + i];
        return make_float4(t[0], t[1], t[2], t[3]);
    };

    for (int it = 0; it < NIT; ++it) {
        const int x = xs - PRE + it;
        const bool out = x >= xs && zcnt > 0;
        // loads of the output row issued first, so that stages A and B hide their latency
        float4 pu = make_float4(0.f, 0.f, 0.f, 0.f), pv = pu, pa = pu, pe2 = pu, psd = pu, pmd = pu, pcn = pu, rcn = pu;
        if (out) {
            pu = ld4(k.um);
            pv = ld4(k.vm);
            pa = ld4(k.A);
            if constexpr (ADJ) {
                pcn = ld4(k.pc);
                rcn = ld4(k.rc);
            }
            if constexpr (ARR) {
                if constexpr (!ADJ) {
                    pe2 = ld4(k.tE2);
                    psd = ld4(k.tSD);
                }
                pmd = ld4(k.tMD);
            }
        }
        b2ptx::mbar_wait(&full[it % NB], (it / NB) & 1);
        const int q = x + R;
#pragma unroll
        for (int i = 0; i < 2 * R; ++i) uq[i] = uq[i + 1];
        uq[2 * R] = b2ptx::lds128(s_u + ring_<NU>(q) * BZ + my);

        // ---- stage A: Gz at row g = x + H - 1 (inputs: rows x .. x+R-1) ----
        const int g = x + H - 1;
        if (g >= xs - H) {
            const float *fs_row = ARR ? s_c + ring_<NCR>(g) * 2 * BZ : nullptr;
            float zz[12];
            float4 xr[R];
            float4 fs = make_float4(0.f, 0.f, 0.f, 0.f), fc = fs;
            // own column, u
#pragma unroll
            for (int j = 0; j < R; ++j) xr[j] = uq[R + j];
            zwin(s_u + ring_<NU>(g) * BZ + my, zz);
            if constexpr (ARR) {
                fs = b2ptx::lds128(fs_row + my);
                fc = b2ptx::lds128(fs_row + BZ + my);
            }
            const float4 gu = gz4(xr, zz, fs, fc);
            // own column, v
#pragma unroll
            for (int j = 0; j < R; ++j) xr[j] = b2ptx::lds128(s_v + ring_<NU>(x + j) * BZ + my);
            zwin(s_v + ring_<NU>(g) * BZ + my, zz);
            const float4 gv = gz4(xr, zz, fs, fc);
            *reinterpret_cast<float4 *>(s_gu + ring_<NG>(g) * BZ + my) = gu;
            *reinterpret_cast<float4 *>(s_gv + ring_<NG>(g) * BZ + my) = gv;
#pragma unroll
            for (int i = 0; i < R - 1; ++i) {
                gqu[i] = gqu[i + 1];
                gqv[i] = gqv[i + 1];
            }
            gqu[R - 1] = gu;
            gqv[R - 1] = gv;
            // the segment's halo groups: one per consumer warp
            if (lane == 0) {
                const float *ring = hfv ? s_v : s_u;
#pragma unroll
                for (int j = 0; j < R; ++j) xr[j] = b2ptx::lds128(ring + ring_<NU>(x + j) * BZ + hoff);
                zwin(ring + ring_<NU>(g) * BZ + hoff, zz);     // inside the row: RZ >= 8
                if constexpr (ARR) {
                    fs = b2ptx::lds128(fs_row + hoff);
                    fc = b2ptx::lds128(fs_row + BZ + hoff);
                }
                *reinterpret_cast<float4 *>((hfv ? s_gv : s_gu) + ring_<NG>(g) * BZ + hoff) = gz4(xr, zz, fs, fc);
            }
        }
        // Gz of row x written by every consumer warp must be visible before its z neighbours are read
        asm volatile("bar.sync 1, %0;" ::"n"(NC) : "memory");

        // ---- stage B: output row x ----
        if (x >= xs) {
            const float4 c = uq[R];
            const float4 vcn = b2ptx::lds128(s_v + ring_<NU>(x) * BZ + my);
            float zr[12];
            zwin(s_u + ring_<NU>(x) * BZ + my, zr);
            float4 lap = make_float4(wc * c.x, wc * c.y, wc * c.z, wc * c.w);
#pragma unroll
            for (int i = 1; i <= R; ++i) {
                lap.x = fmaf(k.w2z[i], zr[4 - i] + zr[4 + i], lap.x);
                lap.y = fmaf(k.w2z[i], zr[5 - i] + zr[5 + i], lap.y);
                lap.z = fmaf(k.w2z[i], zr[6 - i] + zr[6 + i], lap.z);
                lap.w = fmaf(k.w2z[i], zr[7 - i] + zr[7 + i], lap.w);
            }
#pragma unroll
            for (int i = 1; i <= R; ++i) {
                const float4 a = uq[R - i], bb = uq[R + i];
                lap.x = fmaf(k.w2x[i], a.x + bb.x, lap.x); lap.y = fmaf(k.w2x[i], a.y + bb.y, lap.y);
                lap.z = fmaf(k.w2x[i], a.z + bb.z, lap.z); lap.w = fmaf(k.w2x[i], a.w + bb.w, lap.w);
            }
            // Gzz(u), Gzz(v): outer half-node derivatives of (factor * Gz) at offsets -H .. H-1
            float4 zu4 = make_float4(0.f, 0.f, 0.f, 0.f), zv4 = zu4;
#pragma unroll
            for (int j = 0; j < R; ++j) {                       // x: rows x-H+j, sin(th) at those rows
                float4 w = make_float4(k.w1x[j], k.w1x[j], k.w1x[j], k.w1x[j]);
                if constexpr (ARR) {
                    const float4 f = b2ptx::lds128(s_c + ring_<NCR>(x - H + j) * 2 * BZ + my);
                    w = make_float4(f.x * k.w1x[j], f.y * k.w1x[j], f.z * k.w1x[j], f.w * k.w1x[j]);
                }
                zu4.x = fmaf(w.x, gqu[j].x, zu4.x); zu4.y = fmaf(w.y, gqu[j].y, zu4.y);
                zu4.z = fmaf(w.z, gqu[j].z, zu4.z); zu4.w = fmaf(w.w, gqu[j].w, zu4.w);
                zv4.x = fmaf(w.x, gqv[j].x, zv4.x); zv4.y = fmaf(w.y, gqv[j].y, zv4.y);
                zv4.z = fmaf(w.z, gqv[j].z, zv4.z); zv4.w = fmaf(w.w, gqv[j].w, zv4.w);
            }
            {                                                   // z: row x, cos(th) at z+j-H
                float au[12], av[12], cz[12];
                zwin(s_gu + ring_<NG>(x) * BZ + my, au);
                zwin(s_gv + ring_<NG>(x) * BZ + my, av);
                if constexpr (ARR) zwin(s_c + ring_<NCR>(x) * 2 * BZ + BZ + my, cz);
#pragma unroll
                for (int j = 0; j < R; ++j) {
                    const int o = 4 + j - H;
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float w = ARR ? cz[o + e] * k.w1z[j] : k.w1z[j];
                        float &ru = e == 0 ? zu4.x : e == 1 ? zu4.y : e == 2 ? zu4.z : zu4.w;
                        float &rv = e == 0 ? zv4.x : e == 1 ? zv4.y : e == 2 ? zv4.z : zv4.w;
                        ru = fmaf(w, au[o + e], ru);
                        rv = fmaf(w, av[o + e], rv);
                    }
                }
            }
            float4 ou, ov;
#define B2_TTI2D_UPD(F)                                                                                      \
            if constexpr (ADJ)                                                                                   \
                tti_update_adj_point(lap.F, zu4.F, zv4.F, pcn.F, rcn.F, pu.F, pv.F, pa.F, ARR ? pmd.F : k.m_dt2, \
                                     ou.F, ov.F);                                                                \
            else                                                                                                 \
                tti_update_point(lap.F, zu4.F, zv4.F, c.F, vcn.F, pu.F, pv.F, pa.F, ARR ? pmd.F : k.m_dt2,       \
                                 ARR ? pe2.F : k.e2, ARR ? psd.F : k.sd, ou.F, ov.F);
            B2_TTI2D_UPD(x) B2_TTI2D_UPD(y) B2_TTI2D_UPD(z) B2_TTI2D_UPD(w)
#undef B2_TTI2D_UPD
            if (zcnt == 4) {
                *reinterpret_cast<float4 *>(k.u1 + gi) = ou;
                *reinterpret_cast<float4 *>(k.v1 + gi) = ov;
            } else if (zcnt > 0) {
                const float tu[4] = {ou.x, ou.y, ou.z, ou.w}, tv[4] = {ov.x, ov.y, ov.z, ov.w};
                for (int i = 0; i < zcnt; ++i) { k.u1[gi + i] = tu[i]; k.v1[gi + i] = tv[i]; }
            }
        }
        __syncwarp();
        if (lane == 0) b2ptx::mbar_arrive(&empty[it % NB]);
        gi += k.sr;
    }
}

__global__ void __launch_bounds__(256)
k_tti_coef_arr(const float *__restrict__ damp, const float *__restrict__ md, float inv_dt, float *__restrict__ A, size_t n) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) A[i] = 1.0f / (md[i] + (damp ? damp[i] * inv_dt : 0.f));
}

__global__ void __launch_bounds__(256)
k_tti_coef(const float *__restrict__ damp, float m_dt2, float inv_dt, float *__restrict__ A, size_t n) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) A[i] = 1.0f / (m_dt2 + (damp ? damp[i] * inv_dt : 0.f));
}

static bool tti_use_ws(int R);
constexpr int kTtiWsTY = 24;
template <int R> struct TtiTile;
template <> struct TtiTile<2> { static constexpr int TY = 32; };
template <> struct TtiTile<4> { static constexpr int TY = 28; };
// array-parameter sweep: more live registers per thread (factor queue, per-point tables) and the factor ring in shared
// memory. 30 rows at radius 2 (15 + 1 warps -> at most 128 registers); 20 rows at radius 4, the most whose rings fit in
// shared memory (220 KB)
template <int R> struct TtiArrTile;
template <> struct TtiArrTile<2> { static constexpr int TY = 30; };
template <> struct TtiArrTile<4> { static constexpr int TY = 20; };

// scratch cached across calls
// 0: A, 1-2: Gz(u), Gz(v) (two-pass), 3-8: per-point tables, 9-10: the adjoint's mixes
static ScratchSlot g_tti_scratch[11];

// the per-point tables of k_tti_tables (array-valued parameters)
static int tti_tables(TtiPlan &p) {
    int rc;
    B2_SM_COUNT(sms);
    float **t[6] = {&p.tCx, &p.tCy, &p.tCz, &p.tE2, &p.tSD, &p.tMD};
    for (int i = p.ndim == 2; i < 6; ++i)      // a 2-D plan has no rotation factor on its dummy dim: tCx stays NULL
        if ((rc = cached_scratch(g_tti_scratch[3 + i], p.slot_elems, t[i]))) return rc;
    k_tti_tables<<<sms * 8, 256, 0, stream()>>>(p.vp_a, p.eps_a, p.delta_a, p.theta_a, p.phi_a, p.vp, p.epsilon,
                                                 p.delta, p.theta, p.phi, 1.0f / (p.dt * p.dt), p.tCx, p.tCy, p.tCz,
                                                 p.tE2, p.tSD, p.tMD, p.slot_elems, p.ndim == 2);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

// tensor maps of the 2-D sweep over the field pair (u, v) of `tsize` slots: boxes of one row segment
static int tti2d_maps(const TtiPlan &p, const float *u, const float *v, int tsize, TtiPlan &out) {
    constexpr int BOXZ = Tti2dCfg<2, false>::BOXZ;
    const int dims[4] = {p.a[2], p.a[1], p.a[0], tsize};
    int rc;
    if ((rc = encode_tmap(&out.tm_u, u, 4, dims, BOXZ, 1, "tti"))) return rc;
    return encode_tmap(&out.tm_v, v, 4, dims, BOXZ, 1, "tti");
}

static int tti_plan_init_2d(TtiPlan &p, int kernel) {
    const bool ok = kernel != 1 && (p.R == 2 || p.R == 4) && p.a[2] % 4 == 0 && p.o[2] % 4 == 0 &&
                    (uintptr_t)p.u % 16 == 0 && (uintptr_t)p.v % 16 == 0;
    if (kernel == 2 && !ok) {
        set_error("tti: 2-D single-pass kernel forced but layout does not qualify (radius=%d, z extent %d and "
                  "z start %d must be multiples of 4, u and v 16-byte aligned)", p.R, p.a[2], p.o[2]);
        return B2_ERR_INVALID;
    }
    p.use_2d = ok;
    int rc;
    if (p.has_arrays && (rc = tti_tables(p))) return rc;
    if (!ok) {
        if ((rc = cached_scratch(g_tti_scratch[1], p.slot_elems, &p.gzu))) return rc;
        return cached_scratch(g_tti_scratch[2], p.slot_elems, &p.gzv);
    }
    if ((rc = cached_scratch(g_tti_scratch[0], p.slot_elems, &p.coefA))) return rc;
    B2_SM_COUNT(sms);
    const float inv_dt = 1.0f / p.dt;
    if (p.has_arrays)
        k_tti_coef_arr<<<sms * 8, 256, 0, stream()>>>(p.damp, p.tMD, inv_dt, p.coefA, p.slot_elems);
    else
        k_tti_coef<<<sms * 8, 256, 0, stream()>>>(p.damp, (1.0f / (p.vp * p.vp)) * (inv_dt * inv_dt), inv_dt,
                                                  p.coefA, p.slot_elems);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    if ((rc = tti2d_maps(p, p.u, p.v, p.tsize, p))) return rc;
    if (p.has_arrays) {       // sin(th), cos(th) of `Gzz_centered_2d`
        constexpr int BOXZ = Tti2dCfg<2, false>::BOXZ;
        const int dims1[4] = {p.a[2], p.a[1], p.a[0], 1};
        if ((rc = encode_tmap(&p.tm_cy, p.tCy, 4, dims1, BOXZ, 1, "tti"))) return rc;
        if ((rc = encode_tmap(&p.tm_cz, p.tCz, 4, dims1, BOXZ, 1, "tti"))) return rc;
    }
    return B2_OK;
}

int tti_plan_init(TtiPlan &p, int kernel) {
    p.kernel = kernel;
    if (p.R % 2 != 0 || p.R < 2 || p.R > B2_MAX_RADIUS) {
        set_error("tti: radius %d unsupported (space_order must be a multiple of 4, <= 16)", p.R);
        return B2_ERR_INVALID;
    }
    p.has_arrays = p.vp_a || p.eps_a || p.delta_a || p.theta_a || p.phi_a;
    if (p.ndim == 2) return tti_plan_init_2d(p, kernel);
    bool ok = (p.R == 2 || p.R == 4) && (p.a[2] % 4 == 0) && (p.o[2] % 4 == 0) &&
              ((uintptr_t)p.u % 16 == 0) && ((uintptr_t)p.v % 16 == 0) && (p.slot_elems % 4 == 0) &&
              p.n[1] >= 8 && p.n[2] >= 16;
    // array-valued parameters: the fused kernel takes only layouts with at least one float4 group of halo in z and R
    // rows in y on either side of the box, and planes of fewer than 2^31 points
    if (p.has_arrays)
        ok = ok && p.o[2] >= 4 && p.a[2] - (p.o[2] + p.n[2]) >= 4 &&
             p.o[1] >= p.R && p.a[1] - (p.o[1] + p.n[1]) >= p.R && (long long)p.a[1] * p.a[2] < (1ll << 31);
    if (kernel == 1) ok = false;
    if (kernel == 2 && !ok) {
        set_error("tti: fused kernel forced but layout does not qualify (radius=%d a2=%d o2=%d)", p.R, p.a[2], p.o[2]);
        return B2_ERR_INVALID;
    }
    p.use_fused = ok;
    p.arr_fused = ok && p.has_arrays;
    int rc;
    B2_SM_COUNT(sms);
    auto tables = [&]() -> int { return tti_tables(p); };
    if (ok) {
        if ((rc = cached_scratch(g_tti_scratch[0], p.slot_elems, &p.coefA))) return rc;
        const float inv_dt = 1.0f / p.dt;
        int ty;
        if (p.arr_fused) {
            if ((rc = tables())) return rc;
            k_tti_coef_arr<<<sms * 8, 256, 0, stream()>>>(p.damp, p.tMD, inv_dt, p.coefA, p.slot_elems);
            ty = p.R == 2 ? TtiArrTile<2>::TY : TtiArrTile<4>::TY;
        } else {
            const float md = (1.0f / (p.vp * p.vp)) * (1.0f / (p.dt * p.dt));
            k_tti_coef<<<sms * 8, 256, 0, stream()>>>(p.damp, md, inv_dt, p.coefA, p.slot_elems);
            ty = p.R == 2 ? TtiTile<2>::TY : (tti_use_ws(4) ? kTtiWsTY : TtiTile<4>::TY);
        }
        count_launch();
        B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
        p.tm_rows = ty + 2 * p.R;
        const int dims[4] = {p.a[2], p.a[1], p.a[0], p.tsize}, dims1[4] = {p.a[2], p.a[1], p.a[0], 1};
        if ((rc = encode_tmap(&p.tm_u, p.u, 4, dims, 72, ty + 2 * p.R, "tti"))) return rc;
        if ((rc = encode_tmap(&p.tm_v, p.v, 4, dims, 72, ty + 2 * p.R, "tti"))) return rc;
        if (p.arr_fused) {  // boxes of the Gz tile (TY + R rows) over the factor tables
            if ((rc = encode_tmap(&p.tm_cx, p.tCx, 4, dims1, 72, ty + p.R, "tti"))) return rc;
            if ((rc = encode_tmap(&p.tm_cy, p.tCy, 4, dims1, 72, ty + p.R, "tti"))) return rc;
            if ((rc = encode_tmap(&p.tm_cz, p.tCz, 4, dims1, 72, ty + p.R, "tti"))) return rc;
        }
        return B2_OK;
    }
    if ((rc = cached_scratch(g_tti_scratch[1], p.slot_elems, &p.gzu))) return rc;
    if ((rc = cached_scratch(g_tti_scratch[2], p.slot_elems, &p.gzv))) return rc;
    if (p.has_arrays && (rc = tables())) return rc;
    return B2_OK;
}

int tti_plan_retarget(const TtiPlan &p, float *u, float *v, TtiPlan &out) {
    out = p;
    out.u = u;
    out.v = v;
    if (!p.use_fused && !p.use_2d) return B2_OK;
    if ((uintptr_t)u % 16 != 0 || (uintptr_t)v % 16 != 0) {
        set_error("tti: the second field pair is not 16-byte aligned, so it cannot run the fused kernel of the first");
        return B2_ERR_INVALID;
    }
    int rc;
    if (p.use_2d) return tti2d_maps(p, u, v, p.tsize, out);
    const int dims[4] = {p.a[2], p.a[1], p.a[0], p.tsize};
    if ((rc = encode_tmap(&out.tm_u, u, 4, dims, 72, p.tm_rows, "tti"))) return rc;
    return encode_tmap(&out.tm_v, v, 4, dims, 72, p.tm_rows, "tti");
}

int tti_plan_adjoint(const TtiPlan &p, TtiPlan &out) {
    float *a = nullptr, *b = nullptr;
    int rc;
    if ((rc = cached_scratch(g_tti_scratch[9], p.slot_elems, &a))) return rc;
    if ((rc = cached_scratch(g_tti_scratch[10], p.slot_elems, &b))) return rc;
    out = p;                // tables, A and two-pass scratch shared; u / v stay p / r
    out.ma = a;
    out.mb = b;
    out.adj = true;
    if (p.use_2d) return tti2d_maps(p, a, b, 1, out);
    if (p.use_fused) {      // one slot each (cudaMalloc'ed, so 16-byte aligned): the sweep reads slot 0 of the maps
        // the scalar so=8 adjoint sweeps with k_tti_fused<4> where the forward takes k_tti_ws (its own tile height)
        if (!p.arr_fused) out.tm_rows = (p.R == 2 ? TtiTile<2>::TY : TtiTile<4>::TY) + 2 * p.R;
        const int dims1[4] = {p.a[2], p.a[1], p.a[0], 1};
        if ((rc = encode_tmap(&out.tm_u, a, 4, dims1, 72, out.tm_rows, "tti"))) return rc;
        if ((rc = encode_tmap(&out.tm_v, b, 4, dims1, 72, out.tm_rows, "tti"))) return rc;
    }
    return B2_OK;
}


// Born source term, 48 B/point: dm, u0 and v0 at t+1, t, t-1 and A (or the parameters of the denominator) read once,
// du[t+1] and dv[t+1] read and written. V4: four consecutive z points per thread with 16-byte accesses; the streams
// read once go through `ld.global.nc.L1::no_allocate`.
__device__ __forceinline__ float4 ld_once4(const float *p) {
    float4 r;
    asm("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
        : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}

__device__ __forceinline__ void tti_born_point4(const TtiBK &k, int x, int y, int z) {
    const long long idx = (long long)(k.o0 + x) * k.sx + (long long)(k.o1 + y) * k.sy + (k.o2 + z);
    const long long j = (long long)(k.dg0 + x) * k.dsx + (long long)(k.dg1 + y) * k.dsy + (k.dg2 + z);
    const float4 d = ld_once4(k.dm + j);
    const float4 a1 = ld_once4(k.u1 + idx), a0 = ld_once4(k.u0 + idx), am = ld_once4(k.um + idx);
    const float4 b1 = ld_once4(k.v1 + idx), b0 = ld_once4(k.v0 + idx), bm = ld_once4(k.vm + idx);
    float4 du = *reinterpret_cast<const float4 *>(k.du1 + idx);
    float4 dv = *reinterpret_cast<const float4 *>(k.dv1 + idx);
    const float dd[4] = {d.x, d.y, d.z, d.w};
    const float u1[4] = {a1.x, a1.y, a1.z, a1.w}, u0[4] = {a0.x, a0.y, a0.z, a0.w}, um[4] = {am.x, am.y, am.z, am.w};
    const float v1[4] = {b1.x, b1.y, b1.z, b1.w}, v0[4] = {b0.x, b0.y, b0.z, b0.w}, vm[4] = {bm.x, bm.y, bm.z, bm.w};
    float ou[4] = {du.x, du.y, du.z, du.w}, ov[4] = {dv.x, dv.y, dv.z, dv.w};
    float4 c;
    if (k.A) {
        c = ld_once4(k.A + idx);
    } else {
        const float4 md = k.tMD ? ld_once4(k.tMD + idx) : make_float4(k.m_dt2, k.m_dt2, k.m_dt2, k.m_dt2);
        const float4 dp = k.damp ? ld_once4(k.damp + idx) : make_float4(0.f, 0.f, 0.f, 0.f);
        c = make_float4(md.x + dp.x * k.inv_dt, md.y + dp.y * k.inv_dt, md.z + dp.z * k.inv_dt,
                        md.w + dp.w * k.inv_dt);
    }
    const float cc[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float qu = tti_born_q(dd[e], u1[e], u0[e], um[e], k.inv_dt2);
        const float qv = tti_born_q(dd[e], v1[e], v0[e], vm[e], k.inv_dt2);
        if (k.A) {
            ou[e] += qu * cc[e];
            ov[e] += qv * cc[e];
        } else {
            ou[e] += qu / cc[e];
            ov[e] += qv / cc[e];
        }
    }
    *reinterpret_cast<float4 *>(k.du1 + idx) = make_float4(ou[0], ou[1], ou[2], ou[3]);
    *reinterpret_cast<float4 *>(k.dv1 + idx) = make_float4(ov[0], ov[1], ov[2], ov[3]);
}

template <bool V4>
__global__ void __launch_bounds__(256) k_tti_born_src(const TtiBK k) {
    const int z = (V4 ? 4 : 1) * (blockIdx.x * blockDim.x + threadIdx.x);
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (z >= k.n2 || y >= k.n1) return;
    for (int x = blockIdx.z; x < k.n0; x += gridDim.z) {
        if constexpr (V4) tti_born_point4(k, x, y, z);
        else tti_born_point(k, x, y, z);
    }
}

int tti_born_source(const TtiPlan &p, const TtiPlan &pd, int slot0, int slotm, int slot1, const float *dm,
                    long long dsx, long long dsy, int dmh) {
    TtiBK k;
    k.u1 = p.u + (size_t)slot1 * p.slot_elems;
    k.u0 = p.u + (size_t)slot0 * p.slot_elems;
    k.um = p.u + (size_t)slotm * p.slot_elems;
    k.v1 = p.v + (size_t)slot1 * p.slot_elems;
    k.v0 = p.v + (size_t)slot0 * p.slot_elems;
    k.vm = p.v + (size_t)slotm * p.slot_elems;
    k.du1 = pd.u + (size_t)slot1 * p.slot_elems;
    k.dv1 = pd.v + (size_t)slot1 * p.slot_elems;
    // the fused plans tabulated A; the two-pass plans have m/dt^2 per point only with array parameters
    const bool tabA = p.use_fused || p.use_2d;
    k.A = tabA ? p.coefA : nullptr;
    k.tMD = tabA ? nullptr : p.tMD;
    k.damp = p.damp;
    k.dm = dm;
    k.sx = p.sx;
    k.sy = p.sy;
    k.dsx = dsx;
    k.dsy = dsy;
    k.n0 = p.n[0]; k.n1 = p.n[1]; k.n2 = p.n[2];
    k.o0 = p.o[0]; k.o1 = p.o[1]; k.o2 = p.o[2];
    k.dg0 = p.ndim == 2 ? 0 : p.o[0] - p.so + dmh;      // 2-D: dim 0 is the plan's dummy dim
    k.dg1 = p.o[1] - p.so + dmh; k.dg2 = p.o[2] - p.so + dmh;
    k.inv_dt = 1.0f / p.dt;
    k.inv_dt2 = 1.0f / (p.dt * p.dt);
    k.m_dt2 = (1.0f / (p.vp * p.vp)) * k.inv_dt2;
    auto a16 = [](const void *q) { return (uintptr_t)q % 16 == 0; };
    const bool v4 = k.o2 % 4 == 0 && k.n2 % 4 == 0 && k.sy % 4 == 0 && k.dg2 % 4 == 0 && k.dsy % 4 == 0 &&
                    p.slot_elems % 4 == 0 && a16(p.u) && a16(p.v) && a16(pd.u) && a16(pd.v) && a16(dm) &&
                    (!k.A || a16(k.A)) && (!k.tMD || a16(k.tMD)) && (!k.damp || a16(k.damp));
    dim3 block(64, 4, 1);
    const int nz = v4 ? k.n2 / 4 : k.n2;
    dim3 grid((nz + 63) / 64, (k.n1 + 3) / 4, (unsigned)std::min(k.n0, 65535));
    char sweep[64];
    snprintf(sweep, sizeof(sweep), "%s", b2_last_sweep_kernel());
    note_sweep_kernel("%s+born_%s", sweep, v4 ? "v4" : "s");
    if (v4) k_tti_born_src<true><<<grid, block, 0, stream()>>>(k);
    else k_tti_born_src<false><<<grid, block, 0, stream()>>>(k);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

// a = e2 p + sd r, b = sd p + r over the whole slot; e2 / sd are the scalars or the per-point tables (which cover
// the whole allocation too). V4: four consecutive points per thread, the streams read once bypass L1.
struct TtiMixK {
    const float *__restrict__ p;
    const float *__restrict__ r;
    float *__restrict__ a;
    float *__restrict__ b;
    const float *__restrict__ tE2;
    const float *__restrict__ tSD;
    float e2, sd;
    size_t n;
};

template <bool V4>
__global__ void __launch_bounds__(256) k_tti_adj_mix(const TtiMixK k) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    if constexpr (V4) {
        for (; 4 * i < k.n; i += stride) {
            const float4 p = ld_once4(k.p + 4 * i), r = ld_once4(k.r + 4 * i);
            const float4 e = k.tE2 ? ld_once4(k.tE2 + 4 * i) : make_float4(k.e2, k.e2, k.e2, k.e2);
            const float4 s = k.tSD ? ld_once4(k.tSD + 4 * i) : make_float4(k.sd, k.sd, k.sd, k.sd);
            float4 a, b;
            tti_adj_mix_point(e.x, s.x, p.x, r.x, a.x, b.x);
            tti_adj_mix_point(e.y, s.y, p.y, r.y, a.y, b.y);
            tti_adj_mix_point(e.z, s.z, p.z, r.z, a.z, b.z);
            tti_adj_mix_point(e.w, s.w, p.w, r.w, a.w, b.w);
            *reinterpret_cast<float4 *>(k.a + 4 * i) = a;
            *reinterpret_cast<float4 *>(k.b + 4 * i) = b;
        }
    } else {
        for (; i < k.n; i += stride)
            tti_adj_mix_point(k.tE2 ? k.tE2[i] : k.e2, k.tSD ? k.tSD[i] : k.sd, k.p[i], k.r[i], k.a[i], k.b[i]);
    }
}

int tti_adj_mix(const TtiPlan &pa, int slot0) {
    TtiMixK k;
    k.p = pa.u + (size_t)slot0 * pa.slot_elems;
    k.r = pa.v + (size_t)slot0 * pa.slot_elems;
    k.a = pa.ma;
    k.b = pa.mb;
    k.tE2 = pa.has_arrays ? pa.tE2 : nullptr;
    k.tSD = pa.has_arrays ? pa.tSD : nullptr;
    k.e2 = 1.0f + 2.0f * pa.epsilon;
    k.sd = sqrtf(1.0f + 2.0f * pa.delta);
    k.n = pa.slot_elems;
    auto a16 = [](const void *q) { return q == nullptr || (uintptr_t)q % 16 == 0; };
    const bool v4 = k.n % 4 == 0 && a16(k.p) && a16(k.r) && a16(k.a) && a16(k.b) && a16(k.tE2) && a16(k.tSD);
    B2_SM_COUNT(sms);
    if (v4) k_tti_adj_mix<true><<<sms * 8, 256, 0, stream()>>>(k);
    else k_tti_adj_mix<false><<<sms * 8, 256, 0, stream()>>>(k);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

// The members of TtiFK that both fused launchers fill alike (zero elsewhere): the time levels, A, the layout, the x
// range and its chunks, the tensor-map slot and the adjoint's centre. `ty`: rows of the kernel's yz-tile; `nblk`: the
// CTAs to launch.
template <int R>
static int tti_fk_common(const TtiPlan &p, int ty, int slot0, int slotm, int slot1, int xlo, int xcount, TtiFK &k,
                         unsigned &nblk) {
    constexpr int TZ = TtiCfg<R, 1>::TZ;           // the same for every tile height
    memset(&k, 0, sizeof(k));
    k.u1 = p.u + (size_t)slot1 * p.slot_elems;
    k.v1 = p.v + (size_t)slot1 * p.slot_elems;
    k.um = p.u + (size_t)slotm * p.slot_elems;
    k.vm = p.v + (size_t)slotm * p.slot_elems;
    k.A = p.coefA;
    k.sx = p.sx;
    k.sy = p.sy;
    k.ny = p.n[1];
    k.nz = p.n[2];
    k.ox = p.o[0];
    k.oy = p.o[1];
    k.oz = p.o[2];
    k.xlo = xlo;
    k.xcount = xcount;
    k.ntz = (p.n[2] + TZ - 1) / TZ;
    k.nty = (p.n[1] + ty - 1) / ty;
    int lx = env_int("B2_TTI_LX", 0);
    if (lx <= 0) {
        B2_SM_COUNT(sms);
        lx = choose_chunk_len(sms, k.ntz * k.nty, xcount, 2 * R, 32);
    }
    lx = std::min(lx, xcount);
    k.lx = lx;
    nblk = (unsigned)(k.ntz * k.nty * ((xcount + lx - 1) / lx));
    k.slot0 = p.adj ? 0 : slot0;
    k.pc = p.adj ? p.u + (size_t)slot0 * p.slot_elems : nullptr;
    k.rc = p.adj ? p.v + (size_t)slot0 * p.slot_elems : nullptr;
    return B2_OK;
}

// fused kernel with per-point parameter tables
template <int R>
static int tti_launch_fused_arr(const TtiPlan &p, int slot0, int slotm, int slot1, int xlo, int xcount) {
    constexpr int TY = TtiArrTile<R>::TY;
    using C = TtiCfg<R, TY, true>;
    auto kern = p.adj ? k_tti_fused<R, TY, true, true> : k_tti_fused<R, TY, true>;
    static_assert(C::SMEM <= 232448, "shared memory per CTA");
    static bool attr_set[2] = {false, false};
    if (!attr_set[p.adj]) {
        B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM), B2_ERR_LAUNCH);
        attr_set[p.adj] = true;
    }
    TtiFK k;
    unsigned nblk;
    int rc;
    if ((rc = tti_fk_common<R>(p, TY, slot0, slotm, slot1, xlo, xcount, k, nblk))) return rc;
    k.tCx = p.tCx; k.tCy = p.tCy; k.tCz = p.tCz; k.tE2 = p.tE2; k.tSD = p.tSD; k.tMD = p.tMD;
    k.hint = env_int("B2_TTI_ARR_HINT", 1);
    for (int i = 0; i <= R; ++i) { k.w2x[i] = p.w2[0][i]; k.w2y[i] = p.w2[1][i]; k.w2z[i] = p.w2[2][i]; }
    for (int i = 0; i < R; ++i) { k.w1x[i] = p.w1[0][i]; k.w1y[i] = p.w1[1][i]; k.w1z[i] = p.w1[2][i]; }
    timing_begin();
    note_sweep_kernel("tti_arr_ct2<%d>%s", R, p.adj ? "+adj" : "");
    kern<<<nblk, TY * 16 + 32, C::SMEM, stream()>>>(p.tm_u, p.tm_v, p.tm_cx, p.tm_cy, p.tm_cz, k);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

static bool tti_use_ws(int R) { return R == 4 && env_int("B2_TTI_KERNEL", 3) == 3; }
template <int R>
static int tti_launch_fused(const TtiPlan &p, int slot0, int slotm, int slot1, int xlo, int xcount) {
    // k_tti_ws is register-bound (DESIGN.md §3.5): with the centre loads of the adjoint it spills, so the adjoint
    // sweeps with k_tti_fused<4, .., ADJ>, which does not
    const bool ws = tti_use_ws(R) && !p.adj;
    constexpr int TYF = TtiTile<R>::TY;
    using C = TtiCfg<R, TYF>;
    using CW = TtiWsCfg<kTtiWsTY>;
    auto kern = p.adj ? k_tti_fused<R, TYF, false, true> : k_tti_fused<R, TYF, false>;
    auto kern_ws = k_tti_ws<kTtiWsTY>;
    static bool attr_set[2] = {false, false};
    if (!attr_set[p.adj]) {
        B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM), B2_ERR_LAUNCH);
        B2_CUDA(cudaFuncSetAttribute(kern_ws, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CW::SMEM), B2_ERR_LAUNCH);
        attr_set[p.adj] = true;
    }
    TtiFK k;
    unsigned nblk;
    int rc;
    if ((rc = tti_fk_common<R>(p, ws ? kTtiWsTY : TYF, slot0, slotm, slot1, xlo, xcount, k, nblk))) return rc;
    k.m_dt2 = (1.0f / (p.vp * p.vp)) * (1.0f / (p.dt * p.dt));
    const float st = sinf(p.theta), ct = cosf(p.theta), sp = sinf(p.phi), cp = cosf(p.phi);
    k.cx = st * cp;
    k.cy = st * sp;
    k.cz = ct;
    k.e2 = 1.0f + 2.0f * p.epsilon;
    k.sd = sqrtf(1.0f + 2.0f * p.delta);
    for (int i = 0; i <= R; ++i) { k.w2x[i] = p.w2[0][i]; k.w2y[i] = p.w2[1][i]; k.w2z[i] = p.w2[2][i]; }
    for (int i = 0; i < R; ++i) { k.w1x[i] = k.cx * p.w1[0][i]; k.w1y[i] = k.cy * p.w1[1][i]; k.w1z[i] = k.cz * p.w1[2][i]; }
    for (int i = 0; i <= R && i < 5; ++i) { k.p_w2x[i] = make_float2(k.w2x[i], k.w2x[i]); k.p_w2y[i] = make_float2(k.w2y[i], k.w2y[i]); }
    for (int i = 0; i < R && i < 4; ++i) { k.p_w1x[i] = make_float2(k.w1x[i], k.w1x[i]); k.p_w1y[i] = make_float2(k.w1y[i], k.w1y[i]); }
    {
        const float wc = k.w2x[0] + k.w2y[0] + k.w2z[0];
        k.p_wc = make_float2(wc, wc);
        k.p_e2 = make_float2(k.e2, k.e2);
        k.p_sd = make_float2(k.sd, k.sd);
        k.p_mdt2 = make_float2(k.m_dt2, k.m_dt2);
    }
    timing_begin();
    if (ws) note_sweep_kernel("tti_ws<pf1>");
    else note_sweep_kernel("tti_fused<%d>%s", R, p.adj ? "+adj" : "");
    if (ws)
        kern_ws<<<nblk, kTtiWsTY * 16 + 128, CW::SMEM, stream()>>>(p.tm_u, p.tm_v, k);
    else
        kern<<<nblk, TYF * 16 + 32, C::SMEM, stream()>>>(p.tm_u, p.tm_v, p.tm_u, p.tm_u, p.tm_u, k);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

// the 2-D single-pass sweep over the plan's rows (grid x), every z-segment
template <int R, bool ARR>
static int tti2d_launch(const TtiPlan &p, int slot0, int slotm, int slot1) {
    using C = Tti2dCfg<R, ARR>;
    auto kern = p.adj ? k_tti2d<R, ARR, true> : k_tti2d<R, ARR, false>;
    static bool attr_set[2] = {false, false};
    static int occ[2] = {0, 0};
    if (!attr_set[p.adj]) {
        B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM), B2_ERR_LAUNCH);
        B2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[p.adj], kern, C::NC + 32, C::SMEM), B2_ERR_LAUNCH);
        attr_set[p.adj] = true;
    }
    Tti2dK k;
    memset(&k, 0, sizeof(k));
    k.u1 = p.u + (size_t)slot1 * p.slot_elems;
    k.v1 = p.v + (size_t)slot1 * p.slot_elems;
    k.um = p.u + (size_t)slotm * p.slot_elems;
    k.vm = p.v + (size_t)slotm * p.slot_elems;
    k.A = p.coefA;
    if (ARR) { k.tE2 = p.tE2; k.tSD = p.tSD; k.tMD = p.tMD; }
    k.pc = p.adj ? p.u + (size_t)slot0 * p.slot_elems : nullptr;
    k.rc = p.adj ? p.v + (size_t)slot0 * p.slot_elems : nullptr;
    k.slot0 = p.adj ? 0 : slot0;
    k.sr = p.sy;
    k.nx = p.n[1];
    k.nz = p.n[2];
    k.ox = p.o[1];
    k.oz = p.o[2];
    k.ntz = (k.nz + C::TZ - 1) / C::TZ;
    B2_SM_COUNT(sms);
    k.lx = std::min(choose_chunk_len((long long)sms * std::max(occ[p.adj], 1), k.ntz, k.nx, 2 * R, 32), k.nx);
    const unsigned nblk = (unsigned)(k.ntz * ((k.nx + k.lx - 1) / k.lx));
    k.m_dt2 = (1.0f / (p.vp * p.vp)) * (1.0f / (p.dt * p.dt));
    k.e2 = 1.0f + 2.0f * p.epsilon;
    k.sd = sqrtf(1.0f + 2.0f * p.delta);
    const float st = ARR ? 1.f : sinf(p.theta), ct = ARR ? 1.f : cosf(p.theta);
    for (int i = 0; i <= R; ++i) { k.w2x[i] = p.w2[1][i]; k.w2z[i] = p.w2[2][i]; }
    for (int i = 0; i < R; ++i) { k.w1x[i] = st * p.w1[1][i]; k.w1z[i] = ct * p.w1[2][i]; }
    timing_begin();
    note_sweep_kernel("tti2d%s<%d>%s", ARR ? "_arr" : "", R, p.adj ? "+adj" : "");
    kern<<<nblk, C::NC + 32, C::SMEM, stream()>>>(p.tm_u, p.tm_v, ARR ? p.tm_cy : p.tm_u, ARR ? p.tm_cz : p.tm_u, k);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

int tti_step(const TtiPlan &p, int slot0, int slotm, int slot1, int xlo, int xcount) {
    if (xcount <= 0) return B2_OK;
    if (p.use_2d) {
        if (p.R == 2) return p.has_arrays ? tti2d_launch<2, true>(p, slot0, slotm, slot1)
                                          : tti2d_launch<2, false>(p, slot0, slotm, slot1);
        return p.has_arrays ? tti2d_launch<4, true>(p, slot0, slotm, slot1)
                            : tti2d_launch<4, false>(p, slot0, slotm, slot1);
    }
    if (p.arr_fused)
        return p.R == 2 ? tti_launch_fused_arr<2>(p, slot0, slotm, slot1, xlo, xcount)
                        : tti_launch_fused_arr<4>(p, slot0, slotm, slot1, xlo, xcount);
    if (p.use_fused)
        return p.R == 2 ? tti_launch_fused<2>(p, slot0, slotm, slot1, xlo, xcount)
                        : tti_launch_fused<4>(p, slot0, slotm, slot1, xlo, xcount);
    TtiK k;
    k.u0 = p.adj ? p.ma : p.u + (size_t)slot0 * p.slot_elems;
    k.v0 = p.adj ? p.mb : p.v + (size_t)slot0 * p.slot_elems;
    k.pc = p.u + (size_t)slot0 * p.slot_elems;
    k.rc = p.v + (size_t)slot0 * p.slot_elems;
    k.um = p.u + (size_t)slotm * p.slot_elems;
    k.vm = p.v + (size_t)slotm * p.slot_elems;
    k.u1 = p.u + (size_t)slot1 * p.slot_elems;
    k.v1 = p.v + (size_t)slot1 * p.slot_elems;
    k.damp = p.damp;
    k.gzu = p.gzu;
    k.gzv = p.gzv;
    k.sx = p.sx;
    k.sy = p.sy;
    k.n0 = xcount;
    k.n1 = p.n[1];
    k.n2 = p.n[2];
    k.o0 = p.o[0] + xlo;
    k.o1 = p.o[1];
    k.o2 = p.o[2];
    k.R = p.R;
    k.rx = p.ndim == 2 ? 0 : p.R;
    k.inv_dt = 1.0f / p.dt;
    k.m_dt2 = (1.0f / (p.vp * p.vp)) * (1.0f / (p.dt * p.dt));
    const float st = sinf(p.theta), ct = cosf(p.theta), sp = sinf(p.phi), cp = cosf(p.phi);
    k.cx = st * cp;
    k.cy = st * sp;
    k.cz = ct;
    if (p.ndim == 2) {
        k.cx = 0.f;
        k.cy = st;
    }
    k.e2 = 1.0f + 2.0f * p.epsilon;
    k.sd = sqrtf(1.0f + 2.0f * p.delta);
    memcpy(k.w2, p.w2, sizeof(k.w2));
    memcpy(k.w1, p.w1, sizeof(k.w1));
    k.tCx = p.tCx; k.tCy = p.tCy; k.tCz = p.tCz; k.tE2 = p.tE2; k.tSD = p.tSD; k.tMD = p.tMD;
    dim3 block(64, 4, 1);
    dim3 gridA((k.n2 + k.R + 63) / 64, (k.n1 + k.R + 3) / 4, (unsigned)std::min(xcount + k.rx, 65535));
    timing_begin();
    note_sweep_kernel("tti_two_pass%s", p.adj ? "+adj" : "");
    k_tti_gz<<<gridA, block, 0, stream()>>>(k);
    count_launch();
    dim3 gridB((k.n2 + 63) / 64, (k.n1 + 3) / 4, (unsigned)std::min(xcount, 65535));
    if (p.adj) k_tti_update<true><<<gridB, block, 0, stream()>>>(k);
    else k_tti_update<false><<<gridB, block, 0, stream()>>>(k);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

}  // namespace b2

