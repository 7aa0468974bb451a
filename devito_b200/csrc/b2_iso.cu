// Isotropic acoustic time-update kernels for sm_90a.
//
// Numerical spec (reference: examples/seismic/acoustic/operators.py:71-107 `iso_stencil`,
// `laplacian` :50-68; generated form printed by the reference's own code generator):
//
//   u[t+1] = ( m/dt^2 (2 u[t] - u[t-1]) + damp/dt u[t] + sum_d sum_k w_d[k] u[t][..+k..] )
//            / ( m/dt^2 + damp/dt )
//
// with w_d[k] = finite_diff_weights(2, ...)/h_d^2 (devito/finite_differences/tools.py:231-236).
//
// Kernels:
//   k_iso_generic : one thread per point, any radius <= 8, 2-D or 3-D, any alignment.
//   k_iso_tma     : 2.5-D sweep. A CTA owns a (TY x TZ) yz-tile and marches along x.
//                   A producer warp streams haloed yz-planes of u[t] (and the matching tiles
//                   of u[t-1], damp, vp|m) into shared-memory rings with TMA
//                   (cp.async.bulk.tensor) signalled on mbarriers; consumer threads own four
//                   consecutive z points (float4), keep the x-direction neighbours in a
//                   register queue, read y/z neighbours from the shared plane, and write
//                   u[t+1] with 16-byte coalesced stores. No tensor cores: the update is
//                   HBM-bandwidth bound (16 B/point; 12 B with a scalar vp on the x-planes whose
//                   coefficient A repeats the pinned plane's, see IsoTK::reuse).
//   k_iso_tma2    : the same sweep advancing two time levels per pass (so=8, scalar vp; DESIGN.md §3.7).
#include "b2_iso.cuh"
#include "b2_iso_point.cuh"
#include "b2_ptx.cuh"
#include <cstdlib>
#include <algorithm>
#include <vector>

namespace b2 {

// ------------------------------------------------------------------------------------------
// generic kernel
// ------------------------------------------------------------------------------------------
// point forms (shared with the CPU emulation test): b2_iso_point.cuh
__global__ void __launch_bounds__(256) k_iso_generic(IsoGK k) {
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (z >= k.n2 || y >= k.n1) return;
    for (int x = blockIdx.z; x < k.n0; x += gridDim.z) iso_point(k, x, y, z);
}

// OT4 first pass over the box grown by the radius (n*/o* already describe the grown box)
__global__ void __launch_bounds__(256) k_ot4_w(IsoGK k) {
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (z >= k.n2 || y >= k.n1) return;
    for (int x = blockIdx.z; x < k.n0; x += gridDim.z) ot4_w_point(k, x, y, z);
}

// Time-subsampled snapshot of the iteration box (b2_iso_point.cuh::snapshot_point)
__global__ void __launch_bounds__(256) k_snapshot(SnapK k) {
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (z >= k.n2 || y >= k.n1) return;
    for (int x = blockIdx.z; x < k.n0; x += gridDim.z) snapshot_point(k, x, y, z);
}

int iso_snapshot(const IsoPlan &p, int slot, float *snap, long long dsx, long long dsy, int d0, int d1, int d2) {
    SnapK k;
    k.src = p.u + (size_t)slot * p.slot_elems;
    k.dst = snap;
    k.sx = p.sx; k.sy = p.sy;
    k.dsx = dsx; k.dsy = dsy;
    k.n0 = p.n[0]; k.n1 = p.n[1]; k.n2 = p.n[2];
    k.o0 = p.o[0]; k.o1 = p.o[1]; k.o2 = p.o[2];
    k.d0 = d0; k.d1 = d1; k.d2 = d2;
    dim3 block(64, 4, 1);
    dim3 grid((k.n2 + 63) / 64, (k.n1 + 3) / 4, (unsigned)std::min(k.n0, 65535));
    k_snapshot<<<grid, block, 0, stream()>>>(k);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

// Born source term added to the freshly updated linearised field (b2_iso_point.cuh::born_src_point)
__global__ void __launch_bounds__(256) k_born_src(IsoGK k) {
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (z >= k.n2 || y >= k.n1) return;
    for (int x = blockIdx.z; x < k.n0; x += gridDim.z) born_src_point(k, x, y, z);
}

// Free surface: the sweep kernels compute every row with the plain stencil; this kernel then REDOES
// the rows z <= radius — the only ones with a vertical tap that reaches the surface (z - k == 0, which
// contributes 0 in the reference, not u[0]: u[0] is non-zero right after a source deposited into the
// surface row) or goes above it — and clears the surface row. It touches (radius+1)/n2 of the grid
// (0.5 % at 1024^3, so = 8). The halo above the surface is left alone: sinc sources/receivers deposit
// into / sample it in the reference too.
__global__ void __launch_bounds__(256) k_iso_fs_fix(IsoGK k) {
    const int z = threadIdx.x;                                   // 0 .. r2 (blockDim.x == 16 > B2_MAX_RADIUS)
    const int y = blockIdx.x * blockDim.y + threadIdx.y;
    if (z > k.r2 || y >= k.n1) return;
    for (int x = blockIdx.y; x < k.n0; x += gridDim.y) iso_fs_point(k, x, y, z);
}

// ------------------------------------------------------------------------------------------
// TMA 2.5-D kernel
// ------------------------------------------------------------------------------------------
// The update is evaluated in the algebraically identical division-free form
//     u+ = u + A (m/dt^2 (u - u-) + lap)            scalar m      (A = 1/(m/dt^2 + damp/dt))
//     u+ = u + B (u - u-) + A lap                   array vp|m    (B = m/dt^2 * A)
// with A (and B) tabulated once per call by k_iso_coef: the IEEE division, which cost ~1/5 of
// the issued instructions of the first version of this kernel, leaves the
// inner loop, and A replaces damp (B replaces vp|m) in the streamed arrays, so the HBM traffic
// per point is unchanged (16 B, or 20 B with an array parameter).
template <int R>
struct IsoTK {
    float *__restrict__ u1;      // base of the output time slot
    long long sx, sy;
    int ny, nz;                  // iteration extents (for masking)
    int ox, oy, oz;
    int xlo, xcount, lx;
    int ntz, nty;
    int slot0, slotm;
    float m_dt2;
    float wx[R + 1], wy[R + 1], wz[R + 1];
    // ---- x-slab decomposition, halo step fused into the sweep (all zero / null on a single device) ----
    // The CTAs that produce a boundary plane also store it into the neighbour GPU's halo through the
    // CUDA-IPC mapped peer pointer (16-byte stores over NVLink), and the producer lane of a CTA that
    // needs a halo plane of u[t] first acquires the flag the neighbour released after its previous
    // step. Chunk 0 marches from its high end DOWN to x = 0 when a low neighbour exists, so every CTA
    // touches the neighbour's planes at the very END of its march: by then the flag has long been set.
    int back0;                    // chunk 0 marches backwards
    int nown;                     // planes owned by this rank: peer planes are [0, pw) and [nown - pw, nown)
    int pw;                       // planes published per side (= R)
    float *peer_lo, *peer_hi;     // neighbour field bases (NULL: physical boundary)
    long long off_lo, off_hi;     // element offset of "my plane 0" inside the neighbour's array (output slot)
    const int *flag_lo, *flag_hi; // local flags the neighbours release (NULL: nothing to wait for)
    int want;                     // flag value that says "halos of u[t] are in place" (< 0: already ensured)
    // ---- coefficient reuse (scalar parameter only; NULL: every A tile is streamed) ----
    // reuse[x] = 1 (allocated plane index) when A on plane x equals A on plane pin_x bit for bit over the
    // update box (IsoPlan::coef_reuse): the CTA then takes those planes' A from one tile pinned before the march.
    const unsigned char *reuse;
    int pin_x;
};

constexpr int ceil4(int v) { return (v + 3) / 4 * 4; }
constexpr int align32f(int v) { return (v + 31) / 32 * 32; }   // 128-byte multiples in floats

// Ring layout: the u[t] planes live in a ring of exactly Q = 2R+1 stages, so that inside the
// loop body (unrolled Q times) every shared-memory address is a compile-time offset; plane j
// sits in stage j % Q, and the R planes beyond the one being read for output are the prefetch
// depth. The (u[t-1], A[, B]) tiles of output step s use a second, shorter ring of NS >= R+1
// stages indexed at run time (two loads per iteration only). One full/empty mbarrier pair per
// u-stage covers both: the tiles of step s = j-2R travel with plane j.
template <int R, int TY, int TZ4, int PK>
struct IsoTmaCfg {
    static constexpr int RZ = ceil4(R);
    static constexpr int TZ = 4 * TZ4;
    static constexpr int BY = TY + 2 * R;
    static constexpr int BZ = TZ + 2 * RZ;
    static constexpr int Q = 2 * R + 1;
    static constexpr int NU = Q;
    static constexpr int NS = R + 1;
    static constexpr int PLANE = align32f(BY * BZ);
    static constexpr int TILE = TY * TZ;
    static constexpr int NCW = TY * TZ4 / 32;          // consumer warps
    static constexpr int NTILES = 2 + (PK != B2_PARAM_SCALAR ? 1 : 0);   // prev, A, [B]
    // scalar parameter: the pinned A tile, its mbarrier and one reuse flag per tile-ring stage
    static constexpr int PIN = PK == B2_PARAM_SCALAR ? TILE : 0;
    static constexpr size_t SMEM = (size_t)(NU * PLANE + NS * TILE * NTILES + PIN) * 4 + 2 * NU * 8 +
                                   (PK == B2_PARAM_SCALAR ? 8 + NS * 4 : 0) + 128;
    static_assert(SMEM <= 227 * 1024, "k_iso_tma: shared memory over the 227 KB of one SM");
};

__device__ __forceinline__ float4 f4add(float4 a, float4 b) {
    return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}
__device__ __forceinline__ float4 f4sub(float4 a, float4 b) {
    return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w);
}
__device__ __forceinline__ void f4fma(float4 &acc, float w, float4 v) {
    acc.x = fmaf(w, v.x, acc.x);
    acc.y = fmaf(w, v.y, acc.y);
    acc.z = fmaf(w, v.z, acc.z);
    acc.w = fmaf(w, v.w, acc.w);
}

template <int R, int TY, int TZ4, int PK>
__global__ void __launch_bounds__(TY *TZ4 + 32, 1)
k_iso_tma(const __grid_constant__ CUtensorMap tm_uh, const __grid_constant__ CUtensorMap tm_uc,
          const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
          const IsoTK<R> k) {
    using C = IsoTmaCfg<R, TY, TZ4, PK>;
    constexpr int RZ = C::RZ, TZ = C::TZ, BZ = C::BZ, NU = C::NU, NS = C::NS, Q = C::Q;
    constexpr int PLANE = C::PLANE, TILE = C::TILE, NCW = C::NCW;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *s_u = reinterpret_cast<float *>(smem_raw);
    float *s_prev = s_u + NU * PLANE;
    float *s_a = s_prev + NS * TILE;
    float *s_b = s_a + NS * TILE;                 // array vp|m: the B ring
    float *s_pin = s_b;                           // scalar: the pinned A tile (my_prev + 2 NS TILE)
    uint64_t *full = reinterpret_cast<uint64_t *>(s_b + (PK != B2_PARAM_SCALAR ? NS * TILE : C::PIN));
    uint64_t *empty = full + NU;
    uint64_t *pinbar = empty + NU;                            // scalar: the pinned tile's arrival
    int *s_reused = reinterpret_cast<int *>(pinbar + 1);      // scalar: per tile stage, A is the pinned tile
    const bool pin = PK == B2_PARAM_SCALAR && k.reuse != nullptr;

    int b = blockIdx.x;
    const int iz = b % k.ntz;
    b /= k.ntz;
    const int iy = b % k.nty;
    const int ix = b / k.nty;
    const int z0 = iz * TZ, y0 = iy * TY;
    const int xs = k.xlo + ix * k.lx;
    const int xe = min(xs + k.lx, k.xlo + k.xcount);
    const int NP = (xe - xs) + 2 * R;
    // plane j of the march sits at x = xb + dx * j (relative to the iteration origin); the output of
    // iteration j is the plane x = xb + dx * (j - R)
    const bool back = (ix == 0) && k.back0;
    const int dx = back ? -1 : 1;
    const int xb = back ? xe - 1 + R : xs - R;

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;

    if (tid == 0) {
        for (int i = 0; i < NU; ++i) {
            b2ptx::mbar_init(&full[i], 1);
            b2ptx::mbar_init(&empty[i], NCW);
        }
        if (PK == B2_PARAM_SCALAR) b2ptx::mbar_init(pinbar, 1);
        b2ptx::fence_mbar_init();
    }
    __syncthreads();

    if (warp == NCW) {
        // ---------------- producer warp: one lane drives the TMA engine ----------------
        if (lane == 0) {
            b2ptx::tma_prefetch_desc(&tm_uh);
            b2ptx::tma_prefetch_desc(&tm_uc);
            b2ptx::tma_prefetch_desc(&tm_a);
            if (PK != B2_PARAM_SCALAR) b2ptx::tma_prefetch_desc(&tm_b);
            if (pin) {
                b2ptx::mbar_arrive_expect_tx(pinbar, TILE * 4);
                b2ptx::tma_load_3d(s_pin, &tm_a, pinbar, k.oz + z0, k.oy + y0, k.pin_x);
            }
            int slot = 0, round = 0, ss = 0;
            bool need_lo = k.want >= 0 && k.flag_lo != nullptr, need_hi = k.want >= 0 && k.flag_hi != nullptr;
            for (int j = 0; j < NP; ++j) {
                if (round > 0) b2ptx::mbar_wait(&empty[slot], (round - 1) & 1);
                const int s = j - 2 * R;
                const int xj = xb + dx * j;
                // a plane the neighbour GPU owns: it stored it into our halo at the end of its previous
                // step and then released the flag; acquire it once, then let the TMA engine read
                if (need_lo && xj < 0) {
                    while (b2ptx::ld_acquire_sys(k.flag_lo) < k.want) __nanosleep(40);
                    b2ptx::fence_proxy_async_global();
                    need_lo = false;
                }
                if (need_hi && xj >= k.nown) {
                    while (b2ptx::ld_acquire_sys(k.flag_hi) < k.want) __nanosleep(40);
                    b2ptx::fence_proxy_async_global();
                    need_hi = false;
                }
                const int xo = xj - dx * R;      // output plane of step s
                bool reused = false;
                uint32_t bytes = C::BY * BZ * 4;
                if (s >= 0) {
                    // the flag travels to the consumers with the stage: the arrive below releases it
                    reused = pin && __ldg(k.reuse + k.ox + xo) != 0;
                    if (PK == B2_PARAM_SCALAR) s_reused[ss] = reused;
                    bytes += TILE * 4 * (C::NTILES - (reused ? 1 : 0));
                }
                b2ptx::mbar_arrive_expect_tx(&full[slot], bytes);
                b2ptx::tma_load_4d(s_u + slot * PLANE, &tm_uh, &full[slot], k.oz + z0 - RZ,
                                   k.oy + y0 - R, k.ox + xj, k.slot0);
                if (s >= 0) {
                    b2ptx::tma_load_4d(s_prev + ss * TILE, &tm_uc, &full[slot], k.oz + z0,
                                       k.oy + y0, k.ox + xo, k.slotm);
                    if (!reused)
                        b2ptx::tma_load_3d(s_a + ss * TILE, &tm_a, &full[slot], k.oz + z0, k.oy + y0,
                                           k.ox + xo);
                    if (PK != B2_PARAM_SCALAR)
                        b2ptx::tma_load_3d(s_b + ss * TILE, &tm_b, &full[slot], k.oz + z0,
                                           k.oy + y0, k.ox + xo);
                    if (++ss == NS) ss = 0;
                }
                if (++slot == NU) { slot = 0; ++round; }
            }
        }
        return;
    }

    // ---------------- consumers ----------------
    const int ty = tid / TZ4, tz4 = tid % TZ4;
    const int gy = y0 + ty, gz = z0 + 4 * tz4;
    const bool yok = gy < k.ny;
    const int zcnt = yok ? min(max(k.nz - gz, 0), 4) : 0;
    const float *my_col = s_u + (ty + R) * BZ + RZ + 4 * tz4;
    const float *my_prev = s_prev + ty * TZ + 4 * tz4;
    const long long rowoff = (long long)(k.oy + gy) * k.sy + (k.oz + gz);
    float *outp = k.u1 + (long long)(k.ox + xb - dx * R) * k.sx + rowoff;
    const long long osx = dx * k.sx;
    const bool fuse = (k.peer_lo != nullptr) | (k.peer_hi != nullptr);

    float4 q[Q];
#pragma unroll
    for (int i = 0; i < Q; ++i) q[i] = make_float4(0.f, 0.f, 0.f, 0.f);

    const float wc = k.wx[0] + k.wy[0] + k.wz[0];
    if (pin) b2ptx::mbar_wait(pinbar, 0);
    uint32_t par = 0;               // parity of the u-ring round
    int ssoff = 0;                  // float offset of the tile-ring slot of output step j-2R

    for (int jb = 0; jb < NP; jb += Q) {
#pragma unroll
        for (int p = 0; p < Q; ++p) {
            const int j = jb + p;
            if (j >= NP) break;
            b2ptx::mbar_wait(&full[p], par);
            q[p] = b2ptx::lds128(my_col + p * PLANE);

            if (j >= 2 * R) {
                constexpr int dummy = 0;
                (void)dummy;
                const int pc = (p - R + Q) % Q;                // stage of the centre plane j-R
                const float *cp = my_col + pc * PLANE;
                const float4 c = q[pc];
                // z direction: row segment [-RZ, 4+RZ) around my 4 points
                float zr[4 + 2 * RZ];
#pragma unroll
                for (int m = 0; m < RZ / 4; ++m) {
                    // the outermost segments are only partly used when R is not a multiple of 4
                    // (R = 6: two floats each side): 8-byte loads halve their shared-memory wavefronts
                    if (R % 4 == 2 && m == 0) {
                        const float2 l = *reinterpret_cast<const float2 *>(cp - RZ + 2);
                        zr[0] = 0.f; zr[1] = 0.f; zr[2] = l.x; zr[3] = l.y;
                    } else {
                        const float4 l = b2ptx::lds128(cp - RZ + 4 * m);
                        zr[4 * m + 0] = l.x; zr[4 * m + 1] = l.y; zr[4 * m + 2] = l.z; zr[4 * m + 3] = l.w;
                    }
                    if (R % 4 == 2 && m == RZ / 4 - 1) {
                        const float2 r = *reinterpret_cast<const float2 *>(cp + 4 + 4 * m);
                        zr[RZ + 4 + 4 * m + 0] = r.x; zr[RZ + 4 + 4 * m + 1] = r.y;
                        zr[RZ + 4 + 4 * m + 2] = 0.f; zr[RZ + 4 + 4 * m + 3] = 0.f;
                    } else {
                        const float4 r = b2ptx::lds128(cp + 4 + 4 * m);
                        zr[RZ + 4 + 4 * m + 0] = r.x; zr[RZ + 4 + 4 * m + 1] = r.y;
                        zr[RZ + 4 + 4 * m + 2] = r.z; zr[RZ + 4 + 4 * m + 3] = r.w;
                    }
                }
                zr[RZ + 0] = c.x; zr[RZ + 1] = c.y; zr[RZ + 2] = c.z; zr[RZ + 3] = c.w;
                float4 acc = make_float4(wc * c.x, wc * c.y, wc * c.z, wc * c.w);
#pragma unroll
                for (int i = 1; i <= R; ++i) {
                    acc.x = fmaf(k.wz[i], zr[RZ + 0 - i] + zr[RZ + 0 + i], acc.x);
                    acc.y = fmaf(k.wz[i], zr[RZ + 1 - i] + zr[RZ + 1 + i], acc.y);
                    acc.z = fmaf(k.wz[i], zr[RZ + 2 - i] + zr[RZ + 2 + i], acc.z);
                    acc.w = fmaf(k.wz[i], zr[RZ + 3 - i] + zr[RZ + 3 + i], acc.w);
                }
#pragma unroll
                for (int i = 1; i <= R; ++i) {
                    const float4 a = b2ptx::lds128(cp - i * BZ);
                    const float4 bb = b2ptx::lds128(cp + i * BZ);
                    f4fma(acc, k.wy[i], f4add(a, bb));
                }
#pragma unroll
                for (int i = 1; i <= R; ++i)
                    f4fma(acc, k.wx[i], f4add(q[(pc - i + Q) % Q], q[(pc + i) % Q]));

                const float4 pv = b2ptx::lds128(my_prev + ssoff);
                int aoff = NS * TILE + ssoff;
                if (PK == B2_PARAM_SCALAR && s_reused[ssoff / TILE]) aoff = 2 * NS * TILE;   // s_pin
                const float4 ca = b2ptx::lds128(my_prev + aoff);
                const float4 dcp = f4sub(c, pv);
                float4 o;
                if (PK == B2_PARAM_SCALAR) {
                    o.x = fmaf(ca.x, fmaf(k.m_dt2, dcp.x, acc.x), c.x);
                    o.y = fmaf(ca.y, fmaf(k.m_dt2, dcp.y, acc.y), c.y);
                    o.z = fmaf(ca.z, fmaf(k.m_dt2, dcp.z, acc.z), c.z);
                    o.w = fmaf(ca.w, fmaf(k.m_dt2, dcp.w, acc.w), c.w);
                } else {
                    const float4 cb = b2ptx::lds128(my_prev + (2 * NS * TILE) + ssoff);
                    o.x = fmaf(ca.x, acc.x, fmaf(cb.x, dcp.x, c.x));
                    o.y = fmaf(ca.y, acc.y, fmaf(cb.y, dcp.y, c.y));
                    o.z = fmaf(ca.z, acc.z, fmaf(cb.z, dcp.z, c.z));
                    o.w = fmaf(ca.w, acc.w, fmaf(cb.w, dcp.w, c.w));
                }
                float *dst = outp + (long long)j * osx;
                if (zcnt == 4) {
                    *reinterpret_cast<float4 *>(dst) = o;
                } else if (zcnt > 0) {
                    dst[0] = o.x;
                    if (zcnt > 1) dst[1] = o.y;
                    if (zcnt > 2) dst[2] = o.z;
                }
                if (fuse) {
                    // a boundary plane: the same 16 bytes also go into the neighbour's halo (NVLink)
                    const int xo = xb + dx * (j - R);
                    float *pd = nullptr;
                    if (k.peer_lo && xo < k.pw) pd = k.peer_lo + (k.off_lo + (long long)xo * k.sx + rowoff);
                    if (k.peer_hi && xo >= k.nown - k.pw) pd = k.peer_hi + (k.off_hi + (long long)xo * k.sx + rowoff);
                    if (pd) {
                        if (zcnt == 4) {
                            *reinterpret_cast<float4 *>(pd) = o;
                        } else if (zcnt > 0) {
                            pd[0] = o.x;
                            if (zcnt > 1) pd[1] = o.y;
                            if (zcnt > 2) pd[2] = o.z;
                        }
                    }
                }
                ssoff += TILE;
                if (ssoff == NS * TILE) ssoff = 0;
            }
            if (j >= R) {
                __syncwarp();
                if (lane == 0) b2ptx::mbar_arrive(&empty[(p - R + Q) % Q]);
            }
        }
        par ^= 1;
    }
}


// ------------------------------------------------------------------------------------------
// Two-level TMA sweep (so = 8, scalar parameter): one pass over HBM advances u[t] to u[t+1] AND u[t+2]
// ------------------------------------------------------------------------------------------
// A CTA owns a TY x TZ output tile and marches along x. Level 1 computes u[t+1] on the tile grown by R in y
// and z (24 x 72, the cells level 2's y/z taps reach), level 2 computes u[t+2] on the tile, R planes behind.
//   u[t]    : haloed 32 x 80 planes, TMA ring of Q = 2R+1 stages; every level-1 thread keeps its own
//             column's x-history in registers (q1), as k_iso_tma does
//   u[t-1]  : 24 x 72 tiles with the level-1 plane (ring of R+1 stages, like k_iso_tma's tile ring)
//   A       : 24 x 72 tiles likewise, or the pinned tile on the planes whose A repeats (IsoTK::reuse)
//   u[t+1]  : each level-1 plane is also written to a ring of R+2 shared planes (level 2's y/z taps); the
//             256 tile threads keep their own column's level-1 x-history in registers (q2), and level 2's
//             u[t-1] (= u[t]) is already in q1
// Level-1 values outside the update box are the halo's, which the caller guarantees to be zero (iso2_halo_zero).
// u[t+1] goes to its own slot, u[t+2] to a scratch slot: the pass never writes a cell another CTA may still read.
// Source injection of step t into u[t+1] is applied to the level-1 values (IsoInj entries of this CTA's region),
// so that level 2 reads u[t+1] exactly as the one-step loop leaves it; only the owning CTA stores a cell.
constexpr int I2R = 4, I2TY = 16, I2TZ4 = 16;
struct Iso2Cfg {
    static constexpr int R = I2R, RZ = 4, TY = I2TY, TZ4 = I2TZ4, TZ = 4 * TZ4;
    static constexpr int BY = TY + 4 * R, BZ = TZ + 4 * RZ;        // u[t] box: 32 x 80
    static constexpr int EY = TY + 2 * R, EZ = TZ + 2 * RZ;        // level-1 region: 24 x 72
    static constexpr int EZ4 = EZ / 4;
    static constexpr int Q = 2 * R + 1, NS = R + 1, NL = R + 2;
    static constexpr int PLANE = align32f(BY * BZ);
    static constexpr int EPL = EY * EZ;
    static constexpr int NTH1 = EY * EZ4;                          // level-1 threads (432)
    static constexpr int NCW = (NTH1 + 31) / 32;                   // consumer warps (14)
    static constexpr int NT = 32 * NCW + 32;
    static constexpr size_t SMEM = (size_t)(Q * PLANE + NL * EPL + 2 * NS * EPL + EPL) * 4 + 2 * Q * 8 + 8 +
                                   NS * 4 + B2_ISO2_MAX_INJ * sizeof(IsoInj) + 16 + 128;
    static_assert(SMEM <= 227 * 1024, "k_iso_tma2: shared memory over the 227 KB of one SM");
};

struct Iso2K {
    float *__restrict__ u1;       // base of u[t+1]'s slot
    float *__restrict__ u2;       // base of u[t+2]'s scratch slot
    const float *__restrict__ A;  // coefficient table (level 2 reads the planes whose A is not pinned)
    long long sx, sy;
    int nx, ny, nz;
    int ox, oy, oz;
    int lx, ntz, nty;
    int slot0, slotm;             // tensor-map time coordinates of u[t] and u[t-1]
    float m_dt2;
    float wx[I2R + 1], wy[I2R + 1], wz[I2R + 1];
    const unsigned char *reuse;
    int pin_x;
    const IsoInj *inj;
    int ninj;
};

// acc = centre + z, y, x taps in the order k_iso_tma sums them (bit-identical results)
__device__ __forceinline__ float4 iso2_lap(const float *cp, int bz, float4 c, const float4 *q, int pc, float wc,
                                          const float *wx, const float *wy, const float *wz) {
    constexpr int R = I2R, RZ = 4, Q = 2 * R + 1;
    float zr[4 + 2 * RZ];
    const float4 l = b2ptx::lds128(cp - RZ);
    const float4 r = b2ptx::lds128(cp + 4);
    zr[0] = l.x; zr[1] = l.y; zr[2] = l.z; zr[3] = l.w;
    zr[RZ + 0] = c.x; zr[RZ + 1] = c.y; zr[RZ + 2] = c.z; zr[RZ + 3] = c.w;
    zr[RZ + 4] = r.x; zr[RZ + 5] = r.y; zr[RZ + 6] = r.z; zr[RZ + 7] = r.w;
    float4 acc = make_float4(wc * c.x, wc * c.y, wc * c.z, wc * c.w);
#pragma unroll
    for (int i = 1; i <= R; ++i) {
        acc.x = fmaf(wz[i], zr[RZ + 0 - i] + zr[RZ + 0 + i], acc.x);
        acc.y = fmaf(wz[i], zr[RZ + 1 - i] + zr[RZ + 1 + i], acc.y);
        acc.z = fmaf(wz[i], zr[RZ + 2 - i] + zr[RZ + 2 + i], acc.z);
        acc.w = fmaf(wz[i], zr[RZ + 3 - i] + zr[RZ + 3 + i], acc.w);
    }
#pragma unroll
    for (int i = 1; i <= R; ++i) f4fma(acc, wy[i], f4add(b2ptx::lds128(cp - i * bz), b2ptx::lds128(cp + i * bz)));
#pragma unroll
    for (int i = 1; i <= R; ++i) f4fma(acc, wx[i], f4add(q[(pc - i + Q) % Q], q[(pc + i) % Q]));
    return acc;
}

__device__ __forceinline__ float4 iso2_update(float4 c, float4 pv, float4 ca, float4 acc, float m_dt2) {
    const float4 d = f4sub(c, pv);
    return make_float4(fmaf(ca.x, fmaf(m_dt2, d.x, acc.x), c.x), fmaf(ca.y, fmaf(m_dt2, d.y, acc.y), c.y),
                       fmaf(ca.z, fmaf(m_dt2, d.z, acc.z), c.z), fmaf(ca.w, fmaf(m_dt2, d.w, acc.w), c.w));
}

__device__ __forceinline__ void iso2_store(float *dst, float4 o, int zcnt) {
    if (zcnt == 4) {
        *reinterpret_cast<float4 *>(dst) = o;
    } else if (zcnt > 0) {
        dst[0] = o.x;
        if (zcnt > 1) dst[1] = o.y;
        if (zcnt > 2) dst[2] = o.z;
    }
}

__global__ void __launch_bounds__(Iso2Cfg::NT, 1)
k_iso_tma2(const __grid_constant__ CUtensorMap tm_uh, const __grid_constant__ CUtensorMap tm_uc,
           const __grid_constant__ CUtensorMap tm_a, const Iso2K k) {
    using C = Iso2Cfg;
    constexpr int R = C::R, RZ = C::RZ, TY = C::TY, TZ = C::TZ, BZ = C::BZ, EZ = C::EZ, EZ4 = C::EZ4;
    constexpr int Q = C::Q, NS = C::NS, NL = C::NL, PLANE = C::PLANE, EPL = C::EPL, NCW = C::NCW;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *s_u = reinterpret_cast<float *>(smem_raw);
    float *s_l1 = s_u + Q * PLANE;
    float *s_prev = s_l1 + NL * EPL;
    float *s_a = s_prev + NS * EPL;
    float *s_pin = s_a + NS * EPL;
    uint64_t *full = reinterpret_cast<uint64_t *>(s_pin + EPL);
    uint64_t *empty = full + Q;
    uint64_t *pinbar = empty + Q;
    int *s_reused = reinterpret_cast<int *>(pinbar + 1);
    IsoInj *s_inj = reinterpret_cast<IsoInj *>(s_reused + NS + (NS & 1));
    int *s_ninj = reinterpret_cast<int *>(s_inj + B2_ISO2_MAX_INJ);
    const bool pin = k.reuse != nullptr;

    int b = blockIdx.x;
    const int iz = b % k.ntz;
    b /= k.ntz;
    const int iy = b % k.nty;
    const int ix = b / k.nty;
    const int z0 = iz * TZ, y0 = iy * TY;
    const int xs = ix * k.lx;
    const int xe = min(xs + k.lx, k.nx);
    // plane j of the march is x = xs - 2R + j; iteration j computes level 1 on x - R = xs - 3R + j and
    // level 2 on xs - 4R + j
    const int NP = (xe - xs) + 4 * R;

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;

    if (tid == 0) {
        for (int i = 0; i < Q; ++i) {
            b2ptx::mbar_init(&full[i], 1);
            b2ptx::mbar_init(&empty[i], NCW);
        }
        b2ptx::mbar_init(pinbar, 1);
        b2ptx::fence_mbar_init();
        // the injection entries that land in this CTA's level-1 region
        int n = 0;
        for (int i = 0; i < k.ninj; ++i) {
            const IsoInj e = k.inj[i];
            if (e.x >= xs - R && e.x < xe + R && e.y >= y0 - R && e.y < y0 + TY + R && e.z >= z0 - RZ &&
                e.z < z0 + TZ + RZ)
                s_inj[n++] = e;
        }
        *s_ninj = n;
    }
    __syncthreads();

    if (warp == NCW) {
        if (lane == 0) {
            b2ptx::tma_prefetch_desc(&tm_uh);
            b2ptx::tma_prefetch_desc(&tm_uc);
            b2ptx::tma_prefetch_desc(&tm_a);
            if (pin) {
                b2ptx::mbar_arrive_expect_tx(pinbar, EPL * 4);
                b2ptx::tma_load_3d(s_pin, &tm_a, pinbar, k.oz + z0 - RZ, k.oy + y0 - R, k.pin_x);
            }
            int slot = 0, round = 0, ss = 0;
            for (int j = 0; j < NP; ++j) {
                if (round > 0) b2ptx::mbar_wait(&empty[slot], (round - 1) & 1);
                const int x1 = xs - 3 * R + j;                     // level-1 plane of iteration j
                bool reused = false;
                uint32_t bytes = C::BY * BZ * 4;
                if (j >= 2 * R) {
                    reused = pin && __ldg(k.reuse + k.ox + x1) != 0;
                    s_reused[ss] = reused;
                    bytes += EPL * 4 * (reused ? 1 : 2);
                }
                b2ptx::mbar_arrive_expect_tx(&full[slot], bytes);
                b2ptx::tma_load_4d(s_u + slot * PLANE, &tm_uh, &full[slot], k.oz + z0 - 2 * RZ, k.oy + y0 - 2 * R,
                                   k.ox + xs - 2 * R + j, k.slot0);
                if (j >= 2 * R) {
                    b2ptx::tma_load_4d(s_prev + ss * EPL, &tm_uc, &full[slot], k.oz + z0 - RZ, k.oy + y0 - R,
                                       k.ox + x1, k.slotm);
                    if (!reused)
                        b2ptx::tma_load_3d(s_a + ss * EPL, &tm_a, &full[slot], k.oz + z0 - RZ, k.oy + y0 - R,
                                           k.ox + x1);
                    if (++ss == NS) ss = 0;
                }
                if (++slot == Q) { slot = 0; ++round; }
            }
        }
        return;
    }

    // ---------------- consumers: thread -> (ey, ec) of the level-1 region ----------------
    // threads [0, 256): the output tile (level 1 and level 2, whole warps); then the y-halo rows, then the two
    // z-halo columns; threads >= NTH1 only take part in the barriers
    int ey, ec;
    if (tid < TY * C::TZ4) {
        ey = R + tid / C::TZ4; ec = 1 + tid % C::TZ4;
    } else if (tid < TY * C::TZ4 + 2 * R * EZ4) {
        const int h = tid - TY * C::TZ4, r = h / EZ4;
        ey = r < R ? r : r + TY; ec = h % EZ4;
    } else {
        const int h = tid - TY * C::TZ4 - 2 * R * EZ4;
        ey = R + h / 2; ec = (h & 1) ? EZ4 - 1 : 0;
    }
    const bool active = tid < C::NTH1;
    const bool inner = tid < TY * C::TZ4;
    if (!active) { ey = 0; ec = 0; }
    const int gy = y0 - R + ey, gz = z0 - RZ + 4 * ec;             // relative to the iteration origin
    const bool yin = gy >= 0 && gy < k.ny;
    // components of my float4 inside the update box along z (level-1 values outside the box are the halo's: 0)
    const bool zin0 = yin && gz + 0 >= 0 && gz + 0 < k.nz, zin1 = yin && gz + 1 >= 0 && gz + 1 < k.nz;
    const bool zin2 = yin && gz + 2 >= 0 && gz + 2 < k.nz, zin3 = yin && gz + 3 >= 0 && gz + 3 < k.nz;
    const int zcnt = inner && yin ? min(max(k.nz - gz, 0), 4) : 0;
    const float *my_col = s_u + (ey + R) * BZ + RZ + 4 * ec;
    const int eoff = ey * EZ + 4 * ec;
    const long long rowoff = (long long)(k.oy + gy) * k.sy + (k.oz + gz);
    const int ninj = *s_ninj;

    float4 q1[Q], q2[Q];
#pragma unroll
    for (int i = 0; i < Q; ++i) { q1[i] = make_float4(0.f, 0.f, 0.f, 0.f); q2[i] = q1[i]; }

    const float wc = k.wx[0] + k.wy[0] + k.wz[0];
    if (pin) b2ptx::mbar_wait(pinbar, 0);
    uint32_t par = 0;
    int ss = 0;                     // tile-ring stage of the level-1 plane
    int l1w = 0, l1r = R % NL;      // s_l1 stage of level-1 plane j - 2R (written) / j - 3R (read by level 2)
    unsigned pinned = 0;            // bit i: the level-1 plane of iteration j - i took A from the pinned tile

    for (int jb = 0; jb < NP; jb += Q) {
#pragma unroll
        for (int p = 0; p < Q; ++p) {
            const int j = jb + p;
            if (j >= NP) break;
            b2ptx::mbar_wait(&full[p], par);
            q1[p] = b2ptx::lds128(my_col + p * PLANE);

            if (j >= 2 * R) {
                const int x1 = xs - 3 * R + j;
                const int pc = (p - R + Q) % Q;
                const float4 c = q1[pc];
                const float4 acc = iso2_lap(my_col + pc * PLANE, BZ, c, q1, pc, wc, k.wx, k.wy, k.wz);
                const float4 pv = b2ptx::lds128(s_prev + ss * EPL + eoff);
                const int reused = s_reused[ss];
                pinned = (pinned << 1) | (unsigned)reused;
                const float4 ca = b2ptx::lds128((reused ? s_pin : s_a + ss * EPL) + eoff);
                float4 o = iso2_update(c, pv, ca, acc, k.m_dt2);
                const bool xin = x1 >= 0 && x1 < k.nx;
                o.x = xin && zin0 ? o.x : 0.f;
                o.y = xin && zin1 ? o.y : 0.f;
                o.z = xin && zin2 ? o.z : 0.f;
                o.w = xin && zin3 ? o.w : 0.f;
                for (int i = 0; i < ninj; ++i) {
                    const IsoInj e = s_inj[i];
                    if (e.x == x1 && e.y == gy && e.z >= gz && e.z < gz + 4) {
                        const int cz = e.z - gz;
                        if (cz == 0) o.x += e.v;
                        else if (cz == 1) o.y += e.v;
                        else if (cz == 2) o.z += e.v;
                        else o.w += e.v;
                    }
                }
                if (active) *reinterpret_cast<float4 *>(s_l1 + l1w * EPL + eoff) = o;
                q2[p] = o;
                if (x1 >= xs && x1 < xe) iso2_store(k.u1 + (long long)(k.ox + x1) * k.sx + rowoff, o, zcnt);
                if (++ss == NS) ss = 0;
                if (++l1w == NL) l1w = 0;
            }
            if (j >= R) {
                __syncwarp();
                if (lane == 0) b2ptx::mbar_arrive(&empty[(p - R + Q) % Q]);
            }
            if (j >= 4 * R) {
                // level-1 plane x2 (written R iterations ago) is complete in s_l1; the barrier also orders this
                // iteration's level-1 store after every read of its stage (two iterations ago)
                asm volatile("bar.sync 1, %0;" ::"n"(NCW * 32) : "memory");
                if (zcnt > 0) {
                    const int x2 = xs - 4 * R + j;
                    const int pc2 = (p - R + Q) % Q;
                    const float4 c = q2[pc2];
                    const float4 acc = iso2_lap(s_l1 + l1r * EPL + eoff, EZ, c, q2, pc2, wc, k.wx, k.wy, k.wz);
                    float4 ca;
                    if ((pinned >> R) & 1u)
                        ca = b2ptx::lds128(s_pin + eoff);
                    else
                        ca = __ldg(reinterpret_cast<const float4 *>(k.A + (long long)(k.ox + x2) * k.sx + rowoff));
                    const float4 o = iso2_update(c, q1[(p + 1) % Q], ca, acc, k.m_dt2);
                    iso2_store(k.u2 + (long long)(k.ox + x2) * k.sx + rowoff, o, zcnt);
                }
                if (++l1r == NL) l1r = 0;
            }
        }
        par ^= 1;
    }
}

// A = 1/(m/dt^2 + damp/dt), B = m/dt^2 * A on the full allocated array (halo included; halo
// values are never used by the stencil)
__global__ void __launch_bounds__(256)
k_iso_coef(const float *__restrict__ damp, const float *__restrict__ param, int param_kind,
           float m_dt2_scalar, float inv_dt, float inv_dt2, float *__restrict__ A,
           float *__restrict__ B, size_t n) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        float md = m_dt2_scalar;
        if (param_kind == B2_PARAM_VP) {
            const float v = param[i];
            md = inv_dt2 / (v * v);
        } else if (param_kind == B2_PARAM_M) {
            md = param[i] * inv_dt2;
        }
        const float a = 1.0f / (md + damp[i] * inv_dt);
        A[i] = a;
        if (B) B[i] = md * a;
    }
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
// tile configuration per radius (TY, TZ4) and coefficient kind (ARR: an array vp|m streams a third tile):
// sized so that the Q-stage plane ring plus the (R+1)-stage tile ring fit the 227 KB of shared memory of one SM.
// so=8 with a scalar vp: 16 x 128, so that every TMA box row and every warp's store is 512 contiguous bytes
// rather than 256 (profiles/h100_iso_probe.json: the sweep's stream mix copies 7 % faster with 512-byte rows);
// with an array vp|m the third tile ring does not fit beside the 16 x 128 plane ring, and it keeps 32 x 64.
template <int R, bool ARR> struct TileOf;
template <bool ARR> struct TileOf<2, ARR> { static constexpr int TY = 32, TZ4 = 16; };
template <> struct TileOf<4, false> { static constexpr int TY = 16, TZ4 = 32; };
template <> struct TileOf<4, true> { static constexpr int TY = 32, TZ4 = 16; };
template <bool ARR> struct TileOf<6, ARR> { static constexpr int TY = 16, TZ4 = 16; };
template <bool ARR> struct TileOf<8, ARR> { static constexpr int TY = 8, TZ4 = 16; };

// scratch for the coefficient arrays, cached across calls: A, B (TMA path), W (OT4)
static ScratchSlot g_coef[3];

// rows [y0, y1) of the planes [x0, x1) (allocated indices): the y-skewed streamed loop tabulates row blocks
__global__ void __launch_bounds__(256)
k_iso_coef_rows(const float *__restrict__ damp, const float *__restrict__ param, int param_kind, float m_dt2_scalar,
                float inv_dt, float inv_dt2, float *__restrict__ A, float *__restrict__ B, long long sx, int a2,
                int x0, int y0, int ny) {
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    if (z >= a2) return;
    const int x = x0 + blockIdx.z;
    for (int y = y0 + blockIdx.y; y < y0 + ny; y += gridDim.y) {
        const size_t i = (size_t)x * (size_t)sx + (size_t)y * a2 + z;
        float md = m_dt2_scalar;
        if (param_kind == B2_PARAM_VP) {
            const float v = param[i];
            md = inv_dt2 / (v * v);
        } else if (param_kind == B2_PARAM_M) {
            md = param[i] * inv_dt2;
        }
        const float a = 1.0f / (md + damp[i] * inv_dt);
        A[i] = a;
        if (B) B[i] = md * a;
    }
}

int iso_coef_tabulate_rows(const IsoPlan &p, int x0, int x1, int y0, int y1) {
    if (x1 <= x0 || y1 <= y0) return B2_OK;
    const float inv_dt = 1.0f / p.dt, inv_dt2 = 1.0f / (p.dt * p.dt);
    const float md = (1.0f / (p.vp * p.vp)) * inv_dt2;
    dim3 block(256, 1, 1), grid((p.a[2] + 255) / 256, (unsigned)std::min(y1 - y0, 1024), (unsigned)(x1 - x0));
    k_iso_coef_rows<<<grid, block, 0, stream()>>>(p.damp, p.param, p.param_kind, md, inv_dt, inv_dt2, p.coefA, p.coefB,
                                                  p.sx, p.a[2], x0, y0, y1 - y0);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

// tabulate the allocated x-planes [plane_lo, plane_hi) (the streamed time loop does it chunk by chunk, as
// the damping / parameter planes arrive from the host)
int iso_coef_tabulate_planes(const IsoPlan &p, int plane_lo, int plane_hi) {
    if (plane_hi <= plane_lo) return B2_OK;
    const float inv_dt = 1.0f / p.dt, inv_dt2 = 1.0f / (p.dt * p.dt);
    const float md = (1.0f / (p.vp * p.vp)) * inv_dt2;
    const size_t off = (size_t)plane_lo * (size_t)p.sx, cnt = (size_t)(plane_hi - plane_lo) * (size_t)p.sx;
    B2_SM_COUNT(sms);
    k_iso_coef<<<sms * 8, 256, 0, stream()>>>(p.damp + off, p.param ? p.param + off : nullptr, p.param_kind, md, inv_dt,
                                               inv_dt2, p.coefA + off, p.coefB ? p.coefB + off : nullptr, cnt);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

// A over the whole allocated array (scalar parameter), and the reuse flags of the planes in the update box: a warp
// whose damp row segment differs in any bit from the pin plane's (inside the box's rows and columns) clears its
// plane's flag. The pin plane (4 B/point once) stays in L2 while every plane compares against it.
__global__ void __launch_bounds__(256)
k_iso_coef_scan(const float *__restrict__ damp, float m_dt2, float inv_dt, float *__restrict__ A,
                unsigned char *__restrict__ reuse, long long sx, int a0, int a1, int a2, int xpin, int xlo, int xhi,
                int ylo, int yhi, int zlo, int zhi) {
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    const bool zin = z < a2;
    for (int x = blockIdx.z; x < a0; x += gridDim.z) {
        const bool cmp = zin && x >= xlo && x < xhi && z >= zlo && z < zhi;
        bool differ = false;
        for (int y = blockIdx.y; y < a1; y += gridDim.y) {
            if (!zin) continue;
            const size_t row = (size_t)y * a2 + z;
            const float d = damp[(size_t)x * (size_t)sx + row];
            A[(size_t)x * (size_t)sx + row] = 1.0f / (m_dt2 + d * inv_dt);
            if (cmp && y >= ylo && y < yhi)
                differ |= __float_as_uint(d) != __float_as_uint(damp[(size_t)xpin * (size_t)sx + row]);
        }
        if (__any_sync(0xffffffffu, differ) && (threadIdx.x & 31) == 0) reuse[x] = 0;
    }
}

// one byte per allocated x-plane, cached across calls; g_reuse_n: planes the last iso call flagged (0: none)
static unsigned char *g_reuse = nullptr;
static int g_reuse_cap = 0, g_reuse_n = 0;

int iso_coef_tabulate_all(IsoPlan &p) {
    if (p.param_kind != B2_PARAM_SCALAR) return iso_coef_tabulate_planes(p, 0, p.a[0]);
    if (g_reuse_cap < p.a[0]) {
        if (g_reuse) cudaFree(g_reuse);
        g_reuse = nullptr;
        g_reuse_cap = 0;
        B2_CUDA(cudaMalloc(&g_reuse, (size_t)p.a[0]), B2_ERR_MEMORY);
        g_reuse_cap = p.a[0];
    }
    // 1 on the planes of the update box, 0 elsewhere; the scan clears the planes that differ
    B2_CUDA(cudaMemsetAsync(g_reuse, 0, (size_t)p.a[0], stream()), B2_ERR_LAUNCH);
    B2_CUDA(cudaMemsetAsync(g_reuse + p.o[0], 1, (size_t)p.n[0], stream()), B2_ERR_LAUNCH);
    const float inv_dt = 1.0f / p.dt, inv_dt2 = 1.0f / (p.dt * p.dt);
    const float md = (1.0f / (p.vp * p.vp)) * inv_dt2;
    dim3 block(256, 1, 1), grid((p.a[2] + 255) / 256, (unsigned)std::min(p.a[1], 64), (unsigned)std::min(p.a[0], 65535));
    k_iso_coef_scan<<<grid, block, 0, stream()>>>(p.damp, md, inv_dt, p.coefA, g_reuse, p.sx, p.a[0], p.a[1], p.a[2],
                                                  p.o[0] + p.n[0] / 2, p.o[0], p.o[0] + p.n[0], p.o[1],
                                                  p.o[1] + p.n[1], p.o[2], p.o[2] + p.n[2]);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    p.coef_reuse = g_reuse;
    g_reuse_n = p.a[0];
    return B2_OK;
}

int iso_coef_reuse_count() {
    if (g_reuse_n <= 0) return 0;
    std::vector<unsigned char> h((size_t)g_reuse_n);
    if (cudaMemcpyAsync(h.data(), g_reuse, h.size(), cudaMemcpyDeviceToHost, stream()) != cudaSuccess ||
        cudaStreamSynchronize(stream()) != cudaSuccess) {
        set_error("b2_last_iso_coef_reuse: reading the flags back failed");
        return -1;
    }
    int n = 0;
    for (unsigned char f : h) n += f != 0;
    return n;
}

static int iso_coef_tabulate(IsoPlan &p) {
    int rc;
    if ((rc = cached_scratch(g_coef[0], p.slot_elems, &p.coefA))) return rc;
    p.coefB = nullptr;
    if (p.param_kind != B2_PARAM_SCALAR)
        if ((rc = cached_scratch(g_coef[1], p.slot_elems, &p.coefB))) return rc;
    if (p.defer_coef) return B2_OK;          // the caller tabulates plane ranges itself
    return iso_coef_tabulate_all(p);
}

template <int R>
static int plan_tma(IsoPlan &p) {
    const bool arr = p.param_kind != B2_PARAM_SCALAR;
    const int TY = arr ? TileOf<R, true>::TY : TileOf<R, false>::TY;
    const int TZ4 = arr ? TileOf<R, true>::TZ4 : TileOf<R, false>::TZ4;
    constexpr int RZ = ceil4(R);
    const int dims4[4] = {p.a[2], p.a[1], p.a[0], p.tsize};
    const int dims3[3] = {p.a[2], p.a[1], p.a[0]};
    int rc;
    if ((rc = encode_tmap(&p.tm_uh, p.u, 4, dims4, 4 * TZ4 + 2 * RZ, TY + 2 * R, "iso"))) return rc;
    if ((rc = encode_tmap(&p.tm_uc, p.u, 4, dims4, 4 * TZ4, TY, "iso"))) return rc;
    if ((rc = encode_tmap(&p.tm_damp, p.coefA, 3, dims3, 4 * TZ4, TY, "iso"))) return rc;
    if (arr) {
        if ((rc = encode_tmap(&p.tm_par, p.coefB, 3, dims3, 4 * TZ4, TY, "iso"))) return rc;
    } else {
        p.tm_par = p.tm_damp;
    }
    return B2_OK;
}

int iso_plan_init(IsoPlan &p, int kernel) {
    p.coef_reuse = nullptr;
    g_reuse_n = 0;
    const int R = p.radius[2];
    bool ok = (p.radius[0] == R && p.radius[1] == R) && (R == 2 || R == 4 || R == 6 || R == 8);
    ok = ok && p.damp != nullptr;
    ok = ok && (p.a[2] % 4 == 0) && (p.o[2] % 4 == 0);
    ok = ok && ((uintptr_t)p.u % 16 == 0) && ((uintptr_t)p.damp % 16 == 0);
    ok = ok && (p.param_kind == B2_PARAM_SCALAR || (uintptr_t)p.param % 16 == 0);
    ok = ok && (p.slot_elems % 4 == 0);
    // tiny grids gain nothing from the pipelined kernel
    ok = ok && (p.n[1] >= 8 && p.n[2] >= 16);
    if (kernel == 1) ok = false;
    if (p.ot4) {
        // two-pass generic path: W = lap(u)/m over the box grown by R, then the update with lap(W)
        if (kernel == 2) { set_error("iso: the OT4 kernel has no TMA variant yet"); return B2_ERR_INVALID; }
        for (int d = 0; d < 3; ++d) {
            const int rd = p.radius[d];
            if (p.o[d] - 2 * rd < 0 || p.o[d] + p.n[d] - 1 + 2 * rd >= p.a[d]) {
                set_error("iso: OT4 needs a halo of 2*radius = %d points on dim %d", 2 * rd, d);
                return B2_ERR_INVALID;
            }
        }
        p.use_tma = false;
        return cached_scratch(g_coef[2], p.slot_elems, &p.ot4W);
    }
    if (kernel == 2 && !ok) {
        set_error("iso: TMA kernel forced but layout does not qualify (radius=%d a2=%d o2=%d)", R,
                  p.a[2], p.o[2]);
        return B2_ERR_INVALID;
    }
    p.use_tma = ok;
    if (!ok) return B2_OK;
    int rc = iso_coef_tabulate(p);
    if (rc) return rc;
    switch (R) {
        case 2: return plan_tma<2>(p);
        case 4: return plan_tma<4>(p);
        case 6: return plan_tma<6>(p);
        case 8: return plan_tma<8>(p);
    }
    return B2_ERR_INVALID;
}

template <int R, int PK>
static int launch_tma(const IsoPlan &p, int slot0, int slotm, int slot1, int xlo, int xcount,
                      const IsoFuse *fz = nullptr) {
    using T = TileOf<R, PK != B2_PARAM_SCALAR>;
    using C = IsoTmaCfg<R, T::TY, T::TZ4, PK>;
    auto kern = k_iso_tma<R, T::TY, T::TZ4, PK>;
    // the shared-memory size is opted into once, before the kernel's first launch
    static bool attr_set = false;
    if (!attr_set) {
        B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM),
                B2_ERR_LAUNCH);
        attr_set = true;
    }
    IsoTK<R> k;
    k.u1 = p.u + (size_t)slot1 * p.slot_elems;
    k.sx = p.sx;
    k.sy = p.sy;
    k.ny = p.n[1];
    k.nz = p.n[2];
    k.ox = p.o[0];
    k.oy = p.o[1];
    k.oz = p.o[2];
    k.xlo = xlo;
    k.xcount = xcount;
    k.ntz = (p.n[2] + C::TZ - 1) / C::TZ;
    k.nty = (p.n[1] + T::TY - 1) / T::TY;
    // x-chunk length: whole waves over the SMs, but chunks of at least 32 planes
    int lx = env_int("B2_ISO_LX", 0);
    if (lx <= 0) {
        B2_SM_COUNT(sms);
        lx = choose_chunk_len(sms, k.ntz * k.nty, xcount, 2 * R, 32);
    }
    lx = std::min(lx, xcount);
    // fused halo step with neighbours on both sides: at least two chunks, so that the one marching down
    // to x = 0 and the one marching up to x = n-1 each meet the neighbour's planes at their end
    if (fz && (fz->peer_lo || fz->flag_lo) && (fz->peer_hi || fz->flag_hi) && lx >= xcount && xcount >= 4 * R)
        lx = (xcount + 1) / 2;
    k.lx = lx;
    const int ntx = (xcount + lx - 1) / lx;
    k.back0 = 0; k.nown = p.n[0]; k.pw = R;
    k.peer_lo = k.peer_hi = nullptr;
    k.off_lo = k.off_hi = 0;
    k.flag_lo = k.flag_hi = nullptr;
    k.want = -1;
    if (fz) {
        const long long plane = p.sx;
        k.back0 = (fz->peer_lo || fz->flag_lo) ? 1 : 0;
        k.peer_lo = fz->peer_lo;
        k.peer_hi = fz->peer_hi;
        // my owned plane x mirrors plane (halo + n_lo + x) of the low neighbour / (halo - nown + x) of the high one
        k.off_lo = (long long)slot1 * fz->slot_lo + (long long)(p.o[0] + fz->n_lo) * plane;
        k.off_hi = (long long)slot1 * fz->slot_hi + (long long)(p.o[0] - p.n[0]) * plane;
        k.flag_lo = fz->flag_lo;
        k.flag_hi = fz->flag_hi;
        k.want = fz->want;
    }
    k.reuse = PK == B2_PARAM_SCALAR ? p.coef_reuse : nullptr;
    k.pin_x = p.o[0] + p.n[0] / 2;
    k.slot0 = slot0;
    k.slotm = slotm;
    k.m_dt2 = (1.0f / (p.vp * p.vp)) * (1.0f / (p.dt * p.dt));
    for (int i = 0; i <= R; ++i) {
        k.wx[i] = p.w[0][i];
        k.wy[i] = p.w[1][i];
        k.wz[i] = p.w[2][i];
    }
    const unsigned grid = (unsigned)(k.ntz * k.nty * ntx);
    const char *pk = PK == B2_PARAM_VP ? "vp" : (PK == B2_PARAM_M ? "m" : "scalar");
    timing_begin();
    kern<<<grid, T::TY * T::TZ4 + 32, C::SMEM, stream()>>>(p.tm_uh, p.tm_uc, p.tm_damp, p.tm_par, k);
    note_sweep_kernel("iso_tma<%d,%s>", R, pk);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

template <int R>
static int launch_tma_pk(const IsoPlan &p, int s0, int sm, int s1, int xlo, int xcount, const IsoFuse *fz = nullptr) {
    switch (p.param_kind) {
        case B2_PARAM_SCALAR: return launch_tma<R, B2_PARAM_SCALAR>(p, s0, sm, s1, xlo, xcount, fz);
        case B2_PARAM_VP: return launch_tma<R, B2_PARAM_VP>(p, s0, sm, s1, xlo, xcount, fz);
        case B2_PARAM_M: return launch_tma<R, B2_PARAM_M>(p, s0, sm, s1, xlo, xcount, fz);
    }
    return B2_ERR_INVALID;
}

static IsoGK generic_args(const IsoPlan &p, int slot0, int slotm, int slot1, int xlo, int xcount) {
    IsoGK k;
    k.u0 = p.u + (size_t)slot0 * p.slot_elems;
    k.um = p.u + (size_t)slotm * p.slot_elems;
    k.u1 = p.u + (size_t)slot1 * p.slot_elems;
    k.damp = p.damp;
    k.param = p.param;
    k.sx = p.sx;
    k.sy = p.sy;
    k.n0 = xcount;
    k.n1 = p.n[1];
    k.n2 = p.n[2];
    k.o0 = p.o[0] + xlo;
    k.o1 = p.o[1];
    k.o2 = p.o[2];
    k.r0 = p.radius[0];
    k.r1 = p.radius[1];
    k.r2 = p.radius[2];
    k.param_kind = p.param_kind;
    k.inv_dt = 1.0f / p.dt;
    k.inv_dt2 = 1.0f / (p.dt * p.dt);
    k.m_dt2 = (1.0f / (p.vp * p.vp)) * k.inv_dt2;
    memcpy(k.w, p.w, sizeof(k.w));
    k.W = nullptr;
    k.ot4c = p.dt * p.dt / 12.0f;
    k.vp2 = p.vp * p.vp;
    k.U1 = nullptr;
    k.dm = nullptr;
    k.dsx = k.dsy = 0;
    k.dg0 = k.dg1 = k.dg2 = 0;
    return k;
}

int iso_born_source(const IsoPlan &p, int slot0, int slotm, int slot1, float *U1, const float *dm,
                    long long dsx, long long dsy, int dg0, int dg1, int dg2) {
    IsoGK k = generic_args(p, slot0, slotm, slot1, 0, p.n[0]);
    k.U1 = U1;
    k.dm = dm;
    k.dsx = dsx; k.dsy = dsy;
    k.dg0 = dg0; k.dg1 = dg1; k.dg2 = dg2;
    dim3 block(64, 4, 1);
    dim3 grid((k.n2 + 63) / 64, (k.n1 + 3) / 4, (unsigned)std::min(k.n0, 65535));
    k_born_src<<<grid, block, 0, stream()>>>(k);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

int iso_fs_fix(const IsoPlan &p, int slot0, int slotm, int slot1, int xlo, int xcount) {
    if (xcount <= 0) return B2_OK;
    if (p.n[2] <= 2 * p.radius[2]) {
        set_error("free surface: the vertical extent %d is too small for radius %d", p.n[2], p.radius[2]);
        return B2_ERR_INVALID;
    }
    IsoGK k = generic_args(p, slot0, slotm, slot1, xlo, xcount);
    dim3 block(16, 16, 1);
    dim3 grid((k.n1 + 15) / 16, (unsigned)std::min(xcount, 65535), 1);
    k_iso_fs_fix<<<grid, block, 0, stream()>>>(k);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

int iso_step_fused(const IsoPlan &p, int slot0, int slotm, int slot1, const IsoFuse &f) {
    if (!p.use_tma) { set_error("iso: the fused halo step needs the TMA sweep kernel"); return B2_ERR_INVALID; }
    switch (p.radius[2]) {
        case 2: return launch_tma_pk<2>(p, slot0, slotm, slot1, 0, p.n[0], &f);
        case 4: return launch_tma_pk<4>(p, slot0, slotm, slot1, 0, p.n[0], &f);
        case 6: return launch_tma_pk<6>(p, slot0, slotm, slot1, 0, p.n[0], &f);
        case 8: return launch_tma_pk<8>(p, slot0, slotm, slot1, 0, p.n[0], &f);
    }
    return B2_ERR_INVALID;
}

bool iso2_supported(const IsoPlan &p) {
    return p.use_tma && !p.ot4 && p.tsize == 3 && p.param_kind == B2_PARAM_SCALAR && p.radius[0] == I2R &&
           p.radius[1] == I2R && p.radius[2] == I2R && p.n[0] >= 1;
}

// scratch slots of the two-level pass, cached like g_coef; g_s2_box: the array extents and update box they are zero
// outside of
static float *g_s2 = nullptr;
static size_t g_s2_elems = 0;
static int g_s2_box[9] = {-1, -1, -1, -1, -1, -1, -1, -1, -1};
static CUtensorMap g_s2_tm_uh, g_s2_tm_uh_s, g_s2_tm_uc, g_s2_tm_a;

int iso2_reserve(const IsoPlan &p, bool &ok) {
    ok = true;
    if (g_s2_elems == p.slot_elems) return B2_OK;
    if (g_s2) cudaFree(g_s2);
    g_s2 = nullptr;
    g_s2_elems = 0;
    if (cudaMalloc(&g_s2, 2 * p.slot_elems * sizeof(float)) != cudaSuccess) {
        cudaGetLastError();                  // an allocation failure is not sticky: clear it, run one step per sweep
        g_s2 = nullptr;
        ok = false;
        return B2_OK;
    }
    g_s2_elems = p.slot_elems;
    g_s2_box[0] = -1;
    return B2_OK;
}

int iso2_prepare(const IsoPlan &p, float *scratch[2]) {
    using C = Iso2Cfg;
    if (g_s2_elems != p.slot_elems) { set_error("iso2_prepare: scratch not reserved"); return B2_ERR_INVALID; }
    const int box[9] = {p.a[0], p.a[1], p.a[2], p.o[0], p.o[1], p.o[2], p.n[0], p.n[1], p.n[2]};
    if (memcmp(box, g_s2_box, sizeof(box)) != 0) {
        // the pass writes only the update box: everything else stays the zero halo the slots hold
        B2_CUDA(cudaMemsetAsync(g_s2, 0, 2 * p.slot_elems * sizeof(float), stream()), B2_ERR_MEMORY);
        memcpy(g_s2_box, box, sizeof(box));
    }
    const int dims4[4] = {p.a[2], p.a[1], p.a[0], p.tsize};
    const int dims4s[4] = {p.a[2], p.a[1], p.a[0], 2};
    const int dims3[3] = {p.a[2], p.a[1], p.a[0]};
    int rc;
    if ((rc = encode_tmap(&g_s2_tm_uh, p.u, 4, dims4, C::BZ, C::BY, "iso"))) return rc;
    if ((rc = encode_tmap(&g_s2_tm_uh_s, g_s2, 4, dims4s, C::BZ, C::BY, "iso"))) return rc;
    if ((rc = encode_tmap(&g_s2_tm_uc, p.u, 4, dims4, C::EZ, C::EY, "iso"))) return rc;
    if ((rc = encode_tmap(&g_s2_tm_a, p.coefA, 3, dims3, C::EZ, C::EY, "iso"))) return rc;
    scratch[0] = g_s2;
    scratch[1] = g_s2 + p.slot_elems;
    return B2_OK;
}

// one warp per (slot, x, y) row: rows outside the box in x or y are checked whole, the others outside [o2, o2 + n2)
__global__ void __launch_bounds__(256)
k_iso2_halo_nonzero(const float *__restrict__ u, size_t slot_elems, long long sx, int a0, int a1, int a2, int o0,
                    int o1, int o2, int n0, int n1, int n2, int *flag) {
    const long long rows = 3LL * a0 * a1;
    const int lane = threadIdx.x & 31;
    bool nz = false;
    for (long long r = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; r < rows;
         r += (gridDim.x * (long long)blockDim.x) >> 5) {
        const int s = (int)(r / ((long long)a0 * a1));
        const int xy = (int)(r % ((long long)a0 * a1));
        const int x = xy / a1, y = xy % a1;
        const float *row = u + s * slot_elems + (size_t)x * sx + (size_t)y * a2;
        const bool inside = x >= o0 && x < o0 + n0 && y >= o1 && y < o1 + n1;
        for (int z = lane; z < a2; z += 32) {
            if (inside && z >= o2 && z < o2 + n2) continue;
            nz |= row[z] != 0.f;
        }
    }
    if (__any_sync(0xffffffffu, nz) && lane == 0) atomicOr(flag, 1);
}

int iso2_halo_nonzero(const IsoPlan &p, int *flag) {
    B2_SM_COUNT(sms);
    k_iso2_halo_nonzero<<<sms * 8, 256, 0, stream()>>>(p.u, p.slot_elems, p.sx, p.a[0], p.a[1], p.a[2], p.o[0],
                                                        p.o[1], p.o[2], p.n[0], p.n[1], p.n[2], flag);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

int iso_step2(const IsoPlan &p, int slot0, int src_scratch, int slotm, int slot1, int dst_scratch, const IsoInj *inj,
              int ninj) {
    using C = Iso2Cfg;
    static bool attr_set = false;
    if (!attr_set) {
        B2_CUDA(cudaFuncSetAttribute(k_iso_tma2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM),
                B2_ERR_LAUNCH);
        attr_set = true;
    }
    Iso2K k;
    k.u1 = p.u + (size_t)slot1 * p.slot_elems;
    k.u2 = g_s2 + (size_t)dst_scratch * p.slot_elems;
    k.A = p.coefA;
    k.sx = p.sx;
    k.sy = p.sy;
    k.nx = p.n[0]; k.ny = p.n[1]; k.nz = p.n[2];
    k.ox = p.o[0]; k.oy = p.o[1]; k.oz = p.o[2];
    k.ntz = (p.n[2] + C::TZ - 1) / C::TZ;
    k.nty = (p.n[1] + C::TY - 1) / C::TY;
    int lx = env_int("B2_ISO_LX", 0);
    if (lx <= 0) {
        B2_SM_COUNT(sms);
        lx = choose_chunk_len(sms, k.ntz * k.nty, p.n[0], 4 * C::R, 32);
    }
    k.lx = std::min(lx, p.n[0]);
    const int ntx = (p.n[0] + k.lx - 1) / k.lx;
    k.slot0 = src_scratch < 0 ? slot0 : src_scratch;
    k.slotm = slotm;
    k.m_dt2 = (1.0f / (p.vp * p.vp)) * (1.0f / (p.dt * p.dt));
    for (int i = 0; i <= C::R; ++i) {
        k.wx[i] = p.w[0][i];
        k.wy[i] = p.w[1][i];
        k.wz[i] = p.w[2][i];
    }
    k.reuse = p.coef_reuse;
    k.pin_x = p.o[0] + p.n[0] / 2;
    k.inj = inj;
    k.ninj = ninj;
    const unsigned grid = (unsigned)(k.ntz * k.nty * ntx);
    timing_begin();
    k_iso_tma2<<<grid, C::NT, C::SMEM, stream()>>>(src_scratch < 0 ? g_s2_tm_uh : g_s2_tm_uh_s, g_s2_tm_uc,
                                                   g_s2_tm_a, k);
    note_sweep_kernel("iso_tma2<%d,scalar>", C::R);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

int iso_step(const IsoPlan &p, int slot0, int slotm, int slot1, int xlo, int xcount) {
    if (xcount <= 0) return B2_OK;
    if (p.use_tma) {
        switch (p.radius[2]) {
            case 2: return launch_tma_pk<2>(p, slot0, slotm, slot1, xlo, xcount);
            case 4: return launch_tma_pk<4>(p, slot0, slotm, slot1, xlo, xcount);
            case 6: return launch_tma_pk<6>(p, slot0, slotm, slot1, xlo, xcount);
            case 8: return launch_tma_pk<8>(p, slot0, slotm, slot1, xlo, xcount);
        }
        return B2_ERR_INVALID;
    }
    IsoGK k = generic_args(p, slot0, slotm, slot1, xlo, xcount);
    if (p.ot4) {
        IsoGK g = k;                       // first pass on the box grown by the radius
        g.W = p.ot4W;
        g.o0 -= g.r0; g.o1 -= g.r1; g.o2 -= g.r2;
        g.n0 += 2 * g.r0; g.n1 += 2 * g.r1; g.n2 += 2 * g.r2;
        dim3 blk(64, 4, 1);
        dim3 grd((g.n2 + 63) / 64, (g.n1 + 3) / 4, (unsigned)std::min(g.n0, 65535));
        k_ot4_w<<<grd, blk, 0, stream()>>>(g);
        count_launch();
        B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
        k.W = p.ot4W;
    }
    dim3 block(64, 4, 1);
    dim3 grid((k.n2 + 63) / 64, (k.n1 + 3) / 4, (unsigned)std::min(xcount, 65535));
    timing_begin();
    note_sweep_kernel("iso_generic");
    k_iso_generic<<<grid, block, 0, stream()>>>(k);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

}  // namespace b2
