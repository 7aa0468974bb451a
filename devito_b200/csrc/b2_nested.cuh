// The nested operator L of b2_nested_point.cuh as a 2.5-D TMA sweep along x for 3-D grids, R in {2, 4}, shared by the
// self-adjoint update (b2_sa.cu, SaEpi) and the SLS viscoacoustic update (b2_visco.cu, ViscoEpi<ADJ>); the two differ
// only in the epilogue that turns L at a point into the levels written.
//
//   k_nested_tma<R, Epi> : a CTA owns a (TY x TZ) yz-tile and marches along x over an x-chunk; a producer warp streams,
//                          per plane, the plane of f (the field L is applied to) with a (2R-1)-wide y/z halo and the b
//                          plane with an R-wide halo into a shared-memory ring with TMA, signalled on mbarriers. Each
//                          consumer thread owns four consecutive z points: it keeps F_x of the 2R planes the outer
//                          x-difference needs in a register queue (one F_x per plane, from the ring's centre columns),
//                          forms F_y and F_z of its own points from the ring in registers (no CTA barrier: every thread
//                          reads only the ring) and hands L at its four points to the epilogue.
//
// An epilogue is a functor passed to the kernel by value, with
//   __device__ void operator()(float4 acc, const float *U, int ucol, int bcol, long long off, int zcnt) const
// acc: L at the thread's four points; U: the ring slot of their plane (f at U + ucol, b at U + bcol); off: the global
// index of the first point; zcnt: how many of the four lie in the box (1..4; the sweep calls it only when some do).
//
// The host side the two updates share: the plan base NestedPlan, its set-up nested_plan_init (kernel choice, TMA
// eligibility, b expanded into scratch, the tensor maps), and the launches launch_nested_tma and
// launch_nested_generic. What is left to an update is its own arrays, tables, epilogue and injection scale.
#pragma once
#include "b2_common.cuh"
#include "b2_ptx.cuh"
#include <algorithm>
#include <initializer_list>

namespace b2 {

template <int R> struct NestedCfg {
    static constexpr int TY = 16, TZ4 = 16, TZ = 4 * TZ4;
    static constexpr int HU = 2 * R - 1;                  // reach of the nested stencil: the f halo in y
    static constexpr int RZU = (HU + 3) / 4 * 4;          // ... and in z, rounded up to 16 bytes
    static constexpr int RZB = (R + 3) / 4 * 4;           // the b halo in z (R in y)
    static constexpr int BYU = TY + 2 * HU, BZU = TZ + 2 * RZU;
    static constexpr int BYB = TY + 2 * R, BZB = TZ + 2 * RZB;
    static constexpr int UPL = (BYU * BZU + 31) / 32 * 32;    // floats, every TMA destination 128-byte aligned
    static constexpr int BPL = (BYB * BZB + 31) / 32 * 32;
    static constexpr int SLOT = UPL + BPL;
    // planes in flight: the 2R planes the consumers still read, plus the producer's lead
    static constexpr int LEAD = R == 2 ? 4 : 2;
    static constexpr int NU = 2 * R + LEAD;
    static constexpr int NCW = TY * TZ4 / 32;             // consumer warps
    static constexpr size_t SMEM = (size_t)NU * SLOT * 4 + 2 * NU * 8 + 128;
};

// the sweep's geometry: the box, its x-chunks and tiles, and the weights
template <int R> struct NestedGeo {
    long long sx, sy;
    int ny, nz, ox, oy, oz;
    int xlo, xcount, lx, ntz, nty;
    int slot0;                       // slot of f in its tensor map: the 4th coordinate
    float cx[R], cy[R], cz[R];
};

__device__ __forceinline__ float4 f4fma(float w, float4 v, float4 acc) {
    return make_float4(fmaf(w, v.x, acc.x), fmaf(w, v.y, acc.y), fmaf(w, v.z, acc.z), fmaf(w, v.w, acc.w));
}
__device__ __forceinline__ float4 f4sub(float4 a, float4 b) {
    return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w);
}
__device__ __forceinline__ float4 f4mul(float4 a, float4 b) {
    return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
}
__device__ __forceinline__ float4 ldg4(const float *p) {
    return __ldg(reinterpret_cast<const float4 *>(p));
}

// The kernel's argument: the epilogue's operands, then the geometry, in one struct. (Passed as two arguments, the R = 4
// viscoacoustic forward sweep compiles to 168 registers with spills rather than 156 without.)
template <int R, class Epi> struct NestedArgs {
    Epi epi;
    NestedGeo<R> geo;
};

template <int R, class Epi>
__global__ void __launch_bounds__(NestedCfg<R>::TY * NestedCfg<R>::TZ4 + 32, 1)
k_nested_tma(const __grid_constant__ CUtensorMap tm_f, const __grid_constant__ CUtensorMap tm_b,
             const NestedArgs<R, Epi> args) {
    const NestedGeo<R> &k = args.geo;
    using Cf = NestedCfg<R>;
    constexpr int TY = Cf::TY, TZ4 = Cf::TZ4, TZ = Cf::TZ, HU = Cf::HU, RZU = Cf::RZU, RZB = Cf::RZB;
    constexpr int BZU = Cf::BZU, BZB = Cf::BZB, UPL = Cf::UPL, SLOT = Cf::SLOT, NU = Cf::NU, NCW = Cf::NCW;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *ring = reinterpret_cast<float *>(smem_raw);
    uint64_t *full = reinterpret_cast<uint64_t *>(ring + NU * SLOT);
    uint64_t *empty = full + NU;

    int blk = blockIdx.x;
    const int iz = blk % k.ntz;
    blk /= k.ntz;
    const int iy = blk % k.nty;
    const int ix = blk / k.nty;
    const int z0 = iz * TZ, y0 = iy * TY;
    const int xs = k.xlo + ix * k.lx;
    const int xe = min(xs + k.lx, k.xlo + k.xcount);
    // march index a reads the plane x = xb + a; F_x of plane a - R is formed on its arrival and plane a - 2R + 1 is
    // written (it needs F_x of the planes up to a - R)
    const int NP = (xe - xs) + 4 * R - 2;
    const int xb = xs - (2 * R - 1);

    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int i = 0; i < NU; ++i) {
            b2ptx::mbar_init(&full[i], 1);
            b2ptx::mbar_init(&empty[i], NCW);
        }
        b2ptx::fence_mbar_init();
    }
    __syncthreads();

    if (warp == NCW) {
        // ---------------- producer warp: one lane drives the TMA engine ----------------
        if (lane == 0) {
            b2ptx::tma_prefetch_desc(&tm_f);
            b2ptx::tma_prefetch_desc(&tm_b);
            for (int j = 0; j < NP; ++j) {
                const int slot = j % NU, round = j / NU;
                if (round > 0) b2ptx::mbar_wait(&empty[slot], (round - 1) & 1);
                b2ptx::mbar_arrive_expect_tx(&full[slot], (uint32_t)(Cf::BYU * BZU + Cf::BYB * BZB) * 4);
                float *dst = ring + slot * SLOT;
                b2ptx::tma_load_4d(dst, &tm_f, &full[slot], k.oz + z0 - RZU, k.oy + y0 - HU, k.ox + xb + j, k.slot0);
                b2ptx::tma_load_3d(dst + UPL, &tm_b, &full[slot], k.oz + z0 - RZB, k.oy + y0 - R, k.ox + xb + j);
            }
        }
        return;
    }

    // ---------------- consumers ----------------
    const int ty = tid / TZ4, tz4 = tid % TZ4;
    const int gy = y0 + ty, gz = z0 + 4 * tz4;
    const int zcnt = gy < k.ny ? min(max(k.nz - gz, 0), 4) : 0;
    const int ucol = (ty + HU) * BZU + RZU + 4 * tz4;          // my four points in an f plane
    const int bcol = UPL + (ty + R) * BZB + RZB + 4 * tz4;     // ... in a b plane
    const long long rowoff = (long long)(k.oy + gy) * k.sy + (k.oz + gz);

    float4 fx[2 * R];                                          // fx[i] = F_x(plane p - R + i), p the plane written
#pragma unroll
    for (int i = 0; i < 2 * R; ++i) fx[i] = make_float4(0.f, 0.f, 0.f, 0.f);

    for (int a = 0; a < NP; ++a) {
        b2ptx::mbar_wait(&full[a % NU], (a / NU) & 1);
        if (a >= 2 * R - 1) {
            // F_x at plane q = a - R from the centre columns of planes q - R + 1 .. q + R
            const int q = a - R;
            float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int i = 1; i <= R; ++i) {
                const float4 hi = b2ptx::lds128(ring + ((q + i) % NU) * SLOT + ucol);
                const float4 lo = b2ptx::lds128(ring + ((q - i + 1) % NU) * SLOT + ucol);
                s = f4fma(k.cx[i - 1], f4sub(hi, lo), s);
            }
            const float4 bq = b2ptx::lds128(ring + (q % NU) * SLOT + bcol);
#pragma unroll
            for (int i = 0; i < 2 * R - 1; ++i) fx[i] = fx[i + 1];
            fx[2 * R - 1] = f4mul(bq, s);
        }
        if (a >= 4 * R - 2) {
            const int p = a - 2 * R + 1;
            const float *U = ring + (p % NU) * SLOT;
            // x: sum_k c_k (F_x(p + k - 1) - F_x(p - k))
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int i = 1; i <= R; ++i) acc = f4fma(k.cx[i - 1], f4sub(fx[R + i - 1], fx[R - i]), acc);
            // y: F_y at the rows ty - R .. ty + R - 1 from my columns of rows ty - 2R + 1 .. ty + 2R - 1
            {
                float4 uc[4 * R - 1];
#pragma unroll
                for (int m = 0; m < 4 * R - 1; ++m) uc[m] = b2ptx::lds128(U + ucol + (m - (2 * R - 1)) * BZU);
#pragma unroll
                for (int j = -R; j < R; ++j) {
                    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    for (int i = 1; i <= R; ++i)
                        s = f4fma(k.cy[i - 1], f4sub(uc[j + i + 2 * R - 1], uc[j - i + 1 + 2 * R - 1]), s);
                    const float4 fy = f4mul(b2ptx::lds128(U + bcol + j * BZB), s);
                    acc = f4fma(j >= 0 ? k.cy[j] : -k.cy[-j - 1], fy, acc);
                }
            }
            // z: F_z at the columns 4 tz4 - R .. 4 tz4 + 3 + R - 1 of row ty
            {
                float zr[4 + 2 * RZU], br[4 + 2 * RZB], fz[2 * R + 3];
                const float *zrow = U + (ty + HU) * BZU + 4 * tz4;         // column 4 tz4 - RZU
                const float *brow = U + UPL + (ty + R) * BZB + 4 * tz4;    // column 4 tz4 - RZB
#pragma unroll
                for (int g = 0; g < (4 + 2 * RZU) / 4; ++g) {
                    const float4 v = b2ptx::lds128(zrow + 4 * g);
                    zr[4 * g] = v.x; zr[4 * g + 1] = v.y; zr[4 * g + 2] = v.z; zr[4 * g + 3] = v.w;
                }
#pragma unroll
                for (int g = 0; g < (4 + 2 * RZB) / 4; ++g) {
                    const float4 v = b2ptx::lds128(brow + 4 * g);
                    br[4 * g] = v.x; br[4 * g + 1] = v.y; br[4 * g + 2] = v.z; br[4 * g + 3] = v.w;
                }
#pragma unroll
                for (int e = -R; e < R + 3; ++e) {
                    float s = 0.f;
#pragma unroll
                    for (int i = 1; i <= R; ++i) s = fmaf(k.cz[i - 1], zr[RZU + e + i] - zr[RZU + e - i + 1], s);
                    fz[e + R] = br[RZB + e] * s;
                }
                float oz[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    float s = 0.f;
#pragma unroll
                    for (int i = 1; i <= R; ++i) s = fmaf(k.cz[i - 1], fz[c + i - 1 + R] - fz[c - i + R], s);
                    oz[c] = s;
                }
                acc.x += oz[0]; acc.y += oz[1]; acc.z += oz[2]; acc.w += oz[3];
            }
            if (zcnt > 0) args.epi(acc, U, ucol, bcol, (long long)(k.ox + xb + p) * k.sx + rowoff, zcnt);
        }
        // plane a - 2R + 1 is read no more: hand its slot back to the producer
        if (a >= 2 * R - 1) {
            __syncwarp();
            if (lane == 0) b2ptx::mbar_arrive(&empty[(a - 2 * R + 1) % NU]);
        }
    }
}

// The tensor maps of k_nested_tma<R> over box p's allocation: the haloed plane of f (`fslots` slots, the slot the 4th
// coordinate) and the haloed plane of b. `who` names the caller in an encoding error.
template <int R>
int nested_maps(const Box &p, const float *f, int fslots, const float *b, CUtensorMap &tm_f, CUtensorMap &tm_b,
                const char *who) {
    using Cf = NestedCfg<R>;
    const int dims[4] = {p.a[2], p.a[1], p.a[0], fslots};
    int rc;
    if ((rc = encode_tmap(&tm_f, f, 4, dims, Cf::BZU, Cf::BYU, who))) return rc;
    return encode_tmap(&tm_b, b, 3, dims, Cf::BZB, Cf::BYB, who);
}

// What the plans of the self-adjoint update (SaPlan) and the SLS update (ViscoPlan) share. The box: a 2-D grid is
// (1, x, y) with radius 0 on dim 0.
struct NestedPlan : Box {
    int radius[3] = {0, 0, 0};
    float c[3][B2_MAX_RADIUS] = {};          // c[d][k-1] = c_k / h_d
    float dt = 0.f;
    bool adjoint = false;
    // b and vp: an array in the wavefield's space layout, or the scalar next to it
    const float *b_arr = nullptr, *vp_arr = nullptr;
    float b_value = 1.f, vp_value = 1.f;
    float *b = nullptr;                      // b_arr, or library scratch that the update's table kernel fills
    // <name>_tma<R> (3-D, R in {2, 4}, z rows and the box start 16-byte aligned): tensor maps of the haloed plane of
    // the field f that L is applied to (every slot f has, the slot a coordinate) and of the haloed b plane
    bool use_tma = false;
    CUtensorMap tm_f, tm_b;
};

// The plan set-up both updates share, once p's box, radius, weights and parameters are set. Checks `kernel` (0 auto:
// the TMA sweep when the layout qualifies, 1 generic, 2 TMA: 210 with a message when it does not), points p.b at b_arr
// or at the scratch `bslot`, which the caller's table kernel fills with b_value, and encodes the maps of the TMA sweep
// over f (`fslots` slots). `aligned`: the caller's arrays that the sweep accesses 16 bytes at a time (b is checked
// here; library scratch comes from cudaMalloc and is aligned). Messages start with `who`.
inline int nested_plan_init(NestedPlan &p, int kernel, const char *who, ScratchSlot &bslot,
                            std::initializer_list<const void *> aligned, const float *f, int fslots) {
    if (kernel != 0 && kernel != 1 && kernel != 2) {
        set_error("%s: unknown kernel %d", who, kernel);
        return B2_ERR_INVALID;
    }
    // the TMA sweep: 3-D, R in {2, 4} on every axis, z rows and the box start 16-byte aligned (the conditions of
    // k_iso_tma: so % 4 == 0 and nz % 4 == 0 make the row pitch a multiple of 4 floats)
    const int R = p.radius[2];
    bool ok = p.radius[0] == R && p.radius[1] == R && (R == 2 || R == 4);
    ok = ok && p.a[2] % 4 == 0 && p.o[2] % 4 == 0 && p.slot_elems % 4 == 0 && (uintptr_t)p.b_arr % 16 == 0;
    for (const void *x : aligned) ok = ok && (uintptr_t)x % 16 == 0;
    if (kernel == 2 && !ok) {
        set_error("%s: TMA kernel forced but the layout does not qualify (3-D, radius 2 or 4, z extent and z start "
                  "multiples of 4, 16-byte aligned arrays; radius=%d a2=%d o2=%d)", who, R, p.a[2], p.o[2]);
        return B2_ERR_INVALID;
    }
    int rc;
    if (p.b_arr) {
        p.b = const_cast<float *>(p.b_arr);
    } else if ((rc = cached_scratch(bslot, p.slot_elems, &p.b))) {
        return rc;
    }
    p.use_tma = ok && kernel != 1;
    if (!p.use_tma) return B2_OK;
    return R == 2 ? nested_maps<2>(p, f, fslots, p.b, p.tm_f, p.tm_b, who)
                  : nested_maps<4>(p, f, fslots, p.b, p.tm_f, p.tm_b, who);
}

// One sweep of k_nested_tma<R, Epi> over plan p's box with its weights and maps, f at slot `slot0` of tm_f. The
// variant is noted as "<name>_tma<R>" (b2_last_sweep_kernel), with "+adj" on the adjoint.
template <int R, class Epi>
int launch_nested_tma(const NestedPlan &p, int slot0, const Epi &epi, const char *name) {
    using Cf = NestedCfg<R>;
    auto kern = k_nested_tma<R, Epi>;
    static bool attr_set = false;           // the shared-memory size is opted into before the first launch
    if (!attr_set) {
        B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cf::SMEM), B2_ERR_LAUNCH);
        attr_set = true;
    }
    NestedArgs<R, Epi> args;
    args.epi = epi;
    NestedGeo<R> &k = args.geo;
    k.sx = p.sx;
    k.sy = p.sy;
    k.ny = p.n[1];
    k.nz = p.n[2];
    k.ox = p.o[0];
    k.oy = p.o[1];
    k.oz = p.o[2];
    k.xlo = 0;
    k.xcount = p.n[0];
    k.ntz = (p.n[2] + Cf::TZ - 1) / Cf::TZ;
    k.nty = (p.n[1] + Cf::TY - 1) / Cf::TY;
    B2_SM_COUNT(sms);
    k.lx = std::min(choose_chunk_len(sms, k.ntz * k.nty, p.n[0], 4 * R - 2, 32), p.n[0]);
    k.slot0 = slot0;
    for (int i = 0; i < R; ++i) {
        k.cx[i] = p.c[0][i];
        k.cy[i] = p.c[1][i];
        k.cz[i] = p.c[2][i];
    }
    const int ntx = (p.n[0] + k.lx - 1) / k.lx;
    timing_begin();
    note_sweep_kernel("%s_tma<%d>%s", name, R, p.adjoint ? "+adj" : "");
    kern<<<k.ntz * k.nty * ntx, Cf::TY * Cf::TZ4 + 32, Cf::SMEM, stream()>>>(p.tm_f, p.tm_b, args);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

// One sweep of a one-thread-per-point kernel (k_sa_generic, k_visco_generic) over plan p's box: fills the members its
// argument K shares with the others (strides, box, radius and weights; the caller sets the rest) and launches 64 x 4
// threads per block on z and y, blocks looping over x. The variant is noted as "<name>_generic", with "+adj" on the
// adjoint.
template <class K>
int launch_nested_generic(void (*kern)(K), K k, const NestedPlan &p, const char *name) {
    k.sx = p.sx;
    k.sy = p.sy;
    k.n0 = p.n[0]; k.n1 = p.n[1]; k.n2 = p.n[2];
    k.o0 = p.o[0]; k.o1 = p.o[1]; k.o2 = p.o[2];
    for (int d = 0; d < 3; ++d) {
        k.r[d] = p.radius[d];
        for (int i = 0; i < B2_MAX_RADIUS; ++i) k.c[d][i] = p.c[d][i];
    }
    dim3 block(64, 4, 1);
    dim3 grid((k.n2 + 63) / 64, (k.n1 + 3) / 4, (unsigned)std::min(k.n0, 65535));
    timing_begin();
    note_sweep_kernel("%s_generic%s", name, p.adjoint ? "+adj" : "");
    kern<<<grid, block, 0, stream()>>>(k);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

}  // namespace b2
