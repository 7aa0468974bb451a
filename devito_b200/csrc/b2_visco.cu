// Second-order SLS viscoacoustic update (the reference's `sls_2nd_order`, examples/seismic/viscoacoustic/
// operators.py:124-192). Scheme and tables: b2_visco_point.cuh.
//
//   k_visco_coef     : once per call, the tables Kd, Kg, Kt, W, Wm over the whole allocated slot into library scratch
//                      (from vp, b, qp, f0, dt and damp, each an array or a scalar), so that the sweeps have one form
//                      for scalar and array parameters; a scalar b is expanded into scratch too.
//   k_visco_adj_mix  : adjoint only, pointwise over the whole allocated slot, halo included: r[t-1] inside the box and
//                      s = ((1 + tt) p[t] + r[t-1]) / b everywhere, because the sweep reads s up to 2R-1 outside the
//                      box. L is linear, so the reference's two nested terms L((1+tt) rho p) + L(rho r[t-1]) are L(s).
//   k_visco_generic  : one thread per point, any even space order <= 16, 2-D and 3-D, any alignment. Its point body is
//                      b2_visco_point.cuh (run on the CPU by tests/support/emu_visco.cu, with the tables and the mix).
//   k_visco_tma<R,A> : 2.5-D sweep along x for 3-D grids, R in {2, 4}, with the structure of k_sa_tma<R>: a producer
//                      warp streams the haloed plane of the field L is applied to (p[t], or s on the adjoint) and the
//                      haloed b plane through a TMA ring; each consumer thread keeps F_x of 2R planes in registers,
//                      forms F_y and F_z of its four z points in registers and runs the epilogue of
//                      b2_visco_point.cuh with 16-byte loads and stores. The flux stage is a copy of k_sa_tma's, not
//                      shared with it (DESIGN §3.3k).
//
// Algorithmic bytes per point and step (DESIGN §3.3k): forward 44 (p[t], b, p[t-1], r[t], five tables; writes r[t+1],
// p[t+1]); adjoint 64 (the mix reads p[t], r[t], Kd, Kg, Kt, b and writes r[t-1], s: 32; the sweep reads s, b, p[t],
// p[t+1], Kd, W, Wm and writes p[t-1]: 32).
#include "b2_visco.cuh"
#include "b2_ptx.cuh"
#include <algorithm>
#include <cmath>

namespace b2 {

__global__ void __launch_bounds__(256) k_visco_generic(ViscoK k) {
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (z >= k.n2 || y >= k.n1) return;
    for (int x = blockIdx.z; x < k.n0; x += gridDim.z) visco_point(k, x, y, z);
}

__global__ void __launch_bounds__(256) k_visco_adj_mix(ViscoMixK k) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < k.n; i += (size_t)gridDim.x * blockDim.x)
        visco_mix_at(k, i);
}

// ------------------------------------------------------------------------------------------
// 2.5-D TMA sweep
// ------------------------------------------------------------------------------------------
template <int R> struct ViscoTmaCfg {
    static constexpr int TY = 16, TZ4 = 16, TZ = 4 * TZ4;
    static constexpr int HU = 2 * R - 1;                  // reach of the nested stencil: the field's halo in y
    static constexpr int RZU = (HU + 3) / 4 * 4;          // ... and in z, rounded up to 16 bytes
    static constexpr int RZB = (R + 3) / 4 * 4;           // the b halo in z (R in y)
    static constexpr int BYU = TY + 2 * HU, BZU = TZ + 2 * RZU;
    static constexpr int BYB = TY + 2 * R, BZB = TZ + 2 * RZB;
    static constexpr int UPL = (BYU * BZU + 31) / 32 * 32;    // floats, every TMA destination 128-byte aligned
    static constexpr int BPL = (BYB * BZB + 31) / 32 * 32;
    static constexpr int SLOT = UPL + BPL;
    static constexpr int LEAD = R == 2 ? 4 : 2;
    static constexpr int NU = 2 * R + LEAD;
    static constexpr int NCW = TY * TZ4 / 32;             // consumer warps
    static constexpr size_t SMEM = (size_t)NU * SLOT * 4 + 2 * NU * 8 + 128;
};

template <int R> struct ViscoTK {
    const float *p0, *pm;            // p[t], p[t - dir] slots (p[t] read on the adjoint only: the ring holds s)
    float *p1;                       // p[t + dir] slot
    const float *r0;                 // r[t] slot (forward)
    float *r1;                       // r[t+1] slot (forward)
    const float *K[VK_NTAB];
    long long sx, sy;
    int ny, nz, ox, oy, oz;
    int xlo, xcount, lx, ntz, nty;
    int slot0;                       // slot of the field in the ring's tensor map: the 4th coordinate
    float cx[R], cy[R], cz[R];
};

__device__ __forceinline__ float4 vk_f4fma(float w, float4 v, float4 acc) {
    return make_float4(fmaf(w, v.x, acc.x), fmaf(w, v.y, acc.y), fmaf(w, v.z, acc.z), fmaf(w, v.w, acc.w));
}
__device__ __forceinline__ float4 vk_f4sub(float4 a, float4 b) {
    return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w);
}
__device__ __forceinline__ float4 vk_f4mul(float4 a, float4 b) {
    return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
}
__device__ __forceinline__ float4 vk_ldg4(const float *p) {
    return __ldg(reinterpret_cast<const float4 *>(p));
}
#define VK_AT(v, c) ((c) == 0 ? (v).x : (c) == 1 ? (v).y : (c) == 2 ? (v).z : (v).w)

template <int R, bool ADJ>
__global__ void __launch_bounds__(ViscoTmaCfg<R>::TY * ViscoTmaCfg<R>::TZ4 + 32, 1)
k_visco_tma(const __grid_constant__ CUtensorMap tm_f, const __grid_constant__ CUtensorMap tm_b, const ViscoTK<R> k) {
    using Cf = ViscoTmaCfg<R>;
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
    const int ucol = (ty + HU) * BZU + RZU + 4 * tz4;          // my four points in a field plane
    const int bcol = UPL + (ty + R) * BZB + RZB + 4 * tz4;     // ... in a b plane
    const long long rowoff = (long long)(k.oy + gy) * k.sy + (k.oz + gz);

    float4 fx[2 * R];                                          // fx[i] = F_x(plane p - R + i), p the plane written
#pragma unroll
    for (int i = 0; i < 2 * R; ++i) fx[i] = make_float4(0.f, 0.f, 0.f, 0.f);

    for (int a = 0; a < NP; ++a) {
        b2ptx::mbar_wait(&full[a % NU], (a / NU) & 1);
        if (a >= 2 * R - 1) {
            const int q = a - R;
            float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int i = 1; i <= R; ++i) {
                const float4 hi = b2ptx::lds128(ring + ((q + i) % NU) * SLOT + ucol);
                const float4 lo = b2ptx::lds128(ring + ((q - i + 1) % NU) * SLOT + ucol);
                s = vk_f4fma(k.cx[i - 1], vk_f4sub(hi, lo), s);
            }
            const float4 bq = b2ptx::lds128(ring + (q % NU) * SLOT + bcol);
#pragma unroll
            for (int i = 0; i < 2 * R - 1; ++i) fx[i] = fx[i + 1];
            fx[2 * R - 1] = vk_f4mul(bq, s);
        }
        if (a >= 4 * R - 2) {
            const int p = a - 2 * R + 1;
            const float *U = ring + (p % NU) * SLOT;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int i = 1; i <= R; ++i) acc = vk_f4fma(k.cx[i - 1], vk_f4sub(fx[R + i - 1], fx[R - i]), acc);
            {
                float4 uc[4 * R - 1];
#pragma unroll
                for (int m = 0; m < 4 * R - 1; ++m) uc[m] = b2ptx::lds128(U + ucol + (m - (2 * R - 1)) * BZU);
#pragma unroll
                for (int j = -R; j < R; ++j) {
                    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    for (int i = 1; i <= R; ++i)
                        s = vk_f4fma(k.cy[i - 1], vk_f4sub(uc[j + i + 2 * R - 1], uc[j - i + 1 + 2 * R - 1]), s);
                    const float4 fy = vk_f4mul(b2ptx::lds128(U + bcol + j * BZB), s);
                    acc = vk_f4fma(j >= 0 ? k.cy[j] : -k.cy[-j - 1], fy, acc);
                }
            }
            {
                float zr[4 + 2 * RZU], br[4 + 2 * RZB], fz[2 * R + 3];
                const float *zrow = U + (ty + HU) * BZU + 4 * tz4;
                const float *brow = U + UPL + (ty + R) * BZB + 4 * tz4;
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
            if (zcnt > 0) {
                // the epilogue of b2_visco_point.cuh (visco_update) on four points
                const long long off = (long long)(k.ox + xb + p) * k.sx + rowoff;
                const float4 kd = vk_ldg4(k.K[VK_D] + off), w = vk_ldg4(k.K[VK_W] + off);
                const float4 wm = vk_ldg4(k.K[VK_WM] + off);
                const float4 p0 = ADJ ? vk_ldg4(k.p0 + off) : b2ptx::lds128(U + ucol);
                const float4 pm = vk_ldg4(k.pm + off);
                float4 src = acc, rn = acc;
                if (!ADJ) {
                    const float4 bc = b2ptx::lds128(U + bcol);
                    const float4 kg = vk_ldg4(k.K[VK_G] + off), kt = vk_ldg4(k.K[VK_T] + off);
                    const float4 r0 = vk_ldg4(k.r0 + off);
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        const float lb = VK_AT(acc, c) / VK_AT(bc, c);
                        const float r = (VK_AT(kd, c) - VK_AT(kg, c)) * VK_AT(r0, c) + VK_AT(kg, c) * VK_AT(kt, c) * lb;
                        const float sv = (1.f + VK_AT(kt, c)) * lb - r;
                        if (c == 0) { rn.x = r; src.x = sv; }
                        else if (c == 1) { rn.y = r; src.y = sv; }
                        else if (c == 2) { rn.z = r; src.z = sv; }
                        else { rn.w = r; src.w = sv; }
                    }
                }
                float4 o;
                o.x = w.x * src.x + wm.x * (2.f * p0.x - pm.x) + (kd.x - wm.x) * p0.x;
                o.y = w.y * src.y + wm.y * (2.f * p0.y - pm.y) + (kd.y - wm.y) * p0.y;
                o.z = w.z * src.z + wm.z * (2.f * p0.z - pm.z) + (kd.z - wm.z) * p0.z;
                o.w = w.w * src.w + wm.w * (2.f * p0.w - pm.w) + (kd.w - wm.w) * p0.w;
                float *dp = k.p1 + off;
                float *dr = ADJ ? nullptr : k.r1 + off;
                if (zcnt == 4) {
                    *reinterpret_cast<float4 *>(dp) = o;
                    if (!ADJ) *reinterpret_cast<float4 *>(dr) = rn;
                } else {
                    dp[0] = o.x;
                    if (zcnt > 1) dp[1] = o.y;
                    if (zcnt > 2) dp[2] = o.z;
                    if (!ADJ) {
                        dr[0] = rn.x;
                        if (zcnt > 1) dr[1] = rn.y;
                        if (zcnt > 2) dr[2] = rn.z;
                    }
                }
            }
        }
        // plane a - 2R + 1 is read no more: hand its slot back to the producer
        if (a >= 2 * R - 1) {
            __syncwarp();
            if (lane == 0) b2ptx::mbar_arrive(&empty[(a - 2 * R + 1) % NU]);
        }
    }
}

typedef CUresult (*PFN_encodeTiledVisco)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                         const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                         CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                         CUtensorMapFloatOOBfill);

// tensor map over a ([t,] x, y, z) f32 array, dims innermost first; box = (bz, by, 1[, 1])
static int visco_tmap(CUtensorMap *tm, const void *base, int rank, const int *dims_zyxt, int bz, int by) {
    static PFN_encodeTiledVisco enc = nullptr;
    if (!enc) {
        void *fp = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess) {
            set_error("cuTensorMapEncodeTiled entry point not available");
            return B2_ERR_DEVICE;
        }
        enc = reinterpret_cast<PFN_encodeTiledVisco>(fp);
    }
    cuuint64_t gdim[4], gstr[3];
    cuuint32_t box[4] = {(cuuint32_t)bz, (cuuint32_t)by, 1, 1}, estr[4] = {1, 1, 1, 1};
    cuuint64_t stride = 4;
    for (int i = 0; i < rank; ++i) {
        gdim[i] = (cuuint64_t)dims_zyxt[i];
        stride *= gdim[i];
        if (i < rank - 1) gstr[i] = stride;
    }
    CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void *>(base), gdim, gstr, box,
                     estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("b2_visco_forward: cuTensorMapEncodeTiled failed (%d) rank=%d box=(%d,%d)", (int)r, rank, bz, by);
        return B2_ERR_DEVICE;
    }
    return B2_OK;
}

template <int R>
static int visco_plan_tma(ViscoPlan &p) {
    using Cf = ViscoTmaCfg<R>;
    // forward: the ring streams p[t] (every slot of p, the slot a coordinate); adjoint: the single slot s
    const int dims4[4] = {p.a[2], p.a[1], p.a[0], p.adjoint ? 1 : p.tsize};
    const int dims3[3] = {p.a[2], p.a[1], p.a[0]};
    int rc;
    if ((rc = visco_tmap(&p.tm_f, p.adjoint ? p.s : p.p, 4, dims4, Cf::BZU, Cf::BYU))) return rc;
    return visco_tmap(&p.tm_b, p.b, 3, dims3, Cf::BZB, Cf::BYB);
}

template <int R, bool ADJ>
static int launch_visco_tma(const ViscoPlan &p, int t0, int t2, int t1) {
    using Cf = ViscoTmaCfg<R>;
    auto kern = k_visco_tma<R, ADJ>;
    static bool attr_set = false;           // the shared-memory size is opted into before the first launch
    if (!attr_set) {
        B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cf::SMEM), B2_ERR_LAUNCH);
        attr_set = true;
    }
    auto at = [&](float *x, int t) { return x + (size_t)t * p.slot_elems; };
    ViscoTK<R> k;
    k.p0 = at(p.p, t0);
    k.pm = at(p.p, t2);
    k.p1 = at(p.p, t1);
    k.r0 = ADJ ? nullptr : at(p.r, t0);
    k.r1 = ADJ ? nullptr : at(p.r, t1);
    for (int i = 0; i < VK_NTAB; ++i) k.K[i] = p.K[i];
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
    k.slot0 = ADJ ? 0 : t0;
    for (int i = 0; i < R; ++i) {
        k.cx[i] = p.c[0][i];
        k.cy[i] = p.c[1][i];
        k.cz[i] = p.c[2][i];
    }
    const int ntx = (p.n[0] + k.lx - 1) / k.lx;
    timing_begin();
    note_sweep_kernel("visco_tma<%d>%s", R, ADJ ? "+adj" : "");
    kern<<<k.ntz * k.nty * ntx, Cf::TY * Cf::TZ4 + 32, Cf::SMEM, stream()>>>(p.tm_f, p.tm_b, k);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

// the tables of b2_visco_point.cuh over the slot (and bx = b when b is a scalar), evaluated in double
__global__ void __launch_bounds__(256) k_visco_coef(ViscoCoefK k) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < k.n; i += (size_t)gridDim.x * blockDim.x)
        visco_coef_point(k, i);
}

// scratch cached across calls (re-allocated when the size changes): the tables, b, s
static float *g_visco_scratch[VK_NTAB + 2] = {};
static size_t g_visco_scratch_elems[VK_NTAB + 2] = {};
static int visco_scratch(int which, size_t elems, float **out) {
    if (g_visco_scratch_elems[which] != elems) {
        if (g_visco_scratch[which]) cudaFree(g_visco_scratch[which]);
        g_visco_scratch[which] = nullptr;
        g_visco_scratch_elems[which] = 0;
        B2_CUDA(cudaMalloc(&g_visco_scratch[which], elems * sizeof(float)), B2_ERR_MEMORY);
        g_visco_scratch_elems[which] = elems;
    }
    *out = g_visco_scratch[which];
    return B2_OK;
}

int visco_plan_init(ViscoPlan &p, int kernel) {
    if (kernel != 0 && kernel != 1 && kernel != 2) {
        set_error("b2_visco_forward: unknown kernel %d", kernel);
        return B2_ERR_INVALID;
    }
    // the TMA sweep: 3-D, R in {2, 4} on every axis, z rows and the box start 16-byte aligned (the conditions of
    // k_sa_tma)
    const int R = p.radius[2];
    bool ok = p.radius[0] == R && p.radius[1] == R && (R == 2 || R == 4);
    ok = ok && p.a[2] % 4 == 0 && p.o[2] % 4 == 0 && p.slot_elems % 4 == 0;
    ok = ok && (uintptr_t)p.p % 16 == 0 && (uintptr_t)p.r % 16 == 0 && (uintptr_t)p.b_arr % 16 == 0;
    if (kernel == 2 && !ok) {
        set_error("b2_visco_forward: TMA kernel forced but the layout does not qualify (3-D, radius 2 or 4, z extent "
                  "and z start multiples of 4, 16-byte aligned arrays; radius=%d a2=%d o2=%d)", R, p.a[2], p.o[2]);
        return B2_ERR_INVALID;
    }
    int rc;
    for (int i = 0; i < VK_NTAB; ++i)
        if ((rc = visco_scratch(i, p.slot_elems, &p.K[i]))) return rc;
    if (p.b_arr) {
        p.b = const_cast<float *>(p.b_arr);
    } else if ((rc = visco_scratch(VK_NTAB, p.slot_elems, &p.b))) {
        return rc;
    }
    if (p.adjoint && (rc = visco_scratch(VK_NTAB + 1, p.slot_elems, &p.s))) return rc;
    const size_t n = p.slot_elems;
    const int blocks = (int)std::min<size_t>((n + 255) / 256, 65535);
    ViscoCoefK ck;
    for (int i = 0; i < VK_NTAB; ++i) ck.K[i] = p.K[i];
    ck.bx = p.b_arr ? nullptr : p.b;
    ck.vp = p.vp_arr; ck.qp = p.qp_arr; ck.damp = p.damp;
    ck.vp_value = p.vp_value; ck.qp_value = p.qp_value; ck.b_value = p.b_value;
    ck.f0 = p.f0; ck.dt = p.dt;
    ck.n = n;
    k_visco_coef<<<blocks, 256, 0, stream()>>>(ck);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    p.use_tma = ok && kernel != 1;
    if (!p.use_tma) return B2_OK;
    return R == 2 ? visco_plan_tma<2>(p) : visco_plan_tma<4>(p);
}

static int visco_mix(const ViscoPlan &p, int t0, int t2, int t1) {
    ViscoMixK k;
    for (int i = 0; i < VK_NTAB; ++i) k.K[i] = p.K[i];
    k.b = p.b;
    k.p0 = p.p + (size_t)t0 * p.slot_elems;
    k.r0 = p.r + (size_t)t0 * p.slot_elems;
    k.rw = p.r + (size_t)t1 * p.slot_elems;
    k.s = p.s;
    k.sx = p.sx;
    k.sy = p.sy;
    k.o0 = p.o[0]; k.o1 = p.o[1]; k.o2 = p.o[2];
    k.n0 = p.n[0]; k.n1 = p.n[1]; k.n2 = p.n[2];
    k.n = p.slot_elems;
    const int blocks = (int)std::min<size_t>((k.n + 255) / 256, 65535);
    timing_begin();
    k_visco_adj_mix<<<blocks, 256, 0, stream()>>>(k);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

int visco_step(const ViscoPlan &p, int t0, int t2, int t1) {
    int rc;
    if (p.adjoint && (rc = visco_mix(p, t0, t2, t1))) return rc;
    if (p.use_tma) {
        if (p.radius[2] == 2)
            return p.adjoint ? launch_visco_tma<2, true>(p, t0, t2, t1) : launch_visco_tma<2, false>(p, t0, t2, t1);
        return p.adjoint ? launch_visco_tma<4, true>(p, t0, t2, t1) : launch_visco_tma<4, false>(p, t0, t2, t1);
    }
    auto at = [&](float *x, int t) { return x + (size_t)t * p.slot_elems; };
    ViscoK k;
    k.p0 = at(p.p, t0);
    k.pm = at(p.p, t2);
    k.p1 = at(p.p, t1);
    k.f = p.adjoint ? p.s : k.p0;
    k.r0 = p.adjoint ? nullptr : at(p.r, t0);
    k.r1 = p.adjoint ? nullptr : at(p.r, t1);
    k.b = p.b;
    for (int i = 0; i < VK_NTAB; ++i) k.K[i] = p.K[i];
    k.sx = p.sx;
    k.sy = p.sy;
    k.n0 = p.n[0]; k.n1 = p.n[1]; k.n2 = p.n[2];
    k.o0 = p.o[0]; k.o1 = p.o[1]; k.o2 = p.o[2];
    for (int d = 0; d < 3; ++d) {
        k.r[d] = p.radius[d];
        for (int i = 0; i < B2_MAX_RADIUS; ++i) k.c[d][i] = p.c[d][i];
    }
    k.adjoint = p.adjoint ? 1 : 0;
    dim3 block(64, 4, 1);
    dim3 grid((k.n2 + 63) / 64, (k.n1 + 3) / 4, (unsigned)std::min(k.n0, 65535));
    timing_begin();
    note_sweep_kernel(p.adjoint ? "visco_generic+adj" : "visco_generic");
    k_visco_generic<<<grid, block, 0, stream()>>>(k);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

}  // namespace b2
