// Self-adjoint variable-density visco-acoustic update (the reference's `iso_stencil`,
// examples/seismic/self_adjoint/operators.py:4-65): nested half-node first derivatives with the buoyancy b between
// them, u_new = dt^2 vp^2/b * sum_d (b u.d(x0=d+h/2)).d(x0=d-h/2) + (2 - dt w) u + (dt w - 1) u_old.
//
//   k_sa_coef    : once per call, C = dt^2 vp^2 / b over the whole allocated slot into library scratch (a scalar vp or
//                  b is tabulated the same way; a scalar b is also expanded into a scratch array), so that the sweep
//                  has one form. The source terms scale by the same table.
//   k_sa_generic : one thread per point, any even space order <= 16, 2-D and 3-D, any alignment. Its point body is
//                  b2_sa_point.cuh (emulated on the CPU by tests/support/emu_sa.cu). Per point and step it reads
//                  u[t], u[t-dir], C and w at the point and b, u[t] on the (2R-1)-wide star, and writes one level:
//                  24 B/point algorithmic (DESIGN §3.3h).
//   k_sa_tma<R>  : 2.5-D sweep along x for 3-D grids, R in {2, 4}. A CTA owns a (TY x TZ) yz-tile and marches
//                  along x; a producer warp streams, per plane, the u[t] plane with a (2R-1)-wide y/z halo and the b
//                  plane with an R-wide halo into a shared-memory ring with TMA, signalled on mbarriers. Each consumer
//                  thread owns four consecutive z points: it keeps F_x of the 2R planes the outer x-difference needs in
//                  a register queue (one F_x per plane, from the ring's centre columns), forms F_y and F_z of its own
//                  points from the ring in registers (no CTA barrier: every thread reads only the ring), reads C, w and
//                  u[t-dir] once with 16-byte loads and writes u[t+dir] with 16-byte stores.
#include "b2_sa.cuh"
#include "b2_sa_point.cuh"
#include "b2_ptx.cuh"
#include <algorithm>

namespace b2 {

__global__ void __launch_bounds__(256) k_sa_generic(SaK k) {
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (z >= k.n2 || y >= k.n1) return;
    for (int x = blockIdx.z; x < k.n0; x += gridDim.z) sa_point(k, x, y, z);
}

// ------------------------------------------------------------------------------------------
// 2.5-D TMA sweep
// ------------------------------------------------------------------------------------------
template <int R> struct SaTmaCfg {
    static constexpr int TY = 16, TZ4 = 16, TZ = 4 * TZ4;
    static constexpr int HU = 2 * R - 1;                  // reach of the nested stencil: the u halo in y
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

template <int R> struct SaTK {
    const float *um;                 // u[t - dir] slot
    float *u1;                       // u[t + dir] slot
    const float *C, *w;              // w may be null
    long long sx, sy;
    int ny, nz, ox, oy, oz;
    int xlo, xcount, lx, ntz, nty;
    int slot0;                       // u[t] slot: the 4th tensor-map coordinate
    float cx[R], cy[R], cz[R];
    float dt;
};

__device__ __forceinline__ float4 sa_f4fma(float w, float4 v, float4 acc) {
    return make_float4(fmaf(w, v.x, acc.x), fmaf(w, v.y, acc.y), fmaf(w, v.z, acc.z), fmaf(w, v.w, acc.w));
}
__device__ __forceinline__ float4 sa_f4sub(float4 a, float4 b) {
    return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w);
}
__device__ __forceinline__ float4 sa_f4mul(float4 a, float4 b) {
    return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w);
}
__device__ __forceinline__ float4 sa_ldg4(const float *p) {
    return __ldg(reinterpret_cast<const float4 *>(p));
}

template <int R>
__global__ void __launch_bounds__(SaTmaCfg<R>::TY * SaTmaCfg<R>::TZ4 + 32, 1)
k_sa_tma(const __grid_constant__ CUtensorMap tm_u, const __grid_constant__ CUtensorMap tm_b, const SaTK<R> k) {
    using Cf = SaTmaCfg<R>;
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
            b2ptx::tma_prefetch_desc(&tm_u);
            b2ptx::tma_prefetch_desc(&tm_b);
            for (int j = 0; j < NP; ++j) {
                const int slot = j % NU, round = j / NU;
                if (round > 0) b2ptx::mbar_wait(&empty[slot], (round - 1) & 1);
                b2ptx::mbar_arrive_expect_tx(&full[slot], (uint32_t)(Cf::BYU * BZU + Cf::BYB * BZB) * 4);
                float *dst = ring + slot * SLOT;
                b2ptx::tma_load_4d(dst, &tm_u, &full[slot], k.oz + z0 - RZU, k.oy + y0 - HU, k.ox + xb + j, k.slot0);
                b2ptx::tma_load_3d(dst + UPL, &tm_b, &full[slot], k.oz + z0 - RZB, k.oy + y0 - R, k.ox + xb + j);
            }
        }
        return;
    }

    // ---------------- consumers ----------------
    const int ty = tid / TZ4, tz4 = tid % TZ4;
    const int gy = y0 + ty, gz = z0 + 4 * tz4;
    const int zcnt = gy < k.ny ? min(max(k.nz - gz, 0), 4) : 0;
    const int ucol = (ty + HU) * BZU + RZU + 4 * tz4;          // my four points in a u plane
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
                s = sa_f4fma(k.cx[i - 1], sa_f4sub(hi, lo), s);
            }
            const float4 bq = b2ptx::lds128(ring + (q % NU) * SLOT + bcol);
#pragma unroll
            for (int i = 0; i < 2 * R - 1; ++i) fx[i] = fx[i + 1];
            fx[2 * R - 1] = sa_f4mul(bq, s);
        }
        if (a >= 4 * R - 2) {
            const int p = a - 2 * R + 1;
            const float *U = ring + (p % NU) * SLOT;
            // x: sum_k c_k (F_x(p + k - 1) - F_x(p - k))
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int i = 1; i <= R; ++i) acc = sa_f4fma(k.cx[i - 1], sa_f4sub(fx[R + i - 1], fx[R - i]), acc);
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
                        s = sa_f4fma(k.cy[i - 1], sa_f4sub(uc[j + i + 2 * R - 1], uc[j - i + 1 + 2 * R - 1]), s);
                    const float4 fy = sa_f4mul(b2ptx::lds128(U + bcol + j * BZB), s);
                    acc = sa_f4fma(j >= 0 ? k.cy[j] : -k.cy[-j - 1], fy, acc);
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
            if (zcnt > 0) {
                const long long off = (long long)(k.ox + xb + p) * k.sx + rowoff;
                const float4 c = b2ptx::lds128(U + ucol);
                const float4 cv = sa_ldg4(k.C + off);
                const float4 pv = sa_ldg4(k.um + off);
                const float4 wv = k.w ? sa_ldg4(k.w + off) : make_float4(0.f, 0.f, 0.f, 0.f);
                float4 o;
                o.x = fmaf(cv.x, acc.x, fmaf(2.f - k.dt * wv.x, c.x, (k.dt * wv.x - 1.f) * pv.x));
                o.y = fmaf(cv.y, acc.y, fmaf(2.f - k.dt * wv.y, c.y, (k.dt * wv.y - 1.f) * pv.y));
                o.z = fmaf(cv.z, acc.z, fmaf(2.f - k.dt * wv.z, c.z, (k.dt * wv.z - 1.f) * pv.z));
                o.w = fmaf(cv.w, acc.w, fmaf(2.f - k.dt * wv.w, c.w, (k.dt * wv.w - 1.f) * pv.w));
                float *dst = k.u1 + off;
                if (zcnt == 4) {
                    *reinterpret_cast<float4 *>(dst) = o;
                } else {
                    dst[0] = o.x;
                    if (zcnt > 1) dst[1] = o.y;
                    if (zcnt > 2) dst[2] = o.z;
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

typedef CUresult (*PFN_encodeTiledSa)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                      const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                      CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                      CUtensorMapFloatOOBfill);

// tensor map over a ([t,] x, y, z) f32 array, dims innermost first; box = (bz, by, 1[, 1])
static int sa_tmap(CUtensorMap *tm, const void *base, int rank, const int *dims_zyxt, int bz, int by) {
    static PFN_encodeTiledSa enc = nullptr;
    if (!enc) {
        void *fp = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess) {
            set_error("cuTensorMapEncodeTiled entry point not available");
            return B2_ERR_DEVICE;
        }
        enc = reinterpret_cast<PFN_encodeTiledSa>(fp);
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
        set_error("b2_sa_forward: cuTensorMapEncodeTiled failed (%d) rank=%d box=(%d,%d)", (int)r, rank, bz, by);
        return B2_ERR_DEVICE;
    }
    return B2_OK;
}

template <int R>
static int sa_plan_tma(SaPlan &p) {
    using Cf = SaTmaCfg<R>;
    const int dims4[4] = {p.a[2], p.a[1], p.a[0], p.tsize};
    const int dims3[3] = {p.a[2], p.a[1], p.a[0]};
    int rc;
    if ((rc = sa_tmap(&p.tm_u, p.u, 4, dims4, Cf::BZU, Cf::BYU))) return rc;
    return sa_tmap(&p.tm_b, p.b, 3, dims3, Cf::BZB, Cf::BYB);
}

template <int R>
static int launch_sa_tma(const SaPlan &p, int slot0, int slotm, int slot1) {
    using Cf = SaTmaCfg<R>;
    auto kern = k_sa_tma<R>;
    static bool attr_set = false;           // the shared-memory size is opted into before the first launch
    if (!attr_set) {
        B2_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cf::SMEM), B2_ERR_LAUNCH);
        attr_set = true;
    }
    SaTK<R> k;
    k.um = p.u + (size_t)slotm * p.slot_elems;
    k.u1 = p.u + (size_t)slot1 * p.slot_elems;
    k.C = p.C;
    k.w = p.w;
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
    k.dt = p.dt;
    const int ntx = (p.n[0] + k.lx - 1) / k.lx;
    timing_begin();
    note_sweep_kernel("sa_tma<%d>%s", R, p.adjoint ? "+adj" : "");
    kern<<<k.ntz * k.nty * ntx, Cf::TY * Cf::TZ4 + 32, Cf::SMEM, stream()>>>(p.tm_u, p.tm_b, k);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

// C = dt^2 vp^2 / b (and bx = b when b is a scalar) over n elements
__global__ void __launch_bounds__(256) k_sa_coef(float *__restrict__ C, float *__restrict__ bx,
                                                 const float *__restrict__ vp, const float *__restrict__ b,
                                                 float vp_value, float b_value, float dt2, size_t n) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float v = vp ? vp[i] : vp_value;
        const float bb = b ? b[i] : b_value;
        C[i] = dt2 * v * v / bb;
        if (bx) bx[i] = b_value;
    }
}

// scratch cached across calls (re-allocated when the size changes)
static float *g_sa_scratch[2] = {};
static size_t g_sa_scratch_elems[2] = {};
static int sa_scratch(int which, size_t elems, float **out) {
    if (g_sa_scratch_elems[which] != elems) {
        if (g_sa_scratch[which]) cudaFree(g_sa_scratch[which]);
        g_sa_scratch[which] = nullptr;
        g_sa_scratch_elems[which] = 0;
        B2_CUDA(cudaMalloc(&g_sa_scratch[which], elems * sizeof(float)), B2_ERR_MEMORY);
        g_sa_scratch_elems[which] = elems;
    }
    *out = g_sa_scratch[which];
    return B2_OK;
}

int sa_plan_init(SaPlan &p, int kernel) {
    if (kernel != 0 && kernel != 1 && kernel != 2) {
        set_error("b2_sa_forward: unknown kernel %d", kernel);
        return B2_ERR_INVALID;
    }
    int rc;
    if ((rc = sa_scratch(0, p.slot_elems, &p.C))) return rc;
    if (p.b_arr) {
        p.b = const_cast<float *>(p.b_arr);
    } else if ((rc = sa_scratch(1, p.slot_elems, &p.b))) {
        return rc;
    }
    const size_t n = p.slot_elems;
    const int blocks = (int)std::min<size_t>((n + 255) / 256, 65535);
    k_sa_coef<<<blocks, 256, 0, stream()>>>(p.C, p.b_arr ? nullptr : p.b, p.vp_arr, p.b_arr, p.vp_value, p.b_value,
                                            p.dt * p.dt, n);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    // the TMA sweep: 3-D, R in {2, 4} on every axis, z rows and the box start 16-byte aligned (the conditions of
    // k_iso_tma: so % 4 == 0 and nz % 4 == 0 make the row pitch a multiple of 4 floats)
    const int R = p.radius[2];
    bool ok = p.radius[0] == R && p.radius[1] == R && (R == 2 || R == 4);
    ok = ok && p.a[2] % 4 == 0 && p.o[2] % 4 == 0 && p.slot_elems % 4 == 0;
    ok = ok && (uintptr_t)p.u % 16 == 0 && (uintptr_t)p.b % 16 == 0 && (uintptr_t)p.C % 16 == 0;
    ok = ok && (uintptr_t)p.w % 16 == 0;
    if (kernel == 2 && !ok) {
        set_error("b2_sa_forward: TMA kernel forced but the layout does not qualify (3-D, radius 2 or 4, z extent "
                  "and z start multiples of 4, 16-byte aligned arrays; radius=%d a2=%d o2=%d)", R, p.a[2], p.o[2]);
        return B2_ERR_INVALID;
    }
    p.use_tma = ok && kernel != 1;
    if (!p.use_tma) return B2_OK;
    return R == 2 ? sa_plan_tma<2>(p) : sa_plan_tma<4>(p);
}

int sa_step(const SaPlan &p, int slot0, int slotm, int slot1) {
    if (p.use_tma)
        return p.radius[2] == 2 ? launch_sa_tma<2>(p, slot0, slotm, slot1) : launch_sa_tma<4>(p, slot0, slotm, slot1);
    SaK k;
    k.u0 = p.u + (size_t)slot0 * p.slot_elems;
    k.um = p.u + (size_t)slotm * p.slot_elems;
    k.u1 = p.u + (size_t)slot1 * p.slot_elems;
    k.b = p.b;
    k.C = p.C;
    k.w = p.w;
    k.sx = p.sx;
    k.sy = p.sy;
    k.n0 = p.n[0]; k.n1 = p.n[1]; k.n2 = p.n[2];
    k.o0 = p.o[0]; k.o1 = p.o[1]; k.o2 = p.o[2];
    for (int d = 0; d < 3; ++d) {
        k.r[d] = p.radius[d];
        for (int i = 0; i < B2_MAX_RADIUS; ++i) k.c[d][i] = p.c[d][i];
    }
    k.dt = p.dt;
    dim3 block(64, 4, 1);
    dim3 grid((k.n2 + 63) / 64, (k.n1 + 3) / 4, (unsigned)std::min(k.n0, 65535));
    timing_begin();
    note_sweep_kernel(p.adjoint ? "sa_generic+adj" : "sa_generic");
    k_sa_generic<<<grid, block, 0, stream()>>>(k);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

}  // namespace b2
