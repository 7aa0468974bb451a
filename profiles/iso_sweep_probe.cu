// Bandwidth probe for the isotropic TMA sweep (k_iso_tma, so=8): what HBM gives the sweep's own stream mix
// when nothing is computed. Built and run by iso_sweep_probe.py; not part of the library.
//
// k_copy has the sweep's producer/consumer structure: a CTA owns a (TY x TZ) yz-tile and marches along x over
// LX output planes; per plane one producer lane issues a (TY+2HY) x (TZ+2HZ) box of u[t] and two TY x TZ tiles
// (u[t-1], A) with TMA on a full mbarrier, and the consumer threads store one TY x TZ tile of u[t+1] with
// 16-byte stores, then release the stage. The stage ring has LEAD+1 stages, so the producer runs LEAD planes
// ahead of the consumers, as the sweep's does. The consumers do no arithmetic: the stored value is the u[t-1]
// tile, so the time is that of the memory system alone. NT = 1 drops the A tile: the three-stream mix the sweep
// moves on the planes whose A it takes from its pinned tile (b2_iso.cu::k_iso_tma).
//
// k_stream is a plain float4 read/write stream (grid-stride, one read and one write per element).
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <vector>
#include "b2_ptx.cuh"

#define CK(x)                                                                                    \
    do {                                                                                         \
        cudaError_t e_ = (x);                                                                    \
        if (e_ != cudaSuccess) {                                                                 \
            fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_));         \
            exit(1);                                                                             \
        }                                                                                        \
    } while (0)

constexpr int N = 1024;           // interior points per dimension
constexpr int H = 8;              // allocated halo (>= the largest box halo)
constexpr int A = N + 2 * H;      // allocated extent per dimension
constexpr int R = 4;              // so = 8
constexpr int LX = 64;            // output planes per CTA

struct Grid {
    int ntz, nty, ntx;
};

template <int TY, int TZ, int HY, int HZ, int LEAD, int NT>
struct CopyCfg {
    static constexpr int BY = TY + 2 * HY, BZ = TZ + 2 * HZ;
    static constexpr int UBOX = (BY * BZ + 31) / 32 * 32;
    static constexpr int TILE = TY * TZ;
    static constexpr int NST = LEAD + 1;
    static constexpr int NCT = TILE / 4 < 512 ? TILE / 4 : 512;      // consumer threads
    static constexpr int NCW = NCT / 32;
    static constexpr size_t SMEM = (size_t)NST * (UBOX + NT * TILE) * 4 + 2 * NST * 8 + 128;
};

template <int TY, int TZ, int HY, int HZ, int LEAD, int NT>
__global__ void __launch_bounds__(CopyCfg<TY, TZ, HY, HZ, LEAD, NT>::NCT + 32, 1)
k_copy(const __grid_constant__ CUtensorMap tm_u, const __grid_constant__ CUtensorMap tm_um,
       const __grid_constant__ CUtensorMap tm_a, float *__restrict__ out, Grid g) {
    using C = CopyCfg<TY, TZ, HY, HZ, LEAD, NT>;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *s_u = reinterpret_cast<float *>(smem_raw);
    float *s_t = s_u + C::NST * C::UBOX;                        // per stage: u[t-1] tile[, A tile]
    uint64_t *full = reinterpret_cast<uint64_t *>(s_t + C::NST * NT * C::TILE);
    uint64_t *empty = full + C::NST;

    int b = blockIdx.x;
    const int iz = b % g.ntz;
    b /= g.ntz;
    const int iy = b % g.nty;
    const int ix = b / g.nty;
    const int z0 = H + iz * TZ, y0 = H + iy * TY, xs = H + ix * LX;
    const int NP = LX + 2 * R;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    if (tid == 0) {
        for (int i = 0; i < C::NST; ++i) {
            b2ptx::mbar_init(&full[i], 1);
            b2ptx::mbar_init(&empty[i], C::NCW);
        }
        b2ptx::fence_mbar_init();
    }
    __syncthreads();

    if (warp == C::NCW) {
        if (lane == 0) {
            for (int j = 0; j < NP; ++j) {
                const int st = j % C::NST;
                if (j >= C::NST) b2ptx::mbar_wait(&empty[st], ((j / C::NST) - 1) & 1);
                const bool tiles = j >= 2 * R;
                b2ptx::mbar_arrive_expect_tx(&full[st], (C::BY * C::BZ + (tiles ? NT * C::TILE : 0)) * 4);
                b2ptx::tma_load_3d(s_u + st * C::UBOX, &tm_u, &full[st], z0 - HZ, y0 - HY, xs - R + j);
                if (tiles) {
                    float *t = s_t + st * NT * C::TILE;
                    b2ptx::tma_load_3d(t, &tm_um, &full[st], z0, y0, xs + j - 2 * R);
                    if (NT == 2) b2ptx::tma_load_3d(t + C::TILE, &tm_a, &full[st], z0, y0, xs + j - 2 * R);
                }
            }
        }
        return;
    }

    for (int j = 0; j < NP; ++j) {
        const int st = j % C::NST;
        b2ptx::mbar_wait(&full[st], (j / C::NST) & 1);
        if (j >= 2 * R) {
            const float *t = s_t + st * NT * C::TILE;
            float *op = out + (size_t)(xs + j - 2 * R) * A * A;
#pragma unroll
            for (int f = tid; f < C::TILE / 4; f += C::NCT) {
                const int yy = f / (TZ / 4), zz = 4 * (f % (TZ / 4));
                *reinterpret_cast<float4 *>(op + (size_t)(y0 + yy) * A + z0 + zz) = b2ptx::lds128(t + 4 * f);
            }
        }
        __syncwarp();
        if (lane == 0) b2ptx::mbar_arrive(&empty[st]);
    }
}

// The two-level pass's (k_iso_tma2) stream mix: per CTA LX2 output planes of a 16 x 64 tile (the pass's own x-chunks:
// 4R priming planes per chunk weigh 4x as much as the one-step sweep's R); per plane one 32 x 80 box of
// u[t] (LX + 4R planes), a 24 x 72 tile of u[t-1] on the level-1 planes (LX + 2R) and, with NT == 2, one of A; the
// consumers store a 16 x 64 tile of u[t+1] on the owned level-1 planes and one of u[t+2], R planes behind.
template <int NT>
struct Copy2Cfg {
    static constexpr int TY = 16, TZ = 64, BY = TY + 4 * R, BZ = TZ + 16, EY = TY + 2 * R, EZ = TZ + 8;
    static constexpr int UBOX = (BY * BZ + 31) / 32 * 32, ETILE = EY * EZ;
    static constexpr int NST = R + 1;                                 // the pass's lead of R planes
    static constexpr int NCT = 448;
    static constexpr int LX2 = 205;                                   // choose_chunk_len at 1024^3: 5 chunks
    static constexpr size_t SMEM = (size_t)NST * (UBOX + NT * ETILE) * 4 + 2 * NST * 8 + 128;
};

template <int NT>
__global__ void __launch_bounds__(Copy2Cfg<NT>::NCT + 32, 1)
k_copy2(const __grid_constant__ CUtensorMap tm_u, const __grid_constant__ CUtensorMap tm_um,
        const __grid_constant__ CUtensorMap tm_a, float *__restrict__ out1, float *__restrict__ out2, Grid g) {
    using C = Copy2Cfg<NT>;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *s_u = reinterpret_cast<float *>(smem_raw);
    float *s_t = s_u + C::NST * C::UBOX;
    uint64_t *full = reinterpret_cast<uint64_t *>(s_t + C::NST * NT * C::ETILE);
    uint64_t *empty = full + C::NST;
    constexpr int NCW = C::NCT / 32;

    int b = blockIdx.x;
    const int iz = b % g.ntz;
    b /= g.ntz;
    const int iy = b % g.nty;
    const int ix = b / g.nty;
    const int z0 = H + iz * C::TZ, y0 = H + iy * C::TY, xs = H + ix * C::LX2, xe = min(xs + C::LX2, H + N);
    const int NP = (xe - xs) + 4 * R;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        for (int i = 0; i < C::NST; ++i) {
            b2ptx::mbar_init(&full[i], 1);
            b2ptx::mbar_init(&empty[i], NCW);
        }
        b2ptx::fence_mbar_init();
    }
    __syncthreads();
    if (warp == NCW) {
        if (lane == 0) {
            for (int j = 0; j < NP; ++j) {
                const int st = j % C::NST;
                if (j >= C::NST) b2ptx::mbar_wait(&empty[st], ((j / C::NST) - 1) & 1);
                const bool tiles = j >= 2 * R && j < NP - R;               // level-1 planes xs - R .. xs + LX + R
                b2ptx::mbar_arrive_expect_tx(&full[st], (C::BY * C::BZ + (tiles ? NT * C::ETILE : 0)) * 4);
                b2ptx::tma_load_3d(s_u + st * C::UBOX, &tm_u, &full[st], z0 - 8, y0 - 2 * R, xs - 2 * R + j);
                if (tiles) {
                    float *t = s_t + st * NT * C::ETILE;
                    const int x1 = xs - 3 * R + j;
                    b2ptx::tma_load_3d(t, &tm_um, &full[st], z0 - 4, y0 - R, x1);
                    if (NT == 2) b2ptx::tma_load_3d(t + C::ETILE, &tm_a, &full[st], z0 - 4, y0 - R, x1);
                }
            }
        }
        return;
    }
    const int yy = tid / 16, zz = 4 * (tid % 16);                     // threads 0..255: one float4 of the tile
    for (int j = 0; j < NP; ++j) {
        const int st = j % C::NST;
        b2ptx::mbar_wait(&full[st], (j / C::NST) & 1);
        const float4 v = b2ptx::lds128(s_u + st * C::UBOX + (yy + 2 * R) * C::BZ + 8 + zz);
        const int x1 = xs - 3 * R + j, x2 = x1 - R;
        if (tid < 256 && x1 >= xs && x1 < xe)
            *reinterpret_cast<float4 *>(out1 + (size_t)x1 * A * A + (size_t)(y0 + yy) * A + z0 + zz) = v;
        if (tid < 256 && x2 >= xs && x2 < xe)
            *reinterpret_cast<float4 *>(out2 + (size_t)x2 * A * A + (size_t)(y0 + yy) * A + z0 + zz) = v;
        __syncwarp();
        if (lane == 0) b2ptx::mbar_arrive(&empty[st]);
    }
}

__global__ void k_stream(const float4 *__restrict__ src, float4 *__restrict__ dst, size_t n4) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = src[i];
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static CUtensorMap tmap(const float *base, int bz, int by) {
    static PFN_encodeTiled enc = nullptr;
    if (!enc) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
        enc = reinterpret_cast<PFN_encodeTiled>(p);
    }
    CUtensorMap tm;
    cuuint64_t gdim[3] = {A, A, A}, gstr[2] = {(cuuint64_t)A * 4, (cuuint64_t)A * A * 4};
    cuuint32_t box[3] = {(cuuint32_t)bz, (cuuint32_t)by, 1}, estr[3] = {1, 1, 1};
    if (enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float *>(base), gdim, gstr, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
        fprintf(stderr, "cuTensorMapEncodeTiled failed box=(%d,%d)\n", bz, by);
        exit(1);
    }
    return tm;
}

static float *g_u, *g_um, *g_a, *g_out;
static const int kReps = 5;

template <int TY, int TZ, int HY, int HZ, int LEAD, int NT = 2>
static void run_copy(const char *name, bool first) {
    using C = CopyCfg<TY, TZ, HY, HZ, LEAD, NT>;
    auto kern = k_copy<TY, TZ, HY, HZ, LEAD, NT>;
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
    CUtensorMap tu = tmap(g_u, C::BZ, C::BY), tum = tmap(g_um, TZ, TY), ta = tmap(g_a, TZ, TY);
    Grid g{N / TZ, N / TY, N / LX};
    const unsigned grid = g.ntz * g.nty * g.ntx;
    kern<<<grid, C::NCT + 32, C::SMEM>>>(tu, tum, ta, g_out, g);       // warm-up
    CK(cudaGetLastError());
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0));
    for (int r = 0; r < kReps; ++r) kern<<<grid, C::NCT + 32, C::SMEM>>>(tu, tum, ta, g_out, g);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    ms /= kReps;
    const double pts = (double)(g.ntz * TZ) * (g.nty * TY) * (g.ntx * LX);
    const double alg = 16.0 * pts;
    const double moved = (double)grid * ((double)(LX + 2 * R) * C::BY * C::BZ * 4 + (double)LX * C::TILE * 4 * (NT + 1));
    printf("%s{\"name\": \"%s\", \"u_box\": [%d, %d], \"tile\": [%d, %d], \"tiles_in\": %d, \"lead\": %d, \"smem\": %zu, "
           "\"ms\": %.4f, \"alg_gbs\": %.1f, \"moved_gbs\": %.1f, \"moved_per_alg\": %.4f}",
           first ? "" : ", ", name, C::BY, C::BZ, TY, TZ, NT, LEAD, C::SMEM, ms, alg / ms * 1e-6, moved / ms * 1e-6,
           moved / alg);
    CK(cudaEventDestroy(e0));
    CK(cudaEventDestroy(e1));
}

static float *g_out2;

template <int NT>
static void run_copy2(const char *name) {
    using C = Copy2Cfg<NT>;
    auto kern = k_copy2<NT>;
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
    CUtensorMap tu = tmap(g_u, C::BZ, C::BY), tum = tmap(g_um, C::EZ, C::EY), ta = tmap(g_a, C::EZ, C::EY);
    Grid g{N / C::TZ, N / C::TY, (N + C::LX2 - 1) / C::LX2};
    const unsigned grid = g.ntz * g.nty * g.ntx;
    kern<<<grid, C::NCT + 32, C::SMEM>>>(tu, tum, ta, g_out, g_out2, g);
    CK(cudaGetLastError());
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0));
    for (int r = 0; r < kReps; ++r) kern<<<grid, C::NCT + 32, C::SMEM>>>(tu, tum, ta, g_out, g_out2, g);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    ms /= kReps;
    const double tiles = (double)g.ntz * g.nty;
    const double moved = tiles * ((double)(N + 4 * R * g.ntx) * C::BY * C::BZ * 4 +
                                  (double)(N + 2 * R * g.ntx) * C::ETILE * 4 * NT + 2.0 * N * C::TY * C::TZ * 4);
    printf(", {\"name\": \"%s\", \"u_box\": [%d, %d], \"tile\": [%d, %d], \"tiles_in\": %d, \"lead\": %d, "
           "\"smem\": %zu, \"chunk\": %d, \"ms\": %.4f, \"ms_per_step\": %.4f, \"moved_gbs\": %.1f}",
           name, C::BY, C::BZ, C::EY, C::EZ, NT, C::NST - 1, C::SMEM, C::LX2, ms, ms / 2, moved / ms * 1e-6);
    CK(cudaEventDestroy(e0));
    CK(cudaEventDestroy(e1));
}

int main() {
    const size_t elems = (size_t)A * A * A;
    CK(cudaMalloc(&g_u, elems * 4));
    CK(cudaMalloc(&g_um, elems * 4));
    CK(cudaMalloc(&g_a, elems * 4));
    CK(cudaMalloc(&g_out, elems * 4));
    CK(cudaMalloc(&g_out2, elems * 4));
    CK(cudaMemset(g_u, 0, elems * 4));
    CK(cudaMemset(g_um, 0, elems * 4));
    CK(cudaMemset(g_a, 0, elems * 4));
    int sms = 0;
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));

    printf("{\"copy\": [");
    // the so=8 sweep's boxes (32 x 64 tile) at leads 1 .. 7; a 28 x 64 tile (15 instead of 17 warps) up to lead 8
    run_copy<32, 64, 4, 4, 1>("sweep_32x64", true);
    run_copy<32, 64, 4, 4, 2>("sweep_32x64", false);
    run_copy<32, 64, 4, 4, 3>("sweep_32x64", false);
    run_copy<32, 64, 4, 4, 4>("sweep_32x64", false);
    run_copy<32, 64, 4, 4, 6>("sweep_32x64", false);
    run_copy<32, 64, 4, 4, 7>("sweep_32x64", false);
    run_copy<28, 64, 4, 4, 4>("sweep_28x64", false);
    run_copy<28, 64, 4, 4, 6>("sweep_28x64", false);
    run_copy<28, 64, 4, 4, 8>("sweep_28x64", false);
    // u[t] without its halo (no re-read) and 512-byte rows instead of 256-byte ones
    run_copy<32, 64, 0, 0, 4>("nohalo_32x64", false);
    run_copy<32, 64, 0, 0, 7>("nohalo_32x64", false);
    run_copy<16, 128, 0, 0, 4>("nohalo_16x128", false);
    run_copy<16, 128, 0, 0, 7>("nohalo_16x128", false);
    // the sweep's 16 x 128 boxes with the A tile (16 B/point) and without it (the planes whose A is pinned, 12 B/point)
    run_copy<16, 128, 4, 4, 4>("sweep_16x128", false);
    run_copy<16, 128, 4, 4, 4, 1>("sweep_16x128_noA", false);
    // the two-level pass's boxes (k_iso_tma2): A pinned (tiles_in 1, most planes of the headline) and streamed (2)
    run_copy2<1>("two_level_16x64_noA");
    run_copy2<2>("two_level_16x64");
    printf("]");

    // plain read/write stream over 2 x 4.4 GB
    const size_t n4 = elems / 4;
    k_stream<<<sms * 8, 512>>>(reinterpret_cast<const float4 *>(g_u), reinterpret_cast<float4 *>(g_out), n4);
    CK(cudaGetLastError());
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0));
    for (int r = 0; r < kReps; ++r)
        k_stream<<<sms * 8, 512>>>(reinterpret_cast<const float4 *>(g_u), reinterpret_cast<float4 *>(g_out), n4);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    ms /= kReps;
    printf(", \"stream\": {\"bytes\": %zu, \"ms\": %.4f, \"gbs\": %.1f}, \"sms\": %d}\n", elems * 8, ms,
           elems * 8.0 / ms * 1e-6, sms);
    cudaFree(g_u);
    cudaFree(g_um);
    cudaFree(g_a);
    cudaFree(g_out);
    cudaFree(g_out2);
    return 0;
}
