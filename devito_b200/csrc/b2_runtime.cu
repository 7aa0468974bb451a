// Runtime plumbing of libb200stencil: stream, error string, staging of `struct dataobj`
// arrays (host <-> device, mirroring the reference's `acc enter data copyin / exit data
// copyout` placed by DeviceAwareDataManager, devito/passes/iet/definitions.py:636-671),
// launch counter, kernel timing, small device-memory utilities.
#include "b2_common.cuh"
#include "b2_iso.cuh"
#include <cstdarg>
#include <cstdlib>
#include <vector>

namespace b2 {

thread_local std::string g_last_error;
cudaStream_t g_stream = nullptr;
cudaStream_t g_user_stream = nullptr;
unsigned long long g_launches = 0;

static bool g_timing_on = false;
static std::vector<cudaEvent_t> g_timing_events;   // pairs (begin, end)
static size_t g_timing_used = 0;

void set_error(const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
}

static char g_sweep_kernel[64] = "";

void note_sweep_kernel(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_sweep_kernel, sizeof(g_sweep_kernel), fmt, ap);
    va_end(ap);
}

static int g_bound_device = -1;

int use_device(int dev) {
    if (g_bound_device >= 0 && dev != g_bound_device) {
        set_error("libb200stencil is bound to device %d in this process (one process per GPU); "
                  "device %d requested", g_bound_device, dev);
        return B2_ERR_INVALID;
    }
    cudaError_t e = cudaSetDevice(dev);
    if (e != cudaSuccess) {
        set_error("cudaSetDevice(%d) -> %s", dev, cudaGetErrorString(e));
        return B2_ERR_DEVICE;
    }
    g_bound_device = dev;
    return B2_OK;
}

int sm_count() {
    static int n = 0;
    if (n > 0) return n;
    int dev = 0, v = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess) e = cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess || v <= 0) {
        set_error("SM count of the current device unavailable: %s", cudaGetErrorString(e));
        return 0;
    }
    n = v;
    return n;
}

std::mutex &api_mutex() {
    static std::mutex m;
    return m;
}

cudaStream_t stream() {
    if (g_user_stream) return g_user_stream;
    if (!g_stream) cudaStreamCreateWithFlags(&g_stream, cudaStreamNonBlocking);
    return g_stream;
}

void timing_begin() {
    if (!g_timing_on) return;
    if (g_timing_used + 2 > g_timing_events.size()) {
        if (g_timing_events.size() >= 16384) return;   // bounded pool
        cudaEvent_t a, b;
        cudaEventCreate(&a);
        cudaEventCreate(&b);
        g_timing_events.push_back(a);
        g_timing_events.push_back(b);
    }
    cudaEventRecord(g_timing_events[g_timing_used], stream());
}

void timing_end() {
    if (!g_timing_on) return;
    if (g_timing_used + 2 > g_timing_events.size()) return;
    cudaEventRecord(g_timing_events[g_timing_used + 1], stream());
    g_timing_used += 2;
}

// Small staging buffers (sparse tables, source/receiver traces) are recycled through a size-keyed
// pool instead of cudaMalloc/cudaFree per call: cudaFree synchronises the whole device and both
// cost ~0.1-1 ms, which showed up as a fixed per-apply overhead in the first benchmark.
// Large staging buffers (the wavefields of a host-staged apply: 13.5 GB at 1024^3) are recycled too — a
// production run applies the same operator shot after shot — up to B2_STAGING_CACHE_GB (default 24, under a
// third of an 80 GB H100) of cached bytes; beyond that, or when an allocation fails, the cache is drained.
static std::vector<std::pair<size_t, void *>> g_pool_free;
static const size_t kPoolSmall = 64u << 20;
static size_t g_pool_big_bytes = 0;

static size_t pool_big_cap() {
    static size_t cap = 0;
    static bool init = false;
    if (!init) {
        const char *e = getenv("B2_STAGING_CACHE_GB");
        cap = (size_t)((e ? atof(e) : 24.0) * (double)(1ull << 30));
        init = true;
    }
    return cap;
}

static void pool_drain_big() {
    for (size_t i = 0; i < g_pool_free.size();) {
        if (g_pool_free[i].first > kPoolSmall) {
            cudaFree(g_pool_free[i].second);
            g_pool_big_bytes -= g_pool_free[i].first;
            g_pool_free.erase(g_pool_free.begin() + i);
        } else {
            ++i;
        }
    }
}

static cudaError_t pool_alloc(void **p, size_t nbytes) {
    for (size_t i = 0; i < g_pool_free.size(); ++i) {
        if (g_pool_free[i].first == nbytes) {
            *p = g_pool_free[i].second;
            if (nbytes > kPoolSmall) g_pool_big_bytes -= nbytes;
            g_pool_free.erase(g_pool_free.begin() + i);
            return cudaSuccess;
        }
    }
    cudaError_t e = cudaMalloc(p, nbytes);
    if (e != cudaSuccess && g_pool_big_bytes) {       // make room: drop what we cached and retry once
        cudaGetLastError();
        pool_drain_big();
        e = cudaMalloc(p, nbytes);
    }
    return e;
}

static void pool_release(void *p, size_t nbytes) {
    if (nbytes <= kPoolSmall) {
        if (g_pool_free.size() < 256) { g_pool_free.emplace_back(nbytes, p); return; }
    } else if (g_pool_big_bytes + nbytes <= pool_big_cap() && g_pool_free.size() < 256) {
        g_pool_free.emplace_back(nbytes, p);
        g_pool_big_bytes += nbytes;
        return;
    }
    cudaFree(p);
}

static unsigned long long g_staged_outstanding = 0;    // pool buffers Staging holds (b2_staging_outstanding)

int Staging::array(const b2_dataobj *obj, int ndim, bool written, DevArray *&out, bool copy_in) {
    DevArray &x = arrays_.emplace_back();
    out = &x;
    x.written = written;
    if (!obj) { set_error("stage_in: NULL dataobj"); return B2_ERR_INVALID; }
    if (!obj->size) { set_error("stage_in: dataobj without `size`"); return B2_ERR_INVALID; }
    for (int i = 0; i < ndim; ++i)
        if (obj->size[i] <= 0) { set_error("stage_in: non-positive extent %d on dim %d", obj->size[i], i); return B2_ERR_INVALID; }
    x.ndim = ndim;
    size_t n = 1;
    for (int i = 0; i < ndim; ++i) { x.size[i] = obj->size[i]; n *= (size_t)obj->size[i]; }
    x.nbytes = obj->nbytes ? (size_t)obj->nbytes : n * 4;
    x.h = obj->data;
    if (obj->dmap) {
        x.d = obj->dmap;
        return B2_OK;
    }
    if (!obj->data) { set_error("stage_in: dataobj has neither data nor dmap"); return B2_ERR_INVALID; }
    B2_CUDA(pool_alloc(&x.d, x.nbytes), B2_ERR_MEMORY);
    x.owned = true;
    ++g_staged_outstanding;
    if (copy_in)
        B2_CUDA(cudaMemcpyAsync(x.d, x.h, x.nbytes, cudaMemcpyHostToDevice, stream()),
                B2_ERR_MEMORY);
    return B2_OK;
}

int Staging::scratch(size_t nbytes, DevArray *&out) {
    DevArray &x = arrays_.emplace_back();
    out = &x;
    x.nbytes = nbytes;
    x.pooled = false;
    if (cudaMalloc(&x.d, nbytes) != cudaSuccess) {
        cudaGetLastError();                        // not sticky: later calls must not see it
        x.d = nullptr;
        set_error("device scratch of %zu bytes: out of memory", nbytes);
        return B2_ERR_MEMORY;
    }
    x.owned = true;
    ++g_staged_outstanding;
    return B2_OK;
}

int Staging::finish(int code) {
    cudaError_t e = cudaSuccess;
    if (code == B2_OK || code == B2_ERR_NAN)
        for (const DevArray &x : arrays_)
            if (x.written && (x.owned || x.host_io)) {
                const cudaError_t c = cudaMemcpyAsync(x.h, x.d, x.nbytes, cudaMemcpyDeviceToHost, stream());
                if (e == cudaSuccess) e = c;
            }
    // the copies above, and whatever kernels and copies in flight still use the buffers
    const cudaError_t s = cudaStreamSynchronize(stream());
    if (e == cudaSuccess) e = s;
    for (DevArray &x : arrays_)
        if (x.owned) {
            if (x.pooled) pool_release(x.d, x.nbytes);
            else cudaFree(x.d);
            --g_staged_outstanding;
        }
    arrays_.clear();
    if (code == B2_OK && e != cudaSuccess) {
        set_error("stage_out: %s", cudaGetErrorString(e));
        return B2_ERR_MEMORY;
    }
    return code;
}

int cached_scratch(ScratchSlot &s, size_t elems, float **out) {
    if (s.elems != elems) {
        if (s.p) cudaFree(s.p);
        s.p = nullptr;
        s.elems = 0;
        B2_CUDA(cudaMalloc(&s.p, elems * sizeof(float)), B2_ERR_MEMORY);
        s.elems = elems;
    }
    *out = s.p;
    return B2_OK;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int encode_tmap(CUtensorMap *tm, const void *base, int rank, const int *dims, int bz, int by, const char *who) {
    static PFN_encodeTiled enc = nullptr;     // the driver entry point, looked up on first use
    if (!enc) {
        void *fp = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess) {
            set_error("%s: cuTensorMapEncodeTiled entry point not available", who);
            return B2_ERR_DEVICE;
        }
        enc = reinterpret_cast<PFN_encodeTiled>(fp);
    }
    cuuint64_t gdim[4], gstr[3];
    cuuint32_t box[4] = {(cuuint32_t)bz, (cuuint32_t)by, 1, 1}, estr[4] = {1, 1, 1, 1};
    cuuint64_t stride = 4;
    for (int i = 0; i < rank; ++i) {
        gdim[i] = (cuuint64_t)dims[i];
        stride *= gdim[i];
        if (i < rank - 1) gstr[i] = stride;
    }
    const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void *>(base), gdim, gstr,
                           box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("%s: cuTensorMapEncodeTiled failed (%d) rank=%d box=(%d,%d)", who, (int)r, rank, bz, by);
        return B2_ERR_DEVICE;
    }
    return B2_OK;
}

int grid_halo(const char *who, const char *name, const b2_dataobj *obj, const DevArray &x, int lead,
              const DevArray &u, int nd, int so, int need) {
    const int n0 = u.size[1] - 2 * so;                   // the grid's extent on the first space dim
    const int h = need >= 0 ? need : obj->hsize ? obj->hsize[2 * lead] : (x.size[lead] - n0) / 2;
    for (int d = 0; d < nd; ++d)
        if (h < 0 || x.size[lead + d] != u.size[d + 1] - 2 * so + 2 * h) {
            set_error("%s: %s extent %d on dim %d does not match the grid (halo %d)", who, name, x.size[lead + d], d, h);
            return -1;
        }
    return h;
}

__global__ void k_check_finite(const float *__restrict__ f, size_t n, int *flag) {
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    bool bad = false;
    for (; i < n; i += stride) bad |= !isfinite(f[i]);
    if (bad) atomicOr(flag, 1);
}

int check_finite(const float *f, size_t n, const char *field, int time) {
    static int *d_flag = nullptr;
    if (!d_flag) B2_CUDA(cudaMalloc(&d_flag, sizeof(int)), B2_ERR_MEMORY);
    B2_CUDA(cudaMemsetAsync(d_flag, 0, sizeof(int), stream()), B2_ERR_MEMORY);
    B2_SM_COUNT(sms);
    k_check_finite<<<sms * 4, 256, 0, stream()>>>(f, n, d_flag);
    count_launch();
    int h = 0;
    B2_CUDA(cudaMemcpyAsync(&h, d_flag, sizeof(int), cudaMemcpyDeviceToHost, stream()), B2_ERR_MEMORY);
    B2_CUDA(cudaStreamSynchronize(stream()), B2_ERR_DEVICE);
    if (h) { set_error("NaN/Inf detected in %s at time=%d", field, time); return B2_ERR_NAN; }
    return B2_OK;
}

int sync_call(const char *who) {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream());
    if (e != cudaSuccess) {
        set_error("%s: device error: %s", who, cudaGetErrorString(e));
        return B2_ERR_LAUNCH;
    }
    return B2_OK;
}

static cudaEvent_t g_loop_ev[2] = {nullptr, nullptr};     // created once (the process is bound to one device)

int loop_timer_start(b2_profiler *timers) {
    if (!timers) return B2_OK;
    if (!g_loop_ev[1]) {
        B2_CUDA(cudaEventCreate(&g_loop_ev[0]), B2_ERR_DEVICE);
        B2_CUDA(cudaEventCreate(&g_loop_ev[1]), B2_ERR_DEVICE);
    }
    B2_CUDA(cudaEventRecord(g_loop_ev[0], stream()), B2_ERR_DEVICE);
    return B2_OK;
}

int loop_finish(const char *who, b2_profiler *timers) {
    if (timers) B2_CUDA(cudaEventRecord(g_loop_ev[1], stream()), B2_ERR_DEVICE);
    if (int rc = sync_call(who)) return rc;
    float ms = 0.f;
    if (timers && cudaEventElapsedTime(&ms, g_loop_ev[0], g_loop_ev[1]) == cudaSuccess) timers->section0 += ms * 1e-3;
    return B2_OK;
}

// Imaging condition (reference: `Inc(grad, -u * v.dt2)`, acoustic/operators.py:222; the TTI gradient's
// `Inc(dm, -(u0 * du.dt2 + v0 * dv.dt2))`, tti/operators.py `JacobianAdjOperator`, with the second pair):
// grad[p] -= usave[time][p] * (v[t+1][p] - 2 v[t][p] + v[t-1][p]) / dt^2 (+ the same of us2, w) over the iterated box.
__global__ void __launch_bounds__(256) k_imaging(ImgK k) {
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (z >= k.n2 || y >= k.n1) return;
    for (int x = blockIdx.z; x < k.n0; x += gridDim.z) {
        const long long i = (long long)(k.o0 + x) * k.sx + (long long)(k.o1 + y) * k.sy + (k.o2 + z);
        const long long g = (long long)(k.g0 + x) * k.gsx + (long long)(k.g1 + y) * k.gsy + (k.g2 + z);
        const float d2 = (k.v1[i] - 2.0f * k.v0[i] + k.v2[i]) * k.inv_dt2;
        if (k.us2) {
            const float e2 = (k.w1[i] - 2.0f * k.w0[i] + k.w2[i]) * k.inv_dt2;
            k.grad[g] = k.grad[g] - fmaf(k.us[i], d2, k.us2[i] * e2);
        } else {
            k.grad[g] = k.grad[g] - k.us[i] * d2;
        }
    }
}

int launch_imaging(const ImgK &ik) {
    dim3 blk(64, 4, 1), grd((ik.n2 + 63) / 64, (ik.n1 + 3) / 4, (unsigned)(ik.n0 < 65535 ? ik.n0 : 65535));
    k_imaging<<<grd, blk, 0, stream()>>>(ik);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

}  // namespace b2

using namespace b2;

extern "C" {

int b2_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

const char *b2_last_error(void) { return g_last_error.c_str(); }

int b2_device_pci_bus_id(int deviceid, char *out, int len) {
    if (!out || len < 16) return B2_ERR_INVALID;
    if (cudaDeviceGetPCIBusId(out, len, deviceid) != cudaSuccess) { cudaGetLastError(); return B2_ERR_DEVICE; }
    return B2_OK;
}

const char *b2_version(void) { return "b200stencil 0.1 (sm_90a)"; }

unsigned long long b2_launch_count(void) { return g_launches; }

const char *b2_last_sweep_kernel(void) { return g_sweep_kernel; }

int b2_last_iso_coef_reuse(void) { return iso_coef_reuse_count(); }

void b2_kernel_timing_enable(int on) { g_timing_on = on != 0; }

void b2_kernel_timing_reset(void) { g_timing_used = 0; }

double b2_kernel_timing_ms(int *nlaunches) {
    double total = 0.0;
    int n = 0;
    for (size_t i = 0; i + 1 < g_timing_used; i += 2) {
        float ms = 0.f;
        cudaEventSynchronize(g_timing_events[i + 1]);
        if (cudaEventElapsedTime(&ms, g_timing_events[i], g_timing_events[i + 1]) == cudaSuccess) {
            total += ms;
            ++n;
        }
    }
    if (nlaunches) *nlaunches = n;
    return n ? total / n : 0.0;
}

void *b2_malloc_device(unsigned long nbytes, int deviceid) {
    void *p = nullptr;
    if (use_device(deviceid)) return nullptr;
    if (cudaMalloc(&p, nbytes) != cudaSuccess) { set_error("cudaMalloc(%lu bytes) failed", nbytes); return nullptr; }
    return p;
}

void b2_free_device(void *p, int deviceid) {
    if (use_device(deviceid)) return;
    cudaFree(p);
}

int b2_memcpy_h2d(void *dst, const void *src, unsigned long nbytes, int deviceid) {
    if (int rc = use_device(deviceid)) return rc;
    B2_CUDA(cudaMemcpyAsync(dst, src, nbytes, cudaMemcpyHostToDevice, stream()), B2_ERR_MEMORY);
    B2_CUDA(cudaStreamSynchronize(stream()), B2_ERR_MEMORY);
    return B2_OK;
}

int b2_memcpy_d2h(void *dst, const void *src, unsigned long nbytes, int deviceid) {
    if (int rc = use_device(deviceid)) return rc;
    B2_CUDA(cudaMemcpyAsync(dst, src, nbytes, cudaMemcpyDeviceToHost, stream()), B2_ERR_MEMORY);
    B2_CUDA(cudaStreamSynchronize(stream()), B2_ERR_MEMORY);
    return B2_OK;
}

int b2_memset_device(void *dst, int value, unsigned long nbytes, int deviceid) {
    if (int rc = use_device(deviceid)) return rc;
    B2_CUDA(cudaMemsetAsync(dst, value, nbytes, stream()), B2_ERR_MEMORY);
    return B2_OK;
}

int b2_synchronize(int deviceid) {
    if (int rc = use_device(deviceid)) return rc;
    B2_CUDA(cudaStreamSynchronize(stream()), B2_ERR_DEVICE);
    return B2_OK;
}

void b2_set_stream(void *s) { g_user_stream = (cudaStream_t)s; }

void b2_staging_cache_release(void) {
    std::lock_guard<std::mutex> lock(api_mutex());
    pool_drain_big();
}

unsigned long long b2_staging_outstanding(void) {
    std::lock_guard<std::mutex> lock(api_mutex());
    return g_staged_outstanding;
}

}  // extern "C"
