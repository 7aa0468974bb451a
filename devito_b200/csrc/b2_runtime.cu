// Runtime plumbing of libb200stencil: stream, error string, staging of `struct dataobj`
// arrays (host <-> device, mirroring the reference's `acc enter data copyin / exit data
// copyout` placed by DeviceAwareDataManager, devito/passes/iet/definitions.py:636-671),
// launch counter, kernel timing, small device-memory utilities.
#include "b2_common.cuh"
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

int stage_in(const b2_dataobj *obj, int ndim, DevArray &out, bool copy_in) {
    if (!obj) { set_error("stage_in: NULL dataobj"); return B2_ERR_INVALID; }
    if (!obj->size) { set_error("stage_in: dataobj without `size`"); return B2_ERR_INVALID; }
    for (int i = 0; i < ndim; ++i)
        if (obj->size[i] <= 0) { set_error("stage_in: non-positive extent %d on dim %d", obj->size[i], i); return B2_ERR_INVALID; }
    out.ndim = ndim;
    size_t n = 1;
    for (int i = 0; i < ndim; ++i) { out.size[i] = obj->size[i]; n *= (size_t)obj->size[i]; }
    out.nbytes = obj->nbytes ? (size_t)obj->nbytes : n * 4;
    out.h = obj->data;
    if (obj->dmap) {
        out.d = obj->dmap;
        out.owned = false;
        return B2_OK;
    }
    if (!obj->data) { set_error("stage_in: dataobj has neither data nor dmap"); return B2_ERR_INVALID; }
    B2_CUDA(pool_alloc(&out.d, out.nbytes), B2_ERR_MEMORY);
    out.owned = true;
    if (copy_in)
        B2_CUDA(cudaMemcpyAsync(out.d, out.h, out.nbytes, cudaMemcpyHostToDevice, stream()),
                B2_ERR_MEMORY);
    return B2_OK;
}

int stage_out(DevArray &a, bool copy_back) {
    if (!a.owned) return B2_OK;
    int rc = B2_OK;
    if (copy_back) {
        cudaError_t e = cudaMemcpyAsync(a.h, a.d, a.nbytes, cudaMemcpyDeviceToHost, stream());
        if (e == cudaSuccess) e = cudaStreamSynchronize(stream());
        if (e != cudaSuccess) { set_error("stage_out: %s", cudaGetErrorString(e)); rc = B2_ERR_MEMORY; }
    }
    if (!copy_back) cudaStreamSynchronize(stream());   // pending async H2D/kernels still use it
    pool_release(a.d, a.nbytes);
    a.d = nullptr;
    a.owned = false;
    return rc;
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

}  // extern "C"
