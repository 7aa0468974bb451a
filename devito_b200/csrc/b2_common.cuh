// Shared host/device helpers for libb200stencil (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <string>
#include <mutex>
#include "b200stencil.h"

#define B2_MAX_RADIUS 8

// Error codes (devito/passes/iet/errors.py:192-198 uses 100 and 200..203)
#define B2_OK 0
#define B2_ERR_NAN 100
#define B2_ERR_DEVICE 200
#define B2_ERR_LAUNCH 201
#define B2_ERR_MEMORY 202
#define B2_ERR_COMM 203
#define B2_ERR_INVALID 210

namespace b2 {

extern thread_local std::string g_last_error;
extern cudaStream_t g_stream;               // library stream (lazily created)
extern cudaStream_t g_user_stream;          // optional externally owned stream
extern unsigned long long g_launches;

void set_error(const char *fmt, ...);
cudaStream_t stream();
// The library keeps device-bound state (stream, staging pool, scratch tables, kernel attributes) and
// is built for one process per GPU, like the reference's device path (one MPI rank per GPU):
// use_device() selects `dev` and binds the process to it on first use; a later call naming another
// device fails with B2_ERR_INVALID instead of touching memory of the wrong GPU.
int use_device(int dev);
// serialises the compute entry points (ctypes callers drop the GIL; the global state above is not
// re-entrant)
std::mutex &api_mutex();

// kernel timing (CUDA events around every stencil launch when enabled)
void timing_begin();
void timing_end();

// name of the sweep kernel variant launched (host-side only): read back with b2_last_sweep_kernel, so that a test
// can tell which of the run-time selected variants ran. Set by the launchers next to timing_begin(); cleared at the
// start of every b2_iso_forward / b2_tti_forward call.
void note_sweep_kernel(const char *fmt, ...);

inline void count_launch() { ++g_launches; }

// SMs of the current device (cached on first use; the library serves one device per process);
// 0 after set_error() when the device cannot be queried
int sm_count();
// `int var` = the SM count, or return B2_ERR_DEVICE from the enclosing function
#define B2_SM_COUNT(var)                          \
    const int var = sm_count();                   \
    if (var <= 0) return B2_ERR_DEVICE

// Length of the x-chunks a 2.5-D sweep is cut into. With `tiles` yz-tiles and one CTA per SM the
// grid runs in ceil(tiles*nchunks/SMs) rounds; each chunk re-reads `prime` priming planes. Pick the
// chunk count that minimises (wave quantisation) x (priming overhead) among chunks of at most 256
// planes (longer chunks make a longer kernel tail — the last CTAs running alone cannot saturate
// HBM — as the CTA duration grows).
inline int choose_chunk_len(long long sms, int tiles, int xcount, int prime, int min_len) {
    double best = 1e30;
    int best_n = 1;
    for (int n = 1; n <= 64; ++n) {
        const int lx = (xcount + n - 1) / n;
        if (n > 1 && lx < min_len) break;
        if (lx > 256 && (xcount + n) / (n + 1) >= min_len) continue;
        const double ctas = (double)tiles * n;
        const double rounds = (double)((long long)((ctas + sms - 1) / sms));
        const double cost = rounds * (double)sms / ctas * (1.0 + (double)prime / lx);
        if (cost < best - 1e-9) { best = cost; best_n = n; }
    }
    return (xcount + best_n - 1) / best_n;
}

#define B2_CUDA(call, code)                                                        \
    do {                                                                           \
        cudaError_t _e = (call);                                                   \
        if (_e != cudaSuccess) {                                                   \
            b2::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call,             \
                          cudaGetErrorString(_e));                                 \
            return (code);                                                         \
        }                                                                          \
    } while (0)

// A dense f32/i32 array made device-visible: either resident (dmap) or staged by us.
struct DevArray {
    void *d = nullptr;       // device pointer
    void *h = nullptr;       // host pointer (may be null when resident)
    size_t nbytes = 0;
    bool owned = false;      // we cudaMalloc'ed it -> copy back (if written) + free
    int ndim = 0;
    int size[4] = {1, 1, 1, 1};
};

// ndim: number of entries of obj->size to read
int stage_in(const b2_dataobj *obj, int ndim, DevArray &out, bool copy_in);
int stage_out(DevArray &a, bool copy_back);

// Imaging condition over the iterated box, after the step and its injection (k_imaging, b2_api_iso.cu):
// grad -= us * (v1 - 2 v0 + v2) / dt^2, and with us2 != nullptr also - us2 * (w1 - 2 w0 + w2) / dt^2 (the TTI
// gradient's second pair). 24 B/point with one pair, 40 with two.
struct ImgK {
    float *__restrict__ grad;
    const float *__restrict__ us;
    const float *__restrict__ v0;
    const float *__restrict__ v1;
    const float *__restrict__ v2;
    const float *__restrict__ us2;
    const float *__restrict__ w0;
    const float *__restrict__ w1;
    const float *__restrict__ w2;
    long long sx, sy, gsx, gsy;      // strides of the wavefields / of grad
    int n0, n1, n2, o0, o1, o2, g0, g1, g2;
    float inv_dt2;
};
int launch_imaging(const ImgK &k);

// section timers: CUDA-event accumulation per section, flushed to b2_profiler at exit
struct SectionTimer {
    bool enabled = false;
    cudaEvent_t ev[5];
    void init(bool on);
    void destroy();
};

}  // namespace b2
