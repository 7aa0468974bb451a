// Shared host/device helpers for libb200stencil (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <deque>
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

// integer value of the environment variable `name` (read per call), or `dflt` when it is unset
inline int env_int(const char *name, int dflt) {
    const char *v = getenv(name);
    return v ? atoi(v) : dflt;
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

// ring-buffer slot of time level `time` in an array of T slots
inline int slot(int time, int T) { return ((time % T) + T) % T; }

// TMA tensor map over a dense f32 array of `rank` (3 or 4) dims, extents `dims` innermost first (z, y, x[, t]), box
// (bz, by, 1[, 1]). B2_ERR_DEVICE after set_error naming `who` when the driver cannot encode it.
int encode_tmap(CUtensorMap *tm, const void *base, int rank, const int *dims, int bz, int by, const char *who);

// One buffer of device scratch that a sweep file keeps across calls (released with the process).
struct ScratchSlot {
    float *p = nullptr;
    size_t elems = 0;
};
// `*out` = slot s holding `elems` floats, re-allocated when its size differs (uninitialised then)
int cached_scratch(ScratchSlot &s, size_t elems, float **out);

// A dense f32/i32 array made device-visible: either resident (dmap) or staged by us.
struct DevArray {
    void *d = nullptr;       // device pointer
    void *h = nullptr;       // host pointer (may be null when resident)
    size_t nbytes = 0;
    bool owned = false;      // we allocated it: released when the call ends
    bool written = false;    // the call writes it: copied back to `h` (see Staging::finish)
    bool host_io = false;    // ... even though not owned: the caller's own device buffer next to its host array
    bool pooled = true;      // an owned buffer goes back to the staging pool (false: freed outright)
    int ndim = 0;
    int size[4] = {1, 1, 1, 1};
};

// The arrays one entry-point call makes device-visible. The deque keeps their addresses stable: plans point into them.
class Staging {
  public:
    // Stages `obj` (`ndim` extents): resident arrays (dmap) are used in place, host arrays are copied in (copy_in)
    // to a buffer of the staging pool. `out` is set even when this fails, and finish() releases what it holds.
    int array(const b2_dataobj *obj, int ndim, bool written, DevArray *&out, bool copy_in = true);
    // Device scratch of `nbytes` for the call alone (uninitialised, never copied): freed by finish(), not pooled, so
    // that the memory it held is free again when the call returns.
    int scratch(size_t nbytes, DevArray *&out);
    // Ends the call: the written arrays go back to the host iff `code` is B2_OK or B2_ERR_NAN, every staged buffer
    // is released whatever the code. Returns `code`, or the first copy-back error when `code` is B2_OK.
    int finish(int code);

  private:
    std::deque<DevArray> arrays_;
};

// The halo of `x`, an array of u's grid (u: (time, space...), halo so) after `lead` leading dims: `need` when
// need >= 0 (the array must have u's space layout), else obj->hsize's, else inferred from the extents. Every space
// extent must be the grid's plus twice that halo. Returns the halo, or -1 after set_error naming the array.
int grid_halo(const char *who, const char *name, const b2_dataobj *obj, const DevArray &x, int lead,
              const DevArray &u, int nd, int so, int need = -1);

// errctl (reference: errctl='max', passes/iet/errors.py:59-85): the wavefields are checked every 100th step of the
// loop over [first, ...] and after its `last` step
inline bool errctl_due(int time, int first, int last) { return (time - first) % 100 == 99 || time == last; }
// NaN/Inf check of n floats of `field`, written at step `time`: B2_ERR_NAN after set_error when one is found. Waits for
// the result.
int check_finite(const float *f, size_t n, const char *field, int time);

// Waits for the work the call queued: a launch or device error sets "<who>: device error: ..." and gives
// B2_ERR_LAUNCH.
int sync_call(const char *who);
// The end of a call whose timers report the time loop as section0 only: loop_timer_start() before the loop,
// loop_finish() after it synchronises (sync_call) and adds the loop's time to timers->section0. Null timers: no timing.
int loop_timer_start(b2_profiler *timers);
int loop_finish(const char *who, b2_profiler *timers);

// Imaging condition over the iterated box, after the step and its injection (k_imaging, b2_runtime.cu):
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

// The imaging condition over plan p's box (IsoPlan or TtiPlan) at time level slots t0 (centre), t1, t2 of the
// wavefields f and f2 (f2, us2 null: one pair); `us` / `us2` are the saved wavefields at this time step, `gh` grad's halo.
template <class Plan>
int launch_imaging(const Plan &p, const DevArray &grad, int gh, const float *us, const float *f, const float *us2,
                   const float *f2, int t0, int t1, int t2) {
    auto at = [&](const float *x, int t) { return x ? x + (size_t)t * p.slot_elems : nullptr; };
    ImgK k;
    k.grad = (float *)grad.d;
    k.us = us; k.v0 = at(f, t0); k.v1 = at(f, t1); k.v2 = at(f, t2);
    k.us2 = us2; k.w0 = at(f2, t0); k.w1 = at(f2, t1); k.w2 = at(f2, t2);
    k.sx = p.sx; k.sy = p.sy;
    k.gsy = grad.size[2];
    k.gsx = (long long)grad.size[1] * grad.size[2];
    k.n0 = p.n[0]; k.n1 = p.n[1]; k.n2 = p.n[2];
    k.o0 = p.o[0]; k.o1 = p.o[1]; k.o2 = p.o[2];
    // o[0] == 0 only on the dummy leading dim of a 2-D plan (a grid dim starts at its halo, so >= 1): index 0 there
    k.g0 = p.o[0] == 0 ? 0 : p.o[0] - p.so + gh;
    k.g1 = p.o[1] - p.so + gh; k.g2 = p.o[2] - p.so + gh;
    k.inv_dt2 = 1.0f / (p.dt * p.dt);
    return launch_imaging(k);
}

// The iteration box of a call (x_m .. z_M) in the internal 3-dim convention: a 1-D or 2-D grid gets leading dummy
// dims of extent 1 (origin 0). The plans of the wave entry points derive from it.
struct Box {
    int a[3] = {1, 1, 1};        // allocated extents
    int n[3] = {1, 1, 1};        // iteration extents (<= 0: nothing to do)
    int o[3] = {0, 0, 0};        // array index of the first iterated point
    long long sx = 0, sy = 0;    // element strides of dim0 / dim1 (dim2 stride = 1)
    size_t slot_elems = 0;       // elements of one time slot
    int tsize = 3;               // time slots
    int so = 0;                  // halo on every grid dim
};

// The box of `args` on an `nd`-dim grid (1..3) whose field has the extents `size` (time slots, then the space
// extents) and the halo `halo` on every space dim.
template <class Args>
Box make_box(const Args *args, int nd, const int *size, int halo) {
    const int lo[3] = {args->x_m, args->y_m, args->z_m}, hi[3] = {args->x_M, args->y_M, args->z_M};
    Box b;
    b.tsize = size[0];
    b.so = halo;
    for (int d = 0; d < nd; ++d) {
        const int di = 3 - nd + d;
        b.a[di] = size[d + 1];
        b.n[di] = hi[d] - lo[d] + 1;
        b.o[di] = lo[d] + halo;
    }
    b.sy = b.a[2];
    b.sx = (long long)b.a[1] * b.a[2];
    b.slot_elems = (size_t)b.a[0] * b.a[1] * b.a[2];
    return b;
}

// A wave call's box against its allocation, internal dim 0, 1, 2 in turn: an empty extent sets `empty` (the call has
// nothing to do), a box grown by `reach` cells on either side of a grid dim that leaves [0, a) refuses the call
// (B2_ERR_INVALID after set_error naming `who`). `reach`: how far the stencil reads beyond the point it updates.
inline int check_reach(const char *who, const Box &b, int nd, int reach, bool &empty) {
    empty = false;
    for (int d = 0; d < 3; ++d) {
        if (b.n[d] <= 0) { empty = true; return B2_OK; }
        if (d < 3 - nd) continue;                               // a dummy dim: extent 1, nothing read around it
        if (b.o[d] - reach < 0 || b.o[d] + b.n[d] - 1 + reach >= b.a[d]) {
            set_error("%s: iteration range [%d,%d] + reach %d leaves the allocated array (extent %d) on dim %d", who,
                      b.o[d] - b.so, b.o[d] - b.so + b.n[d] - 1, reach, b.a[d], d - (3 - nd));
            return B2_ERR_INVALID;
        }
    }
    return B2_OK;
}

}  // namespace b2
