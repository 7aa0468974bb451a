// C-ABI entry point b2_iso_forward: the whole time loop of the reference's generated
// `Forward` function (examples/seismic/acoustic/operators.py:113-150 builds it; loop shape
// printed in examples/seismic/tutorials/08_snapshotting.ipynb:473-505):
//
//   for time in [time_m, time_M]:  t0 = time % T, t1 = (time+1) % T, t2 = (time+T-1) % T
//       [haloupdate u[t0]]            (devito/mpi/routines.py:457-510; here NCCL, b2_halo.cu)
//       section0: u[t1] = stencil(u[t0], u[t2], m, damp)
//       section1: u[t1] += inject(src[time])
//       section2: rec[time] = interpolate(u[t0] | u[t1])
#include "b2_iso.cuh"
#include "b2_sparse.cuh"
#include "b2_halo.cuh"
#include <vector>
#include <cstdlib>
#include <string>
#include <chrono>
#include <algorithm>
#include <climits>

using namespace b2;

namespace b2 {

// Section timing with a reusable pool of CUDA events: 4 events per time step.
struct StepEvents {
    std::vector<cudaEvent_t> ev;
    size_t used = 0;
    bool on = false;
    cudaEvent_t next() {
        if (used == ev.size()) {
            cudaEvent_t e;
            cudaEventCreate(&e);
            ev.push_back(e);
        }
        cudaEvent_t e = ev[used++];
        cudaEventRecord(e, stream());
        return e;
    }
};
static StepEvents g_step_events;

// Host-resident snapshots are not staged as a whole (nsnaps wavefields would not fit in HBM for a
// production run): each snapshot is written into one of two device buffers by k_snapshot and drained
// to the caller's array on a copy stream while the stencil keeps running — the out-of-core saving the
// reference does with asynchronous streaming (devito/passes/clusters/buffering.py, passes/iet/
// asynchrony.py). Only the iteration box travels (cudaMemcpy3DAsync), so the halo of the host
// snapshots keeps its values, exactly like `Eq(usave, u)` over the domain.
struct SnapStreamer {
    bool active = false;
    bool registered = false;         // we pinned the caller's array for the duration of the call
    void *host = nullptr;
    size_t host_bytes = 0;
    float *buf[2] = {nullptr, nullptr};
    size_t one = 0;                  // elements of one snapshot (with its halo)
    int count = 0;
    static cudaStream_t copy_stream;
    static cudaEvent_t filled[2], drained[2];

    int begin(void *host_base, size_t nbytes, size_t one_elems) {
        host = host_base;
        host_bytes = nbytes;
        one = one_elems;
        if (!copy_stream) {
            B2_CUDA(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking), B2_ERR_DEVICE);
            for (int i = 0; i < 2; ++i) {
                B2_CUDA(cudaEventCreateWithFlags(&filled[i], cudaEventDisableTiming), B2_ERR_DEVICE);
                B2_CUDA(cudaEventCreateWithFlags(&drained[i], cudaEventDisableTiming), B2_ERR_DEVICE);
            }
        }
        active = true;               // from here on end() has something to release
        count = 0;
        for (int i = 0; i < 2; ++i) B2_CUDA(cudaMalloc(&buf[i], one * sizeof(float)), B2_ERR_MEMORY);
        // pinned memory makes the copies truly asynchronous; pageable memory still works (the driver
        // stages it), already-pinned memory (e.g. torch pin_memory) is reported as such and left alone
        cudaError_t e = cudaHostRegister(host, host_bytes, cudaHostRegisterDefault);
        registered = (e == cudaSuccess);
        if (!registered) cudaGetLastError();
        return B2_OK;
    }

    // device buffer for the next snapshot, safe to overwrite on the compute stream
    int acquire(float **out) {
        const int b = count & 1;
        if (count >= 2) B2_CUDA(cudaStreamWaitEvent(stream(), drained[b], 0), B2_ERR_DEVICE);
        *out = buf[b];
        return B2_OK;
    }

    // the snapshot kernel has been enqueued: drain the box [d, d + n) of the buffer into host slot `index`
    int release(int index, const int *sz /* x,y,z extents of one snapshot */, const int *d, const int *n) {
        const int b = count & 1;
        B2_CUDA(cudaEventRecord(filled[b], stream()), B2_ERR_DEVICE);
        B2_CUDA(cudaStreamWaitEvent(copy_stream, filled[b], 0), B2_ERR_DEVICE);
        cudaMemcpy3DParms prm = {};
        const size_t pitch = (size_t)sz[2] * sizeof(float);
        prm.srcPtr = make_cudaPitchedPtr(buf[b], pitch, sz[2], sz[1]);
        prm.dstPtr = make_cudaPitchedPtr((float *)host + (size_t)index * one, pitch, sz[2], sz[1]);
        prm.srcPos = make_cudaPos((size_t)d[2] * sizeof(float), d[1], d[0]);
        prm.dstPos = prm.srcPos;
        prm.extent = make_cudaExtent((size_t)n[2] * sizeof(float), n[1], n[0]);
        prm.kind = cudaMemcpyDeviceToHost;
        B2_CUDA(cudaMemcpy3DAsync(&prm, copy_stream), B2_ERR_MEMORY);
        B2_CUDA(cudaEventRecord(drained[b], copy_stream), B2_ERR_DEVICE);
        ++count;
        return B2_OK;
    }

    int end() {
        if (!active) return B2_OK;
        active = false;
        cudaError_t e = cudaStreamSynchronize(copy_stream);
        for (int i = 0; i < 2; ++i) { if (buf[i]) cudaFree(buf[i]); buf[i] = nullptr; }
        if (registered) cudaHostUnregister(host);
        registered = false;
        if (e != cudaSuccess) { set_error("snapshot streaming: %s", cudaGetErrorString(e)); return B2_ERR_MEMORY; }
        return B2_OK;
    }
};
cudaStream_t SnapStreamer::copy_stream = nullptr;
cudaEvent_t SnapStreamer::filled[2] = {nullptr, nullptr};
cudaEvent_t SnapStreamer::drained[2] = {nullptr, nullptr};

}  // namespace b2


// ---------------------------------------------------------------------------------------------------------
// Streamed time loop for a HOST-STAGED apply (the reference's per-apply copy semantics,
// devito/passes/iet/definitions.py:636-671, without its serial copy-in / compute / copy-out):
//
// the x axis is cut into chunks of W planes. Chunk c of u (3 slots), damp and the parameter array travels
// host -> device on a copy stream while the compute stream already time-steps the chunks that arrived —
// skewed: in "phase" p, step s = 1..L updates x in [pW - (s-1)R, (p+1)W - (s-1)R), the dependency cone of
// the R-point stencil, so every read is of planes that are uploaded and at the right time level, and the 3
// rotating time slots are never overwritten early (the argument is spelled out in DESIGN.md §3.6). Planes
// left of (p+1)W - (L-1)R are final after phase p and travel device -> host on a second copy stream while
// the later phases compute (PCIe is full duplex). Injection deposits into the cells of the range just
// updated; receivers add the partial sum over the cells of that range to their trace.
//
// Whole-call time ~ compute + first upload chunk + last download chunk instead of upload + compute + download.
// ---------------------------------------------------------------------------------------------------------
namespace b2 {

static double g_last_profile[5] = {0, 0, 0, 0, 0};

struct StreamedLoop {
    cudaStream_t up = nullptr, down = nullptr;
    std::vector<cudaEvent_t> ev;
    size_t used = 0;
    int init() {
        if (!up) {
            B2_CUDA(cudaStreamCreateWithFlags(&up, cudaStreamNonBlocking), B2_ERR_DEVICE);
            B2_CUDA(cudaStreamCreateWithFlags(&down, cudaStreamNonBlocking), B2_ERR_DEVICE);
        }
        used = 0;
        return B2_OK;
    }
    cudaEvent_t next() {
        if (used == ev.size()) {
            cudaEvent_t e;
            cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
            ev.push_back(e);
        }
        return ev[used++];
    }
};
static StreamedLoop g_streamed;

static bool streamed_wanted(const b2_iso_args *a, const IsoPlan &p, const DevArray &u, bool host_io) {
    const char *e = getenv("B2_STREAM");
    if (e && atoi(e) == 0) return false;
    const bool forced = e && atoi(e) == 2;                 // tests: also on small grids
    if (!(u.owned || host_io) || a->ndim != 3 || !p.use_tma || p.tsize != 3) return false;
    if (a->adjoint || a->free_surface || a->ot4 || a->born_U || a->snap || a->grad) return false;
    // under x-slab decomposition the sweep is skewed along y and every sub-launch does the fused halo step
    if (a->halo && !halo_fused_ok(a->halo, p)) return false;
    const int L = a->time_M - a->time_m + 1;
    const int dim = a->halo ? 1 : 0;
    if (L < 4 || p.n[dim] < 8 * p.radius[dim]) return false;
    return forced || u.nbytes >= ((size_t)1 << 30);
}

// `dim` = the axis the sweep is cut and skewed along: 0 (x; chunks are contiguous plane blocks) on a single device,
// 1 (y) under x-slab decomposition — orthogonal to the decomposed axis, so that every rank runs the SAME schedule
// and each sub-launch is an ordinary fused halo step (peer stores + flag acquire inside the sweep kernel) restricted
// to its rows. (Skewing along x would make a rank's low edge run ahead of its high edge in time, i.e. ahead of the
// neighbour it has to exchange with.) Chunks along y are strided: one 2-D copy per time slot and chunk, contiguous
// pieces of W rows x a2 floats.
static int iso_forward_streamed(const b2_iso_args *a, IsoPlan &p, FieldGeom g, DevArray &u, DevArray *damp,
                                DevArray *param, SparseDev &src, SparseDev &rec, float scalar_scale, float dt2,
                                bool damp_io, bool param_io) {
    int rc;
    StreamedLoop &S = g_streamed;
    if ((rc = S.init())) return rc;
    const bool decomposed = a->halo != nullptr;
    int dim = decomposed ? 1 : 0;
    if (!decomposed) if (const char *e = getenv("B2_STREAM_DIM")) dim = atoi(e) == 1 ? 1 : 0;
    const int n = p.n[dim], R = p.radius[dim], so = p.so, ad = p.a[dim], a0 = p.a[0];
    // ranges [ra, rb) count from the first point of the update box; `org` is that point's domain index along
    // `dim` (x_m or y_m), so range cell i is domain cell org + i and allocated index so + org + i
    const int org = g.lo[dim];
    const int L = a->time_M - a->time_m + 1;
    const size_t plane = (size_t)p.sx, rowlen = (size_t)p.a[2];
    int W = 128;
    if (const char *e = getenv("B2_STREAM_W")) W = atoi(e);
    W = std::max(W, 4 * R);
    W = std::min(W, n);
    const int K = (n + W - 1) / W;                                   // upload chunks
    const int P = (n + (L - 1) * R + W - 1) / W;                     // phases of the skewed sweep
    cudaStream_t cs = stream();
    // x planes that travel (dim 1): the halo planes next to a neighbour rank hold ITS data, not the host's
    const int px0 = (dim == 1 && g.nb_lo) ? so : 0;
    const int px1 = (dim == 1 && g.nb_hi) ? so + p.n[0] : a0;

    // one chunk [lo, hi) (allocated index along `dim`) of a (slot, x, y, z) or (x, y, z) array, host <-> device
    auto copy_chunk = [&](float *dev, float *host, size_t slot_off, int lo, int hi, bool to_device, cudaStream_t st) -> int {
        if (hi <= lo) return B2_OK;
        if (dim == 0) {
            const size_t off = slot_off + (size_t)lo * plane, cnt = (size_t)(hi - lo) * plane * sizeof(float);
            B2_CUDA(cudaMemcpyAsync(to_device ? (void *)(dev + off) : (void *)(host + off),
                                    to_device ? (const void *)(host + off) : (const void *)(dev + off), cnt,
                                    to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost, st), B2_ERR_MEMORY);
        } else {
            const size_t off = slot_off + (size_t)px0 * plane + (size_t)lo * rowlen;
            B2_CUDA(cudaMemcpy2DAsync(to_device ? (void *)(dev + off) : (void *)(host + off), plane * sizeof(float),
                                      to_device ? (const void *)(host + off) : (const void *)(dev + off),
                                      plane * sizeof(float), (size_t)(hi - lo) * rowlen * sizeof(float),
                                      (size_t)(px1 - px0), to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost, st),
                    B2_ERR_MEMORY);
        }
        return B2_OK;
    };

    // everything the compute stream did so far (sparse tables, traces) precedes the copies
    cudaEvent_t ev_start = S.next();
    B2_CUDA(cudaEventRecord(ev_start, cs), B2_ERR_DEVICE);
    B2_CUDA(cudaStreamWaitEvent(S.up, ev_start, 0), B2_ERR_DEVICE);
    B2_CUDA(cudaStreamWaitEvent(S.down, ev_start, 0), B2_ERR_DEVICE);

    const int t0_first = slot(a->time_m, 3);
    if (decomposed) {
        // the first sub-launch exchanges the initial level's boundary planes through NCCL (like the first step of a
        // resident call): they must be on the device, all rows, before anything else
        const int Rx = p.radius[0];
        const size_t so0 = (size_t)t0_first * p.slot_elems;
        const int lo_pl[2] = {so, so + p.n[0] - Rx};
        for (int i = 0; i < 2; ++i) {
            const size_t off = so0 + (size_t)lo_pl[i] * plane;
            B2_CUDA(cudaMemcpyAsync((float *)u.d + off, (const float *)u.h + off, (size_t)Rx * plane * sizeof(float),
                                    cudaMemcpyHostToDevice, S.up), B2_ERR_MEMORY);
        }
    }

    if (decomposed) {
        // ... and exchanged with the neighbours (NCCL, like the first step of a resident call) before the sweep starts
        cudaEvent_t ev_b = S.next();
        B2_CUDA(cudaEventRecord(ev_b, S.up), B2_ERR_DEVICE);
        B2_CUDA(cudaStreamWaitEvent(cs, ev_b, 0), B2_ERR_DEVICE);
        if ((rc = halo_exchange_initial(a->halo, p, t0_first))) return rc;
    }

    // ---- enqueue every upload now: the copy stream works through them in order ----
    std::vector<cudaEvent_t> up_ev(K);
    std::vector<int> ulo(K), uhi(K);
    for (int c = 0; c < K; ++c) {
        ulo[c] = c == 0 ? 0 : uhi[c - 1];
        uhi[c] = c == K - 1 ? ad : std::min(ad, so + org + std::min(n, (c + 1) * W) + R);
        for (int t = 0; t < 3; ++t)
            if ((rc = copy_chunk((float *)u.d, (float *)u.h, (size_t)t * p.slot_elems, ulo[c], uhi[c], true, S.up))) return rc;
        if (damp && damp_io && (rc = copy_chunk((float *)damp->d, (float *)damp->h, 0, ulo[c], uhi[c], true, S.up))) return rc;
        if (param && param_io && (rc = copy_chunk((float *)param->d, (float *)param->h, 0, ulo[c], uhi[c], true, S.up))) return rc;
        up_ev[c] = S.next();
        B2_CUDA(cudaEventRecord(up_ev[c], S.up), B2_ERR_DEVICE);
    }

    // traces are accumulated range by range: clear the rows this call writes
    if (rec.present) {
        const int r0 = std::max(a->time_m, 0), r1 = std::min(a->time_M, rec.nt - 1);
        if (r1 >= r0)
            B2_CUDA(cudaMemsetAsync((float *)rec.data->d + (size_t)r0 * rec.npoint_total, 0,
                                    (size_t)(r1 - r0 + 1) * rec.npoint_total * sizeof(float), cs), B2_ERR_MEMORY);
    }

    auto range_geom = [&](int ra, int rb) {
        FieldGeom q = g;
        q.lo[dim] = org + ra;                                        // FieldGeom bounds are domain indices
        q.hi[dim] = org + rb - 1;
        if (dim == 0) {
            q.nb_lo = ra > 0;        // an interior cut: the cells beyond it belong to another range
            q.nb_hi = rb < n;
            q.restrict_x = true;
        } else {
            q.cut_lo1 = ra > 0;
            q.cut_hi1 = rb < n;
            q.restrict_y = true;
        }
        return q;
    };
    IsoFuse fz;
    if (decomposed && (rc = halo_fuse_desc(a->halo, p, fz))) return rc;

    int dlo = 0;                                                     // allocated index (along dim) already sent back
    for (int ph = 0; ph < P; ++ph) {
        if (ph < K) {
            B2_CUDA(cudaStreamWaitEvent(cs, up_ev[ph], 0), B2_ERR_DEVICE);
            if (dim == 0) rc = iso_coef_tabulate_planes(p, ulo[ph], uhi[ph]);
            else rc = iso_coef_tabulate_rows(p, 0, a0, ulo[ph], uhi[ph]);
            if (rc) return rc;
            if (rec.present && !a->rec_toff) {
                // the initial time level is complete on the chunk that just arrived
                const int ra = std::max(0, ulo[ph] - so - org), rb = std::min(n, uhi[ph] - so - org);
                if (rb > ra)
                    if ((rc = launch_interp(rec, range_geom(ra, rb), p.u + (size_t)t0_first * p.slot_elems, nullptr, a->time_m)))
                        return rc;
            }
        }
        for (int s = 1; s <= L; ++s) {
            const int shift = (s - 1) * R;
            const int rb = std::min(n, (ph + 1) * W - shift);
            if (rb <= 0) break;
            const int ra = std::max(0, ph * W - shift);
            if (ra >= rb) continue;
            const int time = a->time_m + s - 1;
            const int t0 = slot(time, 3), t1 = slot(time + 1, 3), t2 = slot(time - 1, 3);
            float *f1 = p.u + (size_t)t1 * p.slot_elems;
            FieldGeom q = range_geom(ra, rb);
            if (dim == 0) {
                if ((rc = iso_step(p, t0, t2, t1, ra, rb - ra))) return rc;
            } else {
                IsoPlan pr = p;                                   // the same plan restricted to the rows [ra, rb)
                pr.o[1] = p.o[1] + ra;
                pr.n[1] = rb - ra;
                if (decomposed) {
                    if ((rc = halo_step_iso_fused(a->halo, pr, t0, t2, t1))) return rc;
                    q.peer_lo = fz.peer_lo; q.peer_hi = fz.peer_hi;
                    q.off_lo = (long long)t1 * fz.slot_lo + (long long)(p.o[0] + fz.n_lo) * p.sx;
                    q.off_hi = (long long)t1 * fz.slot_hi + (long long)(p.o[0] - p.n[0]) * p.sx;
                    q.nown = p.n[0]; q.pw = p.radius[0];
                } else if ((rc = iso_step(pr, t0, t2, t1, 0, p.n[0]))) {
                    return rc;
                }
            }
            if ((rc = launch_inject(src, q, f1, nullptr, time, p.param_kind, p.param, scalar_scale, dt2))) return rc;
            if (decomposed) {
                if ((rc = halo_fused_signal(a->halo, p.u))) return rc;
                // receivers next to a slab boundary sample halo cells of the level just written: the neighbour's
                // stores of this very sub-launch must have landed
                if (rec.present && (rc = halo_p2p_wait(a->halo))) return rc;
            }
            // time level time+1 is now complete on [ra, rb)
            if (rec.present) {
                const int row = a->rec_toff ? time : time + 1;
                FieldGeom qi = q;
                qi.peer_lo = qi.peer_hi = nullptr;
                if (row <= a->time_M && (rc = launch_interp(rec, qi, f1, nullptr, row))) return rc;
            }
        }
        // what lies left of (ph+1)W - (L-1)R has seen all L steps: send it home while the sweep goes on. Until that
        // bound is positive, the last step has not run its first range, whose sources may still deposit into the
        // cells below the box: nothing there is final yet.
        const int fin = (ph + 1) * W - (L - 1) * R;
        int dhi = ph == P - 1 ? ad : (fin > 0 ? std::min(ad, so + org + fin) : 0);
        if (ph == P - 1 || dhi - dlo >= W / 2) {
            if (dhi > dlo) {
                cudaEvent_t e = S.next();
                B2_CUDA(cudaEventRecord(e, cs), B2_ERR_DEVICE);
                B2_CUDA(cudaStreamWaitEvent(S.down, e, 0), B2_ERR_DEVICE);
                for (int t = 0; t < 3; ++t)
                    if ((rc = copy_chunk((float *)u.d, (float *)u.h, (size_t)t * p.slot_elems, dlo, dhi, false, S.down))) return rc;
                dlo = dhi;
            }
        }
    }
    // the call returns when the last planes are home
    cudaEvent_t ev_down = S.next();
    B2_CUDA(cudaEventRecord(ev_down, S.down), B2_ERR_DEVICE);
    B2_CUDA(cudaStreamWaitEvent(cs, ev_down, 0), B2_ERR_DEVICE);
    return B2_OK;
}

}  // namespace b2

namespace b2 {

// ---------------------------------------------------------------------------------------------------------
// Two-level time loop (k_iso_tma2, DESIGN.md §3.7): each pass advances two time levels for one read of u[t] and
// u[t-1]. u[t+1] goes to its slot, u[t+2] to one of two scratch slots used in turn (so the pass never writes
// cells another CTA may still read as u[t-1]); a later pass reads its u[t] from there, and the levels left in
// scratch are copied into their slots at the end. Only taken when every slot is zero outside the update box and
// no source reaches outside it, so a level held in scratch sees the halo its slot would.
// ---------------------------------------------------------------------------------------------------------
static IsoInj *g_inj = nullptr;
static int *g_iso2_flag = nullptr;

static int two_level_wanted(const b2_iso_args *a, const IsoPlan &p, const DevArray &u, const SparseDev &src,
                            const FieldGeom &g, bool streamed, bool host_io, bool &want) {
    want = false;
    const char *e = getenv("B2_ISO2");
    if (e && atoi(e) == 0) return B2_OK;
    const bool forced = e && atoi(e) == 2;                 // tests: also on small grids
    if (streamed || host_io || u.owned || a->ndim != 3 || a->halo || !iso2_supported(p)) return B2_OK;
    if (a->adjoint || a->free_surface || a->ot4 || a->born_U || a->born_dm || a->snap || a->grad || a->errctl)
        return B2_OK;
    if (a->time_M - a->time_m + 1 < 2) return B2_OK;
    if (!forced && u.nbytes < ((size_t)1 << 30)) return B2_OK;
    if (inject_entry_count(src) > B2_ISO2_MAX_INJ) return B2_OK;
    if (!g_inj || !g_iso2_flag) {
        if (g_inj) cudaFree(g_inj);
        if (g_iso2_flag) cudaFree(g_iso2_flag);
        g_inj = nullptr;
        g_iso2_flag = nullptr;
        if (cudaMalloc(&g_inj, B2_ISO2_MAX_INJ * sizeof(IsoInj)) != cudaSuccess ||
            cudaMalloc(&g_iso2_flag, sizeof(int)) != cudaSuccess) {
            cudaGetLastError();                           // no room: one step per sweep
            if (g_inj) cudaFree(g_inj);
            g_inj = nullptr;
            g_iso2_flag = nullptr;
            return B2_OK;
        }
    }
    B2_CUDA(cudaMemsetAsync(g_iso2_flag, 0, sizeof(int), stream()), B2_ERR_MEMORY);
    int rc;
    if ((rc = iso2_halo_nonzero(p, g_iso2_flag))) return rc;
    if ((rc = launch_inject_entries(src, g, a->time_m, p.param_kind, p.param, 0.f, 0.f, nullptr, g_iso2_flag)))
        return rc;
    int flag = 1;
    B2_CUDA(cudaMemcpyAsync(&flag, g_iso2_flag, sizeof(int), cudaMemcpyDeviceToHost, stream()), B2_ERR_MEMORY);
    B2_CUDA(cudaStreamSynchronize(stream()), B2_ERR_DEVICE);
    if (flag != 0) return B2_OK;
    // two more slot-sized buffers: where they do not fit, the call runs one step per sweep as before
    return iso2_reserve(p, want);
}

// `se` (null: no timers): every `stride`-th pass is bracketed like a sampled step of the one-step loop (sweep |
// injection | interpolation) and counts as two sampled steps in `nsampled`.
static int iso_forward_two_level(const b2_iso_args *a, const IsoPlan &p, const FieldGeom &g, const SparseDev &src,
                                 const SparseDev &rec, float scalar_scale, float dt2, StepEvents *se, int stride,
                                 int &nsampled) {
    int rc;
    float *scr[2];
    if ((rc = iso2_prepare(p, scr))) return rc;
    const int ninj = inject_entry_count(src);
    const size_t bytes = p.slot_elems * sizeof(float);
    auto level = [&](int s) { return p.u + (size_t)s * p.slot_elems; };
    int time = a->time_m;
    if ((a->time_M - a->time_m + 1) % 2) {
        // an odd step count: one ordinary step first
        const int t0 = slot(time, 3), t1 = slot(time + 1, 3), t2 = slot(time - 1, 3);
        if ((rc = iso_step(p, t0, t2, t1, 0, p.n[0]))) return rc;
        if ((rc = launch_inject(src, g, level(t1), nullptr, time, p.param_kind, p.param, scalar_scale, dt2))) return rc;
        if ((rc = launch_interp(rec, g, level(a->rec_toff ? t1 : t0), nullptr, time))) return rc;
        ++time;
    }
    int cur = -1;                  // scratch slot that holds u[time] (-1: its own slot)
    // the injection entries of a pass's first step are written after the previous pass (before the first one here)
    if (ninj && (rc = launch_inject_entries(src, g, time, p.param_kind, p.param, scalar_scale, dt2, g_inj, nullptr)))
        return rc;
    for (int pass = 0; time + 1 <= a->time_M; time += 2, ++pass) {
        const int t0 = slot(time, 3), t1 = slot(time + 1, 3), tm = slot(time - 1, 3);
        const int w = cur == 0 ? 1 : 0;
        const bool events = se && pass % stride == 0 && se->used + 4 <= 16384;
        if (events) { se->next(); nsampled += 2; }
        if ((rc = iso_step2(p, t0, cur, tm, t1, w, g_inj, ninj))) return rc;
        if (events) se->next();
        // step time+1's injection into u[time+2], the next pass's entries, then the two receiver rows
        if ((rc = launch_inject(src, g, scr[w], nullptr, time + 1, p.param_kind, p.param, scalar_scale, dt2))) return rc;
        if (ninj && time + 3 <= a->time_M &&
            (rc = launch_inject_entries(src, g, time + 2, p.param_kind, p.param, scalar_scale, dt2, g_inj, nullptr)))
            return rc;
        if (events) se->next();
        const float *u0 = cur < 0 ? level(t0) : scr[cur];
        if ((rc = launch_interp(rec, g, a->rec_toff ? level(t1) : u0, nullptr, time))) return rc;
        if ((rc = launch_interp(rec, g, a->rec_toff ? scr[w] : level(t1), nullptr, time + 1))) return rc;
        if (events) se->next();
        // u[time] is dead unless it is the last pass's u[t]: copied back below
        if (time + 3 > a->time_M && cur >= 0)
            B2_CUDA(cudaMemcpyAsync(level(t0), scr[cur], bytes, cudaMemcpyDeviceToDevice, stream()), B2_ERR_MEMORY);
        cur = w;
    }
    // u[time_M + 1] sits in scratch
    B2_CUDA(cudaMemcpyAsync(level(slot(a->time_M + 1, 3)), scr[cur], bytes, cudaMemcpyDeviceToDevice, stream()),
            B2_ERR_MEMORY);
    return B2_OK;
}

// One step of the single-device loop at `time` (dir +1: forward, -1: adjoint): the sweep writes level time+dir from
// levels time and time-dir, the free-surface rows are redone when asked, then `src` is injected into the level
// written. `se` (may be null) records an event between the sweep and the injection.
static int iso_sweep_inject(const IsoPlan &p, const FieldGeom &g, const SparseDev &src, int time, int dir, bool fs,
                            float scalar_scale, float dt2, StepEvents *se) {
    const int T = p.tsize, t0 = slot(time, T), t1 = slot(time + dir, T), t2 = slot(time - dir, T);
    int rc;
    if ((rc = iso_step(p, t0, t2, t1, 0, p.n[0]))) return rc;
    if (fs && (rc = iso_fs_fix(p, t0, t2, t1, 0, p.n[0]))) return rc;
    if (se) se->next();
    return launch_inject(src, g, p.u + (size_t)t1 * p.slot_elems, nullptr, time, p.param_kind, p.param, scalar_scale,
                         dt2);
}

}  // namespace b2

extern "C" void b2_last_call_profile(double out[5]) {
    for (int i = 0; i < 5; ++i) out[i] = b2::g_last_profile[i];
}

static int iso_forward_body(const b2_iso_args *a, Staging &st, SnapStreamer &streamer,
                            std::chrono::steady_clock::time_point call_t0) {
    const int nd = a->ndim;
    const int so = a->space_order;
    int rc = B2_OK;

    DevArray *u, *damp = nullptr, *param = nullptr, *grad = nullptr, *usave = nullptr, *bornU = nullptr,
             *borndm = nullptr, *snap = nullptr;
    DevArray snap_host;                           // host snapshots streamed out: described, not staged
    SparseDev src, rec;
    IsoPlan p;

    // A large host-staged wavefield is a candidate for the streamed time loop (copies overlapped with a
    // skewed sweep, iso_forward_streamed): its uploads are then issued chunk by chunk, not here. Whether the
    // call really streams is known once the plan exists; otherwise the deferred copies are issued below.
    // host_io: the caller passed BOTH a host array and its own device buffer for u (and possibly damp / the
    // parameter array): the call moves data -> dmap before and dmap -> data after the loop (streamed when
    // possible). Under x-slab decomposition this is how a host-staged apply keeps using the CUDA-IPC registered
    // device allocations of the peer-memory halo path.
    const bool host_io = a->host_io && a->u->dmap && a->u->data;
    const bool maybe_stream = [&] {
        const char *e = getenv("B2_STREAM");
        if (e && atoi(e) == 0) return false;
        if (nd != 3 || !a->u->data || !a->damp) return false;
        if (a->u->dmap && !host_io) return false;
        if (a->adjoint || a->free_surface || a->ot4 || a->born_U || a->born_dm || a->snap || a->grad || a->usave)
            return false;
        return true;
    }();
    if ((rc = st.array(a->u, nd + 1, true, u, !maybe_stream))) return rc;
    u->host_io = host_io;
    if (a->damp && (rc = st.array(a->damp, nd, false, damp, !maybe_stream))) return rc;
    if (a->param_kind != B2_PARAM_SCALAR) {
        if (!a->param) { set_error("b2_iso_forward: param array missing"); return B2_ERR_INVALID; }
        if ((rc = st.array(a->param, nd, false, param, !maybe_stream))) return rc;
    }
    if ((rc = sparse_stage_pair("b2_iso_forward", st, a->src, a->rec, nd, so, src, rec))) return rc;
    int gh = 0;
    if (a->grad || a->usave) {
        if (!a->grad || !a->usave || nd != 3) {
            set_error("b2_iso_forward: the imaging condition needs both grad and usave (3-D)");
            return B2_ERR_INVALID;
        }
        if ((rc = st.array(a->grad, 3, true, grad))) return rc;
        if ((rc = st.array(a->usave, 4, false, usave))) return rc;
        // k_imaging reads usave with u's strides and writes grad inside its extents
        if (grid_halo("b2_iso_forward", "usave", a->usave, *usave, 1, *u, 3, so, so) < 0 ||
            (gh = grid_halo("b2_iso_forward", "grad", a->grad, *grad, 0, *u, 3, so)) < 0)
            return B2_ERR_INVALID;
    }

    const bool born = a->born_U || a->born_dm;
    int dmh = 0;
    if (born) {
        if (!a->born_U || !a->born_dm || nd != 3 || a->adjoint || a->grad || a->free_surface || a->ot4) {
            set_error("b2_iso_forward: Born modelling needs born_U and born_dm, 3-D, forward in time, and is "
                      "not combined with a free surface, OT4 or the imaging condition");
            return B2_ERR_INVALID;
        }
        if ((rc = st.array(a->born_U, 4, true, bornU))) return rc;
        if ((rc = st.array(a->born_dm, 3, false, borndm))) return rc;
        for (int d = 0; d < 4; ++d)
            if (bornU->size[d] != u->size[d]) {
                set_error("b2_iso_forward: born_U must have the layout of u");
                return B2_ERR_INVALID;
            }
        if ((dmh = grid_halo("b2_iso_forward", "born_dm", a->born_dm, *borndm, 0, *u, 3, so)) < 0) return B2_ERR_INVALID;
    }

    int snap_h = 0;
    if (a->snap) {
        if (a->snap_factor < 1 || a->adjoint) {
            set_error("b2_iso_forward: snapshots need snap_factor >= 1 and forward time stepping");
            return B2_ERR_INVALID;
        }
        const bool stream_out = !a->snap->dmap && a->snap->data && nd == 3 &&
                                !(getenv("B2_SNAP_STREAM") && atoi(getenv("B2_SNAP_STREAM")) == 0);
        if (stream_out) {
            // describe the array without allocating it on the device
            if (!a->snap->size) { set_error("b2_iso_forward: snapshot dataobj without `size`"); return B2_ERR_INVALID; }
            snap = &snap_host;
            snap->ndim = nd + 1;
            for (int d = 0; d <= nd; ++d) snap->size[d] = a->snap->size[d];
            snap->h = a->snap->data;
        } else if ((rc = st.array(a->snap, nd + 1, true, snap))) {
            return rc;
        }
        if ((snap_h = grid_halo("b2_iso_forward", "snapshot", a->snap, *snap, 1, *u, nd, so)) < 0) return B2_ERR_INVALID;
        if (a->time_m < 0 || a->time_M / a->snap_factor >= snap->size[0]) {
            set_error("b2_iso_forward: time_M=%d needs %d snapshots, the array holds %d", a->time_M,
                      a->time_M / a->snap_factor + 1, snap->size[0]);
            return B2_ERR_INVALID;
        }
        if (stream_out) {
            const size_t one = (size_t)snap->size[1] * snap->size[2] * snap->size[3];
            if ((rc = streamer.begin(snap->h, one * snap->size[0] * sizeof(float), one))) return rc;
        }
    }

    static_cast<Box &>(p) = make_box(a, nd, u->size, so);
    bool empty;
    if ((rc = check_reach("b2_iso_forward", p, nd, a->radius, empty))) return rc;
    if (empty) {
        u->written = false;       // nothing ran, and u's host -> device copy may still be deferred (maybe_stream)
        return B2_OK;
    }
    for (int d = 3 - nd; d < 3; ++d) p.radius[d] = a->radius;
    p.u = (float *)u->d;
    p.damp = damp ? (const float *)damp->d : nullptr;
    p.param = param ? (const float *)param->d : nullptr;
    p.param_kind = a->param_kind;
    p.vp = a->vp;
    p.dt = a->dt;
    for (int d = 0; d < nd; ++d) {
        const int di = nd == 3 ? d : d + 1;
        if (!a->w[d]) { set_error("b2_iso_forward: weights for dim %d missing", d); return B2_ERR_INVALID; }
        for (int i = 0; i <= a->radius; ++i) p.w[di][i] = a->w[d][i];
    }
    p.ot4 = a->ot4 != 0;
    if (p.ot4 && (a->free_surface || a->grad)) {
        set_error("b2_iso_forward: OT4 is not combined with a free surface or the imaging condition in this version");
        return B2_ERR_INVALID;
    }
    p.defer_coef = maybe_stream || host_io;       // the arrays are not on the device yet
    if ((rc = iso_plan_init(p, a->kernel))) return rc;
    const bool damp_io = damp && (damp->owned || (host_io && a->damp->dmap && a->damp->data));
    const bool param_io = param && (param->owned || (host_io && a->param->dmap && a->param->data));
    const bool streamed = maybe_stream && streamed_wanted(a, p, *u, host_io);
    if ((maybe_stream || host_io) && !streamed) {
        // not streaming after all: the classic order — whole arrays in, tabulate, loop, whole arrays out
        DevArray *arrs[3] = {u, damp_io ? damp : nullptr, param_io ? param : nullptr};
        for (DevArray *x : arrs)
            if (x && (x->owned || host_io))
                if (cudaMemcpyAsync(x->d, x->h, x->nbytes, cudaMemcpyHostToDevice, stream()) != cudaSuccess) {
                    set_error("b2_iso_forward: host -> device copy failed");
                    return B2_ERR_MEMORY;
                }
        p.defer_coef = false;
        if (p.use_tma && (rc = iso_coef_tabulate_all(p))) return rc;
    }
    // Born: a second plan for the linearised field (same geometry and coefficient tables, own tensor maps)
    IsoPlan pU = p;
    if (born) {
        pU.u = (float *)bornU->d;
        if ((rc = iso_plan_init(pU, a->kernel))) return rc;
    }
    if (a->free_surface && p.o[2] != so) {
        set_error("b2_iso_forward: a free surface needs the vertical iteration to start at 0");
        return B2_ERR_INVALID;
    }

    FieldGeom g = field_geom(p, nd, a->halo);
    const float dt2 = a->dt * a->dt;
    const float scalar_scale = dt2 * a->vp * a->vp;
    const int T = p.tsize;
    const bool timing = a->timers != nullptr;
    StepEvents &se = g_step_events;
    se.used = 0;
    const int nsteps = a->time_M - a->time_m + 1;
    // The reference reports section0 (stencil), section1 (injection), section2 (interpolation)
    // (devito/operator/profiling.py:40-123). Four event records per step would cost ~1 % of a step, so the split is
    // SAMPLED: every 16th step is bracketed (every step with B2_PROFILING=advanced), the sparse sections are
    // scaled up, and section0 is the loop's total minus them.
    static const bool adv = getenv("B2_PROFILING") && std::string(getenv("B2_PROFILING")) == "advanced";
    const int sample_stride = adv ? 1 : 16;
    static cudaEvent_t ev_tot[2] = {nullptr, nullptr}, ev_prof[2] = {nullptr, nullptr};
    if (!ev_tot[0]) {
        for (auto &e : ev_tot) cudaEventCreate(&e);
        for (auto &e : ev_prof) cudaEventCreate(&e);
    }
    int step_index = 0, nsampled = 0;
    if (timing) cudaEventRecord(ev_tot[0], stream());

    const bool p2p = a->halo && halo_p2p_active(a->halo, p.u);
    // halo step fused into the sweep kernel (peer stores + flag acquire inside k_iso_tma)
    // (free-surface rows are redone after the sweep and Born steps a second field: those use the copy path)
    const bool fused = p2p && halo_fused_ok(a->halo, p) && !a->free_surface && !born;
    IsoFuse fz;
    if (fused && (rc = halo_fuse_desc(a->halo, p, fz))) return rc;
    if (a->halo && nd == 3 && (a->x_m != 0 || a->x_M != p.a[0] - 2 * so - 1)) {
        set_error("b2_iso_forward: the decomposed dimension must be iterated over the whole slab "
                  "(x_m=%d, x_M=%d, %d owned planes)", a->x_m, a->x_M, p.a[0] - 2 * so);
        return B2_ERR_INVALID;
    }
    if (a->halo) a->halo->reset_primed();           // first step of a call exchanges through NCCL
    const int dir = a->adjoint ? -1 : 1;
    // profile: [0] staging issued before the loop, [1] the loop (device clock)
    cudaEventRecord(ev_prof[0], stream());
    if (streamed) {
        if ((rc = iso_forward_streamed(a, p, g, *u, damp, param, src, rec, scalar_scale, dt2, damp_io, param_io)))
            return rc;
        u->written = false;                       // the loop has brought u home
        g_last_profile[4] = 1.0;
    }
    bool two_level = false;
    if (!streamed && (rc = two_level_wanted(a, p, *u, src, g, streamed, host_io, two_level))) return rc;
    if (two_level && (rc = iso_forward_two_level(a, p, g, src, rec, scalar_scale, dt2, timing ? &se : nullptr,
                                                 std::max(sample_stride / 2, 1), nsampled)))
        return rc;
    if (!streamed && !two_level)
    for (int time = a->adjoint ? a->time_M : a->time_m; a->adjoint ? time >= a->time_m : time <= a->time_M;
         time += dir) {
        const int t0 = slot(time, T);
        const int t1 = slot(time + dir, T);     // written
        const int t2 = slot(time - dir, T);     // the other time level read
        const bool per_step_events = timing && (step_index++ % sample_stride == 0) && se.used + 4 <= 16384;
        if (per_step_events) { se.next(); ++nsampled; }
        float *f1 = p.u + (size_t)t1 * p.slot_elems;
        if (!a->halo) {
            if ((rc = iso_sweep_inject(p, g, src, time, dir, a->free_surface, scalar_scale, dt2,
                                       per_step_events ? &se : nullptr)))
                return rc;
        } else {
            if (fused) {
                if ((rc = halo_step_iso_fused(a->halo, p, t0, t2, t1))) return rc;
                // the injection below must reach the copies of my boundary planes in the neighbours' halos
                g.peer_lo = fz.peer_lo; g.peer_hi = fz.peer_hi;
                g.off_lo = (long long)t1 * fz.slot_lo + (long long)(p.o[0] + fz.n_lo) * p.sx;
                g.off_hi = (long long)t1 * fz.slot_hi + (long long)(p.o[0] - p.n[0]) * p.sx;
                g.nown = p.n[0]; g.pw = p.radius[0];
            } else if ((rc = halo_exchange_and_step_iso(a->halo, p, t0, t2, t1))) {
                return rc;
            }
            if (a->free_surface && (rc = iso_fs_fix(p, t0, t2, t1, 0, p.n[0]))) return rc;
            if (per_step_events) se.next();
            if ((rc = launch_inject(src, g, f1, nullptr, time, p.param_kind, p.param, scalar_scale, dt2)))
                return rc;
        }
        if (fused) {
            // the sweep stored the boundary planes, the injection patched them: release the flags
            if ((rc = halo_fused_signal(a->halo, p.u))) return rc;
            if (a->rec_toff && rec.present && (rc = halo_p2p_wait(a->halo))) return rc;
        } else if (p2p) {
            // boundary planes of u[t1] are final: store them into the neighbours' halos, signal
            if ((rc = halo_p2p_publish(a->halo, p.u, nullptr, p.slot_elems, t1, (size_t)p.sx, p.o[0], p.n[0],
                                       halo_width_iso(p))))
                return rc;
            // receivers that sample the just-written time level may touch halo cells: those
            // arrive with the neighbours' stores of this same step
            if (a->rec_toff && rec.present && (rc = halo_p2p_wait(a->halo))) return rc;
        }
        if (born) {
            // eqn2 of the reference's Born operator comes after the source injection into u[t+1]
            if (a->halo) {
                if ((rc = halo_exchange_and_step_iso(a->halo, pU, t0, t2, t1))) return rc;
            } else if ((rc = iso_step(pU, t0, t2, t1, 0, pU.n[0]))) {
                return rc;
            }
            if ((rc = iso_born_source(p, t0, t2, t1, pU.u + (size_t)t1 * p.slot_elems, (const float *)borndm->d,
                                      (long long)borndm->size[1] * borndm->size[2], borndm->size[2],
                                      a->x_m + dmh, a->y_m + dmh, a->z_m + dmh)))
                return rc;
            // the linearised field's boundary planes are final: publish them like u's
            if (a->halo && halo_p2p_active(a->halo, pU.u) &&
                (rc = halo_p2p_publish(a->halo, pU.u, nullptr, pU.slot_elems, t1, (size_t)pU.sx, pU.o[0], pU.n[0],
                                       halo_width_iso(pU))))
                return rc;
        }
        if (a->snap && time % a->snap_factor == 0) {
            // internal dims: a 2-D grid is (1, x, y), its snapshots (nsnaps, x, y)
            const long long ssy = snap->size[nd];
            const long long ssx = nd == 3 ? (long long)snap->size[2] * snap->size[3] : 0;
            const size_t one = (size_t)(nd == 3 ? snap->size[1] : 1) * snap->size[nd - 1] * snap->size[nd];
            float *dst = nullptr;
            if (streamer.active) {
                if ((rc = streamer.acquire(&dst))) return rc;
            } else {
                dst = (float *)snap->d + (size_t)(time / a->snap_factor) * one;
            }
            const int d0 = nd == 3 ? a->x_m + snap_h : 0;
            const int d1 = (nd == 3 ? a->y_m : a->x_m) + snap_h;
            const int d2 = (nd == 3 ? a->z_m : a->y_m) + snap_h;
            if ((rc = iso_snapshot(p, a->snap_toff ? t1 : t0, dst, ssx, ssy, d0, d1, d2))) return rc;
            if (streamer.active) {
                const int dd[3] = {d0, d1, d2};
                if ((rc = streamer.release(time / a->snap_factor, &snap->size[1], dd, p.n))) return rc;
            }
        }
        if (per_step_events) se.next();
        if (a->halo && !p2p && a->rec_toff && rec.present) {
            // NCCL path: receivers that sample the level just written may reach into the halo, which is only
            // exchanged at the start of the next step -- exchange it now (the peer paths wait on the flags instead)
            if ((rc = halo_exchange_slot(a->halo, born ? pU : p, t1))) return rc;
        }
        const float *fr = (born ? pU.u : p.u) + (size_t)(a->rec_toff ? t1 : t0) * p.slot_elems;
        if ((rc = launch_interp(rec, g, fr, nullptr, time))) return rc;
        if (grad) {
            if (time < 0 || time >= usave->size[0]) {
                set_error("b2_iso_forward: time=%d outside the saved wavefield (nt=%d)", time, usave->size[0]);
                return B2_ERR_INVALID;
            }
            if ((rc = launch_imaging(p, *grad, gh, (const float *)usave->d + (size_t)time * p.slot_elems, p.u, nullptr,
                                     nullptr, t0, t1, t2)))
                return rc;
        }
        if (per_step_events) se.next();
        if (a->errctl && errctl_due(time, a->time_m, a->adjoint ? a->time_m : a->time_M) &&
            (rc = check_finite(f1, p.slot_elems, "u", time)))
            return rc;
    }
    if (a->halo && (rc = halo_p2p_drain(a->halo))) return rc;
    if (timing) cudaEventRecord(ev_tot[1], stream());
    cudaEventRecord(ev_prof[1], stream());
    if (streamed && a->errctl &&
        (rc = check_finite(p.u + (size_t)slot(a->time_M + 1, T) * p.slot_elems, p.slot_elems, "u", a->time_M)))
        return rc;
    if ((rc = sync_call("b2_iso_forward"))) return rc;
    {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, ev_prof[0], ev_prof[1]) == cudaSuccess) g_last_profile[1] = ms;
        g_last_profile[0] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - call_t0).count()
                            - g_last_profile[1];          // everything before the loop (staging in), host clock
    }
    if (timing) {
        float tot = 0.f;
        cudaEventElapsedTime(&tot, ev_tot[0], ev_tot[1]);
        double s1 = 0, s2 = 0;
        for (size_t i = 0; i + 3 < se.used; i += 4) {
            float ms;
            if (cudaEventElapsedTime(&ms, se.ev[i + 1], se.ev[i + 2]) == cudaSuccess) s1 += ms;
            if (cudaEventElapsedTime(&ms, se.ev[i + 2], se.ev[i + 3]) == cudaSuccess) s2 += ms;
        }
        if (nsampled > 0) {
            const double up = (double)nsteps / nsampled;
            s1 *= up;
            s2 *= up;
        }
        if (s1 + s2 > tot) { const double f = tot / (s1 + s2 + 1e-30); s1 *= f * 0.5; s2 *= f * 0.5; }
        a->timers->section0 += (tot - s1 - s2) * 1e-3;
        a->timers->section1 += s1 * 1e-3;
        a->timers->section2 += s2 * 1e-3;
    }
    return B2_OK;
}

extern "C" int b2_iso_forward(const struct b2_iso_args *a) {
    if (!a || !a->u) { set_error("b2_iso_forward: NULL args"); return B2_ERR_INVALID; }
    if (a->ndim != 2 && a->ndim != 3) { set_error("b2_iso_forward: ndim must be 2 or 3"); return B2_ERR_INVALID; }
    if (a->radius < 1 || a->radius > B2_MAX_RADIUS || a->radius > a->space_order) {
        set_error("b2_iso_forward: unsupported radius %d (space_order %d)", a->radius, a->space_order);
        return B2_ERR_INVALID;
    }
    if (a->time_M < a->time_m) return B2_OK;
    std::lock_guard<std::mutex> api_lock(api_mutex());
    if (int rc0 = use_device(a->deviceid)) return rc0;
    note_sweep_kernel("");
    for (double &v : g_last_profile) v = 0.0;
    const auto call_t0 = std::chrono::steady_clock::now();
    Staging st;
    SnapStreamer streamer;
    int rc = iso_forward_body(a, st, streamer, call_t0);
    // profile: [2] the write-back (copies to the host, snapshot drain, release), [3] the whole call; host clock
    const auto d2h_t0 = std::chrono::steady_clock::now();
    rc = st.finish(rc);
    const int rs = streamer.end();
    const auto t1 = std::chrono::steady_clock::now();
    g_last_profile[2] = std::chrono::duration<double, std::milli>(t1 - d2h_t0).count();
    g_last_profile[3] = std::chrono::duration<double, std::milli>(t1 - call_t0).count();
    return rc ? rc : rs;
}

// ---------------------------------------------------------------------------------------------------------
// b2_iso_gradient_revolve: the Gradient operator with the forward wavefield recomputed from checkpoints
// (binomial checkpointing, Griewank & Walther, ACM TOMS 26(1) 2000) instead of read from a saved (nt, x, y, z)
// array. The forward field lives in u's 3 slots; a checkpoint holds the two levels a step reads, u[t] and u[t-1],
// as whole allocated slots (halo included: sinc injection writes there). The actions come from the caller's
// schedule; both plans are built once and every action runs on the library stream.
// ---------------------------------------------------------------------------------------------------------
static bool same_array(const b2_dataobj *x, const b2_dataobj *y) {
    if (x == y) return true;
    return x && y && (x->data || x->dmap) && x->data == y->data && x->dmap == y->dmap && x->nbytes == y->nbytes;
}

extern "C" int b2_revolve_check(const int *actions, int nactions, int ncheckpoints, int fwd_time_m, int fwd_time_M,
                                int grad_time_m, int grad_time_M) {
    const char *who = "b2_revolve_check";
    if (ncheckpoints < 1) { set_error("%s: %d checkpoints (at least 1)", who, ncheckpoints); return B2_ERR_INVALID; }
    if (nactions < 0 || (nactions > 0 && !actions)) { set_error("%s: no action list", who); return B2_ERR_INVALID; }
    std::vector<int> shot((size_t)ncheckpoints);
    std::vector<char> full((size_t)ncheckpoints, 0);
    int cur = fwd_time_m;                 // forward time of the state in u: levels cur and cur-1 are live
    int next = grad_time_M;               // the adjoint time the next reverse must name
    for (int i = 0; i < nactions; ++i) {
        const int kind = actions[3 * i], x = actions[3 * i + 1], y = actions[3 * i + 2];
        switch (kind) {
            case B2_REVOLVE_ADVANCE:
                if (x != cur || y <= x || y - 1 > fwd_time_M) {
                    set_error("%s: action %d advance(%d, %d): the forward state is at time %d, steps run up to "
                              "time_M=%d", who, i, x, y, cur, fwd_time_M);
                    return B2_ERR_INVALID;
                }
                cur = y;
                break;
            case B2_REVOLVE_TAKESHOT:
            case B2_REVOLVE_RESTORE:
                if (x < 0 || x >= ncheckpoints) {
                    set_error("%s: action %d names checkpoint %d of %d", who, i, x, ncheckpoints);
                    return B2_ERR_INVALID;
                }
                if (kind == B2_REVOLVE_TAKESHOT) {
                    if (y != cur) {
                        set_error("%s: action %d takeshot(%d, %d): the forward state is at time %d", who, i, x, y, cur);
                        return B2_ERR_INVALID;
                    }
                    shot[x] = cur;
                    full[x] = 1;
                } else {
                    if (!full[x]) { set_error("%s: action %d restores the empty checkpoint %d", who, i, x); return B2_ERR_INVALID; }
                    cur = shot[x];
                }
                break;
            case B2_REVOLVE_REVERSE:
                if (x != next || x < grad_time_m) {
                    set_error("%s: action %d reverse(%d): the adjoint steps run once each from %d down to %d, the "
                              "next is %d", who, i, x, grad_time_M, grad_time_m, next);
                    return B2_ERR_INVALID;
                }
                if (x != cur && x != cur - 1) {
                    set_error("%s: action %d reverse(%d) needs u[%d], the forward state holds levels %d and %d", who, i,
                              x, x, cur - 1, cur);
                    return B2_ERR_INVALID;
                }
                --next;
                break;
            default:
                set_error("%s: action %d has the unknown kind %d", who, i, kind);
                return B2_ERR_INVALID;
        }
    }
    if (next >= grad_time_m) {
        set_error("%s: the actions reverse down to time %d, not to time_m=%d", who, next + 1, grad_time_m);
        return B2_ERR_INVALID;
    }
    return B2_OK;
}

// What the two argument blocks may be: everything the two loops share (medium, box, time step) is the same.
static int revolve_args_check(const b2_iso_args *f, const b2_iso_args *g) {
    const char *who = "b2_iso_gradient_revolve";
    if (!f || !g || !f->u || !g->u) { set_error("%s: NULL args", who); return B2_ERR_INVALID; }
    const b2_iso_args *both[2] = {f, g};
    for (const b2_iso_args *a : both) {
        const char *which = a == f ? "fwd" : "grad";
        if (a->ndim != 3) { set_error("%s: %s: the imaging condition is 3-D only", who, which); return B2_ERR_INVALID; }
        if (a->radius < 1 || a->radius > B2_MAX_RADIUS || a->radius > a->space_order) {
            set_error("%s: %s: unsupported radius %d (space_order %d)", who, which, a->radius, a->space_order);
            return B2_ERR_INVALID;
        }
        if (a->halo || a->ot4 || a->free_surface || a->born_U || a->born_dm || a->snap || a->host_io || a->rec) {
            set_error("%s: %s: not combined with halo exchange, OT4, a free surface, Born modelling, snapshots, "
                      "host_io or receivers", who, which);
            return B2_ERR_INVALID;
        }
    }
    if (f->adjoint || f->grad || f->usave) {
        set_error("%s: fwd must describe the forward operator (no adjoint, grad or usave)", who);
        return B2_ERR_INVALID;
    }
    if (!g->adjoint || !g->grad) { set_error("%s: grad must describe the Gradient operator (adjoint, grad)", who); return B2_ERR_INVALID; }
    if (!same_array(g->usave, f->u)) {
        set_error("%s: grad's usave must be fwd's u (the forward field is recomputed into it)", who);
        return B2_ERR_INVALID;
    }
    if (same_array(g->u, f->u)) { set_error("%s: the adjoint field must not be the forward field", who); return B2_ERR_INVALID; }
    if (!f->u->size || f->u->size[0] != 3) {
        set_error("%s: fwd's u must be buffered with 3 time slots", who);
        return B2_ERR_INVALID;
    }
    const int fb[6] = {f->x_m, f->x_M, f->y_m, f->y_M, f->z_m, f->z_M}, gb[6] = {g->x_m, g->x_M, g->y_m, g->y_M, g->z_m, g->z_M};
    // the two sweeps share the update-coefficient tables: one medium, one box, one time step
    if (f->space_order != g->space_order || f->radius != g->radius || f->dt != g->dt || f->vp != g->vp ||
        f->param_kind != g->param_kind || !same_array(f->damp, g->damp) || !same_array(f->param, g->param) ||
        memcmp(fb, gb, sizeof fb)) {
        set_error("%s: fwd and grad must share space order, radius, dt, vp, damp, the parameter array and the "
                  "iteration box", who);
        return B2_ERR_INVALID;
    }
    return B2_OK;
}

static int iso_revolve_body(const b2_iso_args *f, const b2_iso_args *ga, const int *act, int nact, int nck,
                            Staging &st) {
    const char *who = "b2_iso_gradient_revolve";
    const int so = f->space_order;
    int rc;
    DevArray *u, *v, *damp = nullptr, *param = nullptr, *grad;
    SparseDev src, none, asrc, anone;
    if ((rc = st.array(f->u, 4, true, u))) return rc;
    if ((rc = st.array(ga->u, 4, true, v))) return rc;
    if (f->damp && (rc = st.array(f->damp, 3, false, damp))) return rc;
    if (f->param_kind != B2_PARAM_SCALAR) {
        if (!f->param) { set_error("%s: param array missing", who); return B2_ERR_INVALID; }
        if ((rc = st.array(f->param, 3, false, param))) return rc;
    }
    if ((rc = sparse_stage_pair(who, st, f->src, nullptr, 3, so, src, none))) return rc;
    if ((rc = sparse_stage_pair(who, st, ga->src, nullptr, 3, so, asrc, anone))) return rc;
    if ((rc = st.array(ga->grad, 3, true, grad))) return rc;
    for (int d = 1; d < 4; ++d)
        if (v->size[d] != u->size[d]) { set_error("%s: the adjoint field must have u's space layout", who); return B2_ERR_INVALID; }
    const int gh = grid_halo(who, "grad", ga->grad, *grad, 0, *u, 3, so);
    if (gh < 0) return B2_ERR_INVALID;

    IsoPlan pf, pa;
    const b2_iso_args *args[2] = {f, ga};
    IsoPlan *plans[2] = {&pf, &pa};
    DevArray *fields[2] = {u, v};
    for (int i = 0; i < 2; ++i) {
        IsoPlan &p = *plans[i];
        const b2_iso_args *a = args[i];
        static_cast<Box &>(p) = make_box(a, 3, fields[i]->size, so);
        bool empty;
        if ((rc = check_reach(who, p, 3, a->radius, empty))) return rc;
        if (empty) return B2_OK;
        for (int d = 0; d < 3; ++d) {
            p.radius[d] = a->radius;
            if (!a->w[d]) { set_error("%s: weights for dim %d missing", who, d); return B2_ERR_INVALID; }
            for (int k = 0; k <= a->radius; ++k) p.w[d][k] = a->w[d][k];
        }
        p.u = (float *)fields[i]->d;
        p.damp = damp ? (const float *)damp->d : nullptr;
        p.param = param ? (const float *)param->d : nullptr;
        p.param_kind = a->param_kind;
        p.vp = a->vp;
        p.dt = a->dt;
        // the second plan re-tabulates the shared coefficient tables with the same medium, box and dt
        if ((rc = iso_plan_init(p, a->kernel))) return rc;
    }

    // the checkpoints, once per call: two whole slots each
    const size_t slot_bytes = pf.slot_elems * sizeof(float);
    std::vector<float *> ck((size_t)nck);
    for (int k = 0; k < nck; ++k) {
        DevArray *x;
        if ((rc = st.scratch(2 * slot_bytes, x))) return rc;
        ck[k] = (float *)x->d;
    }
    auto level = [&](int time) { return pf.u + (size_t)slot(time, 3) * pf.slot_elems; };
    const FieldGeom gf = field_geom(pf, 3), gg = field_geom(pa, 3);
    const float dt2 = f->dt * f->dt, scalar_scale = dt2 * f->vp * f->vp;
    bool two_level = false;
    if ((rc = two_level_wanted(f, pf, *u, src, gf, false, false, two_level))) return rc;
    // the sweeps that ran, in order of first use, space-separated: forward ones, then after ';' the adjoint one
    std::string fwd_k, adj_k;
    auto add_kernel = [](std::string &s) {
        const std::string k = b2_last_sweep_kernel();
        if (k.empty() || (" " + s + " ").find(" " + k + " ") != std::string::npos) return;
        s += (s.empty() ? "" : " ") + k;
    };
    std::vector<int> shot((size_t)nck);
    int cur = f->time_m;
    // errctl on the forward steps keeps b2_iso_forward's cadence: every 100th forward time counted from time_m, and
    // the last forward time the schedule reaches (a recomputed time is checked again)
    int fwd_last = f->time_m;
    for (int i = 0; i < nact; ++i)
        if (act[3 * i] == B2_REVOLVE_ADVANCE) fwd_last = std::max(fwd_last, act[3 * i + 2] - 1);
    // the level each slot of u holds (INT_MIN: none known): a restore copies only the levels not already in place,
    // e.g. the ones the last advance left behind
    int held[3] = {INT_MIN, INT_MIN, INT_MIN};
    held[slot(cur, 3)] = cur;
    held[slot(cur - 1, 3)] = cur - 1;
    if ((rc = loop_timer_start(ga->timers))) return rc;
    for (int i = 0; i < nact; ++i) {
        const int kind = act[3 * i], x = act[3 * i + 1], y = act[3 * i + 2];
        if (kind == B2_REVOLVE_ADVANCE) {
            if (two_level && y - x >= 2) {
                b2_iso_args r = *f;
                r.time_m = x;
                r.time_M = y - 1;
                int nsampled = 0;
                if ((rc = iso_forward_two_level(&r, pf, gf, src, none, scalar_scale, dt2, nullptr, 1, nsampled)))
                    return rc;
                held[0] = held[1] = held[2] = INT_MIN;
                held[slot(y, 3)] = y;
                held[slot(y - 1, 3)] = y - 1;
            } else {
                for (int time = x; time < y; ++time) {
                    if ((rc = iso_sweep_inject(pf, gf, src, time, 1, false, scalar_scale, dt2, nullptr))) return rc;
                    held[slot(time + 1, 3)] = time + 1;
                    if (f->errctl && errctl_due(time, f->time_m, fwd_last) &&
                        (rc = check_finite(level(time + 1), pf.slot_elems, "u", time)))
                        return rc;
                }
            }
            add_kernel(fwd_k);
            cur = y;
        } else if (kind == B2_REVOLVE_TAKESHOT || kind == B2_REVOLVE_RESTORE) {
            const bool take = kind == B2_REVOLVE_TAKESHOT;
            if (!take) cur = shot[x];
            for (int j = 0; j < 2; ++j) {
                float *c = ck[x] + (size_t)j * pf.slot_elems, *l = level(cur - j);
                if (!take && held[slot(cur - j, 3)] == cur - j) continue;
                B2_CUDA(cudaMemcpyAsync(take ? c : l, take ? l : c, slot_bytes, cudaMemcpyDeviceToDevice, stream()),
                        B2_ERR_MEMORY);
                held[slot(cur - j, 3)] = cur - j;
            }
            if (take) shot[x] = cur;
        } else {
            // one adjoint step, then grad -= u[x] * v.dt2 with u[x] live in its slot
            const int T = pa.tsize;
            if ((rc = iso_sweep_inject(pa, gg, asrc, x, -1, false, scalar_scale, dt2, nullptr))) return rc;
            if ((rc = launch_imaging(pa, *grad, gh, level(x), pa.u, nullptr, nullptr, slot(x, T), slot(x - 1, T),
                                     slot(x + 1, T))))
                return rc;
            add_kernel(adj_k);
            if (ga->errctl && errctl_due(x, ga->time_m, ga->time_m) &&
                (rc = check_finite(pa.u + (size_t)slot(x - 1, T) * pa.slot_elems, pa.slot_elems, "v", x)))
                return rc;
        }
    }
    note_sweep_kernel("%s;%s", fwd_k.c_str(), adj_k.c_str());
    return loop_finish(who, ga->timers);
}

extern "C" int b2_iso_gradient_revolve(const struct b2_iso_args *fwd, const struct b2_iso_args *grad,
                                       const int *actions, int nactions, int ncheckpoints) {
    int rc;
    if ((rc = revolve_args_check(fwd, grad))) return rc;
    if ((rc = b2_revolve_check(actions, nactions, ncheckpoints, fwd->time_m, fwd->time_M, grad->time_m, grad->time_M)))
        return rc;
    if (grad->time_M < grad->time_m) return B2_OK;
    std::lock_guard<std::mutex> api_lock(api_mutex());
    if ((rc = use_device(fwd->deviceid))) return rc;
    note_sweep_kernel("");
    Staging st;
    rc = iso_revolve_body(fwd, grad, actions, nactions, ncheckpoints, st);
    return st.finish(rc);
}
