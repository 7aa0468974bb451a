// Sparse source injection and receiver interpolation on the device.
//
// Reference semantics (devito/operations/interpolators.py:510-624 `_interpolate`/`_inject`,
// guards :284-311; generated loops printed by the reference for Forward):
//   for p in [p_m, p_M], rd_x, rd_y, rd_z in [-r+1, r]:
//       cell_d = gp[p][d] + rd_d;   valid iff  d_m - r <= cell_d <= d_M + r
//       inject:      u[t+1][cell + so] += wx[p][rd_x+r-1] wy[..] wz[..] * src[time][p] * dt^2/m(cell)
//       interpolate: rec[time][p]      = sum  wx wy wz * u[t(+1)][cell + so]
// Injection uses atomics (reference: `#pragma omp atomic update` / `acc atomic update`,
// devito/passes/iet/languages/openacc.py:79-80). One warp handles one point; lanes stride over
// the (2r)^ndim support cells; interpolation reduces with warp shuffles.
#include "b2_sparse.cuh"
#include "b2_halo.cuh"
#include <climits>

namespace b2 {

struct SparseK {
    const float *__restrict__ data;   // (nt, npoint_total)
    const int *__restrict__ gp;       // (npoint_total, ndim)
    const float *__restrict__ w0;     // (npoint_total, 2r) for internal dim 0 (may be null: 2-D)
    const float *__restrict__ w1;
    const float *__restrict__ w2;
    int npoint_total;
    int p_m, p_cnt;
    int r, ndim;
    long long sx, sy;
    int so;
    int lo0, lo1, lo2, hi0, hi1, hi2;
    int ext_lo0, ext_hi0;     // how far beyond [lo0, hi0] the support may reach (r, or 0 next to a neighbour)
    int ext_lo1, ext_hi1;     // same for dim 1 (r, or 0 at an interior cut of a y-skewed streamed sweep)
    // fused halo step (FieldGeom): mirror injected boundary cells into the neighbours' halos
    float *peer_lo, *peer_hi;
    long long off_lo, off_hi;
    int nown, pw;
};

__device__ __forceinline__ bool sparse_cell(const SparseK &k, int p, int c, long long &idx, float &wgt,
                                            int &c0o, int &c1o, int &c2o) {
    const int n = 2 * k.r;
    int r2 = c % n;
    int t = c / n;
    int r1 = t % n;
    int r0 = t / n;                       // 0 for 2-D
    const int *g = k.gp + (long long)p * k.ndim;
    int c0, c1, c2;
    float w;
    if (k.ndim == 3) {
        c0 = g[0] + r0 - k.r + 1;
        c1 = g[1] + r1 - k.r + 1;
        c2 = g[2] + r2 - k.r + 1;
        if (c0 < k.lo0 - k.ext_lo0 || c0 > k.hi0 + k.ext_hi0) return false;
        w = k.w0[(long long)p * n + r0] * k.w1[(long long)p * n + r1] * k.w2[(long long)p * n + r2];
    } else {
        c0 = 0;
        c1 = g[0] + r1 - k.r + 1;
        c2 = g[1] + r2 - k.r + 1;
        w = k.w1[(long long)p * n + r1] * k.w2[(long long)p * n + r2];
    }
    if (c1 < k.lo1 - k.ext_lo1 || c1 > k.hi1 + k.ext_hi1) return false;
    if (c2 < k.lo2 - k.r || c2 > k.hi2 + k.r) return false;
    const int s0 = (k.ndim == 3) ? k.so : 0;
    idx = (long long)(c0 + s0) * k.sx + (long long)(c1 + k.so) * k.sy + (c2 + k.so);
    wgt = w;
    c0o = c0; c1o = c1; c2o = c2;
    return true;
}

__global__ void __launch_bounds__(128)
k_inject(SparseK k, float *__restrict__ f0, float *__restrict__ f1, int time, int param_kind,
         const float *__restrict__ param, float scalar_scale, float dt2) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= k.p_cnt) return;
    const int p = k.p_m + warp;
    const int n = 2 * k.r;
    const int ncell = (k.ndim == 3) ? n * n * n : n * n;
    const float sv = k.data[(long long)time * k.npoint_total + p];
    for (int c = lane; c < ncell; c += 32) {
        long long idx;
        float w;
        int c0, c1, c2;
        if (!sparse_cell(k, p, c, idx, w, c0, c1, c2)) continue;
        float scale = scalar_scale;
        if (param_kind == B2_PARAM_VP) {
            const float v = param[idx];
            scale = dt2 * v * v;
        } else if (param_kind == B2_PARAM_M) {
            scale = dt2 / param[idx];
        } else if (param_kind == B2_SCALE_TABLE) {
            scale = param[idx];
        }
        const float val = w * sv * scale;
        atomicAdd(f0 + idx, val);
        if (f1) atomicAdd(f1 + idx, val);
        if (k.pw > 0) {
            // idx = (c0 + so) * sx + row; the neighbour's copy of my plane c0 sits at off + c0 * sx + row
            const long long row = idx - (long long)(c0 + k.so) * k.sx;
            if (k.peer_lo && c0 < k.pw) atomicAdd_system(k.peer_lo + (k.off_lo + (long long)c0 * k.sx + row), val);
            if (k.peer_hi && c0 >= k.nown - k.pw) atomicAdd_system(k.peer_hi + (k.off_hi + (long long)c0 * k.sx + row), val);
        }
    }
}

__global__ void __launch_bounds__(128)
k_interp(SparseK k, const float *__restrict__ f0, const float *__restrict__ f1,
         float *__restrict__ out, int time, int accumulate) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= k.p_cnt) return;
    const int p = k.p_m + warp;
    const int n = 2 * k.r;
    const int ncell = (k.ndim == 3) ? n * n * n : n * n;
    float sum = 0.f;
    for (int c = lane; c < ncell; c += 32) {
        long long idx;
        float w;
        int c0, c1, c2;
        if (!sparse_cell(k, p, c, idx, w, c0, c1, c2)) continue;
        float v = f0[idx];
        if (f1) v += f1[idx];
        sum = fmaf(w, v, sum);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if (lane == 0) {
        // streamed time loop: the support of a point is sampled x-range by x-range (partial sums)
        if (accumulate) { if (sum != 0.f) atomicAdd(out + (long long)time * k.npoint_total + p, sum); }
        else out[(long long)time * k.npoint_total + p] = sum;
    }
}

static SparseK make_k(const SparseDev &s, const FieldGeom &g, bool injecting) {
    SparseK k;
    k.ext_lo0 = ((injecting || g.restrict_x) && g.nb_lo) ? 0 : s.r;
    k.ext_hi0 = ((injecting || g.restrict_x) && g.nb_hi) ? 0 : s.r;
    k.ext_lo1 = (g.restrict_y && g.cut_lo1) ? 0 : s.r;
    k.ext_hi1 = (g.restrict_y && g.cut_hi1) ? 0 : s.r;
    k.peer_lo = injecting ? g.peer_lo : nullptr;
    k.peer_hi = injecting ? g.peer_hi : nullptr;
    k.off_lo = g.off_lo; k.off_hi = g.off_hi;
    k.nown = g.nown;
    k.pw = injecting && s.ndim == 3 && (g.peer_lo || g.peer_hi) ? g.pw : 0;
    k.data = (const float *)s.data->d;
    k.gp = (const int *)s.gp->d;
    if (s.ndim == 3) {
        k.w0 = (const float *)s.w[0]->d;
        k.w1 = (const float *)s.w[1]->d;
        k.w2 = (const float *)s.w[2]->d;
    } else {
        k.w0 = nullptr;
        k.w1 = (const float *)s.w[0]->d;
        k.w2 = (const float *)s.w[1]->d;
    }
    k.npoint_total = s.npoint_total;
    k.p_m = s.p_m;
    k.p_cnt = s.p_M - s.p_m + 1;
    k.r = s.r;
    k.ndim = s.ndim;
    k.sx = g.sx;
    k.sy = g.sy;
    k.so = g.so;
    if (s.ndim == 3) {
        k.lo0 = g.lo[0]; k.lo1 = g.lo[1]; k.lo2 = g.lo[2];
        k.hi0 = g.hi[0]; k.hi1 = g.hi[1]; k.hi2 = g.hi[2];
    } else {
        k.lo0 = 0; k.hi0 = 0;
        k.lo1 = g.lo[0]; k.lo2 = g.lo[1];
        k.hi1 = g.hi[0]; k.hi2 = g.hi[1];
    }
    return k;
}

int sparse_stage_in(Staging &st, const b2_sparse *s, int ndim, bool written, SparseDev &out) {
    out.present = false;
    if (!s) return B2_OK;
    if (s->p_M < s->p_m) return B2_OK;     // empty point range: nothing to do
    if (s->r < 1 || s->r > 8) { set_error("sparse: unsupported radius %d", s->r); return B2_ERR_INVALID; }
    if (!s->data || !s->data->size || !s->gp) { set_error("sparse: missing traces or base cells"); return B2_ERR_INVALID; }
    for (int d = 0; d < ndim; ++d)
        if (!s->w[d]) { set_error("sparse: missing weight table for dim %d", d); return B2_ERR_INVALID; }
    if (s->p_m < 0 || s->p_M >= s->data->size[1]) {
        set_error("sparse: point range [%d,%d] outside [0,%d)", s->p_m, s->p_M, s->data->size[1]);
        return B2_ERR_INVALID;
    }
    DevArray *x;
    int rc;
    if ((rc = st.array(s->data, 2, written, x))) return rc;
    out.data = x;
    if ((rc = st.array(s->gp, 2, false, x))) return rc;
    out.gp = x;
    for (int d = 0; d < ndim; ++d) {
        if ((rc = st.array(s->w[d], 2, false, x))) return rc;
        out.w[d] = x;
    }
    out.nt = out.data->size[0];
    out.npoint_total = out.data->size[1];
    out.p_m = s->p_m;
    out.p_M = s->p_M;
    out.r = s->r;
    out.ndim = ndim;
    out.present = true;
    return B2_OK;
}

int sparse_stage_pair(const char *who, Staging &st, const b2_sparse *src, const b2_sparse *rec, int ndim, int so,
                      SparseDev &src_out, SparseDev &rec_out) {
    int rc;
    if ((rc = sparse_stage_in(st, src, ndim, false, src_out))) return rc;
    if ((rc = sparse_stage_in(st, rec, ndim, true, rec_out))) return rc;
    const bool src_far = src_out.present && src_out.r > so, rec_far = rec_out.present && rec_out.r > so;
    if (src_far || rec_far) {
        set_error("%s: sparse radius %d exceeds the halo (space_order %d)", who, src_far ? src_out.r : rec_out.r, so);
        return B2_ERR_INVALID;
    }
    return B2_OK;
}

FieldGeom field_geom(const Box &b, int nd, const b2_halo_ctx *halo) {
    FieldGeom g;
    g.sx = b.sx;
    g.sy = b.sy;
    g.slot_elems = b.slot_elems;
    g.so = b.so;
    g.ndim = nd;
    for (int d = 0; d < nd; ++d) {
        const int di = 3 - nd + d;
        g.lo[d] = b.o[di] - b.so;
        g.hi[d] = g.lo[d] + b.n[di] - 1;
    }
    if (halo) { g.nb_lo = halo->rank > 0; g.nb_hi = halo->rank < halo->nranks - 1; }
    return g;
}

int launch_inject(const SparseDev &s, const FieldGeom &g, float *f0, float *f1, int time,
                  int param_kind, const float *param, float scalar_scale, float dt2) {
    if (!s.present) return B2_OK;
    if (time < 0 || time >= s.nt) return B2_OK;
    SparseK k = make_k(s, g, true);
    const int warps = k.p_cnt;
    const int blocks = (warps * 32 + 127) / 128;
    k_inject<<<blocks, 128, 0, stream()>>>(k, f0, f1, time, param_kind, param, scalar_scale, dt2);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

// The cells and values k_inject would add at `time`, as entries relative to the iteration origin (cells that
// k_inject skips, or a time outside the traces: x = INT_MIN, never matched); flag |= 1 when a cell lies outside
// the iteration box.
__global__ void __launch_bounds__(128)
k_inject_entries(SparseK k, int time, int valid_time, int param_kind, const float *__restrict__ param,
                 float scalar_scale, float dt2, IsoInj *__restrict__ out, int *__restrict__ flag) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= k.p_cnt) return;
    const int p = k.p_m + warp;
    const int n = 2 * k.r;
    const int ncell = n * n * n;
    for (int c = lane; c < ncell; c += 32) {
        IsoInj e = {INT_MIN, 0, 0, 0.f};
        long long idx;
        float w;
        int c0, c1, c2;
        if (sparse_cell(k, p, c, idx, w, c0, c1, c2)) {
            if (flag && (c0 < k.lo0 || c0 > k.hi0 || c1 < k.lo1 || c1 > k.hi1 || c2 < k.lo2 || c2 > k.hi2))
                atomicOr(flag, 1);
            if (valid_time) {
                const float sv = k.data[(long long)time * k.npoint_total + p];
                float scale = scalar_scale;
                if (param_kind == B2_PARAM_VP) {
                    const float v = param[idx];
                    scale = dt2 * v * v;
                } else if (param_kind == B2_PARAM_M) {
                    scale = dt2 / param[idx];
                }
                e = {c0 - k.lo0, c1 - k.lo1, c2 - k.lo2, w * sv * scale};
            }
        }
        if (out) out[(long long)warp * ncell + c] = e;
    }
}

int inject_entry_count(const SparseDev &s) {
    if (!s.present) return 0;
    const int n = 2 * s.r;
    return (s.p_M - s.p_m + 1) * n * n * n;
}

int launch_inject_entries(const SparseDev &s, const FieldGeom &g, int time, int param_kind, const float *param,
                          float scalar_scale, float dt2, IsoInj *out, int *outside_flag) {
    if (!s.present) return B2_OK;
    if (s.ndim != 3) { set_error("inject entries: 3-D only"); return B2_ERR_INVALID; }
    SparseK k = make_k(s, g, true);
    const int blocks = (k.p_cnt * 32 + 127) / 128;
    k_inject_entries<<<blocks, 128, 0, stream()>>>(k, time, time >= 0 && time < s.nt, param_kind, param,
                                                   scalar_scale, dt2, out, outside_flag);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

int launch_interp(const SparseDev &s, const FieldGeom &g, const float *f0, const float *f1, int time) {
    if (!s.present) return B2_OK;
    if (time < 0 || time >= s.nt) return B2_OK;
    SparseK k = make_k(s, g, false);
    const int warps = k.p_cnt;
    const int blocks = (warps * 32 + 127) / 128;
    k_interp<<<blocks, 128, 0, stream()>>>(k, f0, f1, (float *)s.data->d, time, (g.restrict_x || g.restrict_y) ? 1 : 0);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

}  // namespace b2
