// C-ABI entry point b2_system_forward: explicit time stepping of a first-order linear SYSTEM on a
// (staggered) grid — the generated `ForwardElastic` (examples/seismic/elastic/operators.py:26-65) and its
// relatives — as a tap-table executor: per time step a sequence of stages, each
//     out[t + out_tshift][p] = sum_k coef_k * C_{cfield_k}[p] * F_{field_k}[t + tshift_k][p + off_k].
// One thread per point (z fastest, x strided over gridDim.z); taps in the kernel parameter block. This is
// the generality path of §8f (staggered-grid systems), not a tuned sweep: the acoustic / TTI propagators
// keep their own kernels. tests/system_ref.py restates these semantics in float64.
#include "b2_common.cuh"
#include "b2_sparse.cuh"
#include <algorithm>
#include <vector>

using namespace b2;

namespace b2 {

struct SysK {
    float *__restrict__ out;
    const float *__restrict__ in[B2_SYS_MAX_FIELDS][2];     // [field][tshift]
    const float *__restrict__ cf[B2_SYS_MAX_COEFS];         // coefficient arrays (no halo)
    long long sx, sy;            // field strides
    long long csx, csy;          // coefficient-array strides
    int n0, n1, n2, o0, o1, o2;  // iteration box, array index of its first point
    int c0, c1, c2;              // index of the first iterated point in the coefficient arrays
    int ntaps;
    short fld[B2_SYS_MAX_TAPS], tsh[B2_SYS_MAX_TAPS], cfi[B2_SYS_MAX_TAPS];
    int delta[B2_SYS_MAX_TAPS];
    float coef[B2_SYS_MAX_TAPS];
};

__global__ void __launch_bounds__(256) k_system_stage(const __grid_constant__ SysK k) {
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (z >= k.n2 || y >= k.n1) return;
    for (int x = blockIdx.z; x < k.n0; x += gridDim.z) {
        const long long idx = (long long)(k.o0 + x) * k.sx + (long long)(k.o1 + y) * k.sy + (k.o2 + z);
        const long long cidx = (long long)(k.c0 + x) * k.csx + (long long)(k.c1 + y) * k.csy + (k.c2 + z);
        float acc = 0.f;
        int last = -2;
        float cval = 1.f;
        for (int i = 0; i < k.ntaps; ++i) {
            const int c = k.cfi[i];
            if (c != last) { cval = c >= 0 ? k.cf[c][cidx] : 1.f; last = c; }   // taps are sorted by cfield
            acc = fmaf(k.coef[i] * cval, k.in[k.fld[i]][k.tsh[i]][idx + k.delta[i]], acc);
        }
        k.out[idx] = acc;
    }
}

}  // namespace b2

static int system_forward_body(const b2_system_args *a, Staging &staging) {
    const int nd = a->ndim, h = a->halo;
    std::vector<DevArray *> F(a->nfields), C(a->ncoefs), injp(a->ninject, nullptr);
    std::vector<SparseDev> inj(a->ninject), itp(a->ninterp);
    int rc = B2_OK;
    for (int i = 0; i < a->nfields; ++i) {
        if ((rc = staging.array(a->fields[i], nd + 1, true, F[i]))) return rc;
        if (F[i]->size[0] < 1) { set_error("b2_system_forward: field %d has no time slot", i); return B2_ERR_INVALID; }
        for (int d = 1; d <= nd; ++d)
            if (F[i]->size[d] != F[0]->size[d]) { set_error("b2_system_forward: field %d has another shape", i); return B2_ERR_INVALID; }
    }
    const Box b = make_box(a, nd, F[0]->size, h);
    int calloc_[3] = {1, 1, 1};
    for (int i = 0; i < a->ncoefs; ++i) {
        if ((rc = staging.array(a->coefs[i], nd, false, C[i]))) return rc;
        for (int d = 0; d < nd; ++d) {
            const int di = 3 - nd + d;
            if (i == 0) calloc_[di] = C[i]->size[d];
            if (C[i]->size[d] != calloc_[di] || C[i]->size[d] != b.a[di] - 2 * h) {
                set_error("b2_system_forward: coefficient array %d does not have the grid's shape", i);
                return B2_ERR_INVALID;
            }
        }
    }
    for (int i = 0; i < a->ninject; ++i) {
        if ((rc = sparse_stage_in(staging, a->inject[i].s, nd, false, inj[i]))) return rc;
        if (a->inject[i].param_kind != B2_PARAM_SCALAR) {
            if (!a->inject[i].param) { set_error("b2_system_forward: injection %d lacks its parameter array", i); return B2_ERR_INVALID; }
            if ((rc = staging.array(a->inject[i].param, nd, false, injp[i]))) return rc;
            for (int d = 0; d < nd; ++d)
                if (injp[i]->size[d] != F[0]->size[d + 1]) {
                    set_error("b2_system_forward: the parameter array of injection %d does not have the fields' layout", i);
                    return B2_ERR_INVALID;
                }
        }
    }
    for (int i = 0; i < a->ninterp; ++i)
        if ((rc = sparse_stage_in(staging, a->interp[i].s, nd, true, itp[i]))) return rc;

    SysK k;
    k.sy = b.sy;
    k.sx = b.sx;
    k.csy = calloc_[2];
    k.csx = (long long)calloc_[1] * calloc_[2];
    const size_t slot_len = b.slot_elems;
    if (b.n[0] <= 0 || b.n[1] <= 0 || b.n[2] <= 0) return B2_OK;
    for (int i = 0; i < a->ncoefs; ++i) k.cf[i] = (const float *)C[i]->d;
    for (int i = a->ncoefs; i < B2_SYS_MAX_COEFS; ++i) k.cf[i] = nullptr;
    auto slot_of = [&](int f, int time, int shift) { return slot(time + shift, F[f]->size[0]); };

    // validate the stages once
    for (int s = 0; s < a->nstages; ++s) {
        const b2_sys_stage &st = a->stages[s];
        if (st.out_field < 0 || st.out_field >= a->nfields || st.ntaps < 1 || st.ntaps > B2_SYS_MAX_TAPS || !st.taps ||
            st.ext < 0 || st.ext > h) {
            set_error("b2_system_forward: stage %d is malformed (%d taps, at most %d; box widened by %d, at most %d)", s,
                      st.ntaps, B2_SYS_MAX_TAPS, st.ext, h);
            return B2_ERR_INVALID;
        }
        for (int i = 0; i < st.ntaps; ++i) {
            const b2_sys_tap &t = st.taps[i];
            if (t.field < 0 || t.field >= a->nfields || t.tshift < 0 || t.tshift > 1 || t.cfield >= a->ncoefs ||
                (st.ext > 0 && t.cfield >= 0)) {
                set_error("b2_system_forward: stage %d tap %d is malformed", s, i);
                return B2_ERR_INVALID;
            }
            // the kernel reads and writes in place: a shifted read of the written level would race with the writes
            if (t.field == st.out_field && slot_of(t.field, 0, t.tshift) == slot_of(t.field, 0, st.out_tshift) &&
                (t.off[0] || t.off[1] || t.off[2])) {
                set_error("b2_system_forward: stage %d reads shifted points of the level it writes", s);
                return B2_ERR_INVALID;
            }
            for (int d = 0; d < nd; ++d) {
                const int di = 3 - nd + d;
                if (b.o[di] - st.ext + t.off[d] < 0 || b.o[di] + b.n[di] - 1 + st.ext + t.off[d] >= b.a[di]) {
                    set_error("b2_system_forward: stage %d tap offset %d on dim %d leaves the allocated array", s, t.off[d], d);
                    return B2_ERR_INVALID;
                }
            }
        }
    }
    const FieldGeom g = field_geom(b, nd);

    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    double sec[3] = {0, 0, 0};
    const bool timing = a->timers != nullptr;
    if (timing) for (auto &e : ev) cudaEventCreate(&e);
    dim3 block(64, 4, 1);
    const int nsteps = a->time_M - a->time_m + 1;
    const bool per_step = timing && nsteps <= 2048;
    std::vector<cudaEvent_t> pool;
    auto rec_ev = [&]() { cudaEvent_t e; cudaEventCreate(&e); cudaEventRecord(e, stream()); pool.push_back(e); };
    if (timing && !per_step) cudaEventRecord(ev[0], stream());
    for (int time = a->time_m; time <= a->time_M; ++time) {
        if (per_step) rec_ev();
        for (int s = 0; s < a->nstages; ++s) {
            const b2_sys_stage &st = a->stages[s];
            // the box, widened by ext on the space axes (internal axis 0 of a 2-D grid is the dummy extent 1)
            const int e0 = nd == 3 ? st.ext : 0, e = st.ext;
            k.n0 = b.n[0] + 2 * e0; k.n1 = b.n[1] + 2 * e; k.n2 = b.n[2] + 2 * e;
            k.o0 = b.o[0] - e0; k.o1 = b.o[1] - e; k.o2 = b.o[2] - e;
            // the coefficient arrays have no halo (unused when e > 0: no cfield)
            k.c0 = nd == 3 ? k.o0 - h : 0; k.c1 = k.o1 - h; k.c2 = k.o2 - h;
            const dim3 grid((k.n2 + 63) / 64, (k.n1 + 3) / 4, (unsigned)std::min(k.n0, 65535));
            k.out = (float *)F[st.out_field]->d + (size_t)slot_of(st.out_field, time, st.out_tshift) * slot_len;
            for (int f = 0; f < a->nfields; ++f)
                for (int t = 0; t < 2; ++t)
                    k.in[f][t] = (const float *)F[f]->d + (size_t)slot_of(f, time, t) * slot_len;
            k.ntaps = st.ntaps;
            for (int i = 0; i < st.ntaps; ++i) {
                const b2_sys_tap &t = st.taps[i];
                long long delta = 0;
                for (int d = 0; d < nd; ++d) {
                    const int di = 3 - nd + d;
                    delta += (long long)t.off[d] * (di == 0 ? k.sx : di == 1 ? k.sy : 1);
                }
                k.fld[i] = (short)t.field; k.tsh[i] = (short)t.tshift; k.cfi[i] = (short)t.cfield;
                k.delta[i] = (int)delta; k.coef[i] = t.coef;
            }
            k_system_stage<<<grid, block, 0, stream()>>>(k);
            count_launch();
        }
        if (per_step) rec_ev();
        for (int i = 0; i < a->ninject; ++i) {
            const b2_sys_inject &q = a->inject[i];
            float *f0 = (float *)F[q.fields[0]]->d + (size_t)slot_of(q.fields[0], time, q.tshift) * slot_len;
            float *f1 = q.nfields > 1 ? (float *)F[q.fields[1]]->d + (size_t)slot_of(q.fields[1], time, q.tshift) * slot_len : nullptr;
            // scale modes of k_inject: scalar | dt2 * param^2 | dt2 / param with dt2 := q.scale
            const float *prm = q.param_kind != B2_PARAM_SCALAR ? (const float *)injp[i]->d : nullptr;
            if ((rc = launch_inject(inj[i], g, f0, f1, time, q.param_kind, prm, q.scale, q.scale))) return rc;
            if (q.nfields > 2) {
                float *f2 = (float *)F[q.fields[2]]->d + (size_t)slot_of(q.fields[2], time, q.tshift) * slot_len;
                if ((rc = launch_inject(inj[i], g, f2, nullptr, time, q.param_kind, prm, q.scale, q.scale))) return rc;
            }
        }
        if (per_step) rec_ev();
        for (int i = 0; i < a->ninterp; ++i) {
            const b2_sys_interp &q = a->interp[i];
            const float *f = (const float *)F[q.field]->d + (size_t)slot_of(q.field, time, q.tshift) * slot_len;
            if ((rc = launch_interp(itp[i], g, f, nullptr, time))) return rc;
        }
        if (per_step) rec_ev();
    }
    if (timing && !per_step) cudaEventRecord(ev[1], stream());
    rc = sync_call("b2_system_forward");
    if (timing) {
        float ms = 0.f;
        if (per_step) {
            for (size_t i = 0; i + 3 < pool.size(); i += 4) {
                if (cudaEventElapsedTime(&ms, pool[i], pool[i + 1]) == cudaSuccess) sec[0] += ms;
                if (cudaEventElapsedTime(&ms, pool[i + 1], pool[i + 2]) == cudaSuccess) sec[1] += ms;
                if (cudaEventElapsedTime(&ms, pool[i + 2], pool[i + 3]) == cudaSuccess) sec[2] += ms;
            }
        } else if (rc == B2_OK && cudaEventElapsedTime(&ms, ev[0], ev[1]) == cudaSuccess) {
            sec[0] = ms;
        }
        a->timers->section0 += sec[0] * 1e-3;
        a->timers->section1 += sec[1] * 1e-3;
        a->timers->section2 += sec[2] * 1e-3;
        for (auto &x : ev) cudaEventDestroy(x);
        for (auto &x : pool) cudaEventDestroy(x);
    }
    return rc;
}

extern "C" int b2_system_forward(const struct b2_system_args *a) {
    if (!a || !a->fields || !a->stages) { set_error("b2_system_forward: NULL args"); return B2_ERR_INVALID; }
    if (a->ndim != 2 && a->ndim != 3) { set_error("b2_system_forward: ndim must be 2 or 3"); return B2_ERR_INVALID; }
    if (a->nfields < 1 || a->nfields > B2_SYS_MAX_FIELDS || a->ncoefs < 0 || a->ncoefs > B2_SYS_MAX_COEFS) {
        set_error("b2_system_forward: %d fields / %d coefficient arrays (at most %d / %d)", a->nfields, a->ncoefs,
                  B2_SYS_MAX_FIELDS, B2_SYS_MAX_COEFS);
        return B2_ERR_INVALID;
    }
    if (a->nstages < 0 || a->ninject < 0 || a->ninterp < 0 || (a->ninject && !a->inject) || (a->ninterp && !a->interp)) {
        set_error("b2_system_forward: malformed stage / injection / interpolation counts");
        return B2_ERR_INVALID;
    }
    // sparse terms index the fields: check them before anything is staged
    for (int i = 0; i < a->ninject; ++i) {
        const b2_sys_inject &q = a->inject[i];
        bool ok = q.nfields >= 1 && q.nfields <= 3 && q.param_kind >= B2_PARAM_SCALAR && q.param_kind <= B2_PARAM_M;
        for (int j = 0; ok && j < q.nfields; ++j) ok = q.fields[j] >= 0 && q.fields[j] < a->nfields;
        if (!ok) { set_error("b2_system_forward: injection %d is malformed (fields / parameter kind)", i); return B2_ERR_INVALID; }
    }
    for (int i = 0; i < a->ninterp; ++i)
        if (a->interp[i].field < 0 || a->interp[i].field >= a->nfields) {
            set_error("b2_system_forward: interpolation %d samples field %d of %d", i, a->interp[i].field, a->nfields);
            return B2_ERR_INVALID;
        }
    if (a->time_M < a->time_m) return B2_OK;
    std::lock_guard<std::mutex> api_lock(api_mutex());
    if (int rc0 = use_device(a->deviceid)) return rc0;
    Staging st;
    return st.finish(system_forward_body(a, st));
}
