// C-ABI entry point b2_linear_forward: explicit time stepping of ONE field with a constant-coefficient
// linear stencil — the generated `Kernel` of operators like the reference's 2-D diffusion example
// (examples/cfd/example_diffusion.py:120-133; BASELINE config 1):
//
//   for time in [time_m, time_M]:  f[(time + wshift) % T][p] = sum_k coef_k * f[(time + tshift_k) % T][p + off_k]
//
// One thread per point (k_linear), taps in the kernel parameter block. This is the plumbing-size path
// (512^2 in BASELINE config 1), not a tuned sweep: the hot wave-propagation schemes have their own kernels.
#include "b2_common.cuh"
#include "b2_iso_point.cuh"
#include <algorithm>

using namespace b2;

namespace b2 {

__global__ void __launch_bounds__(256) k_linear(LinK k) {
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    if (z >= k.n2) return;
    // y and x are grid-strided: gridDim.y and gridDim.z are clamped to the hardware's 65 535
    for (int y = blockIdx.y * blockDim.y + threadIdx.y; y < k.n1; y += gridDim.y * blockDim.y)
        for (int x = blockIdx.z; x < k.n0; x += gridDim.z) linear_point(k, x, y, z);
}

}  // namespace b2

static int linear_forward_body(const b2_linear_args *a, Staging &st) {
    const int nd = a->ndim;
    DevArray *f;
    int rc = st.array(a->f, nd + 1, true, f);
    if (rc) return rc;
    const Box b = make_box(a, nd, f->size, a->halo);
    const int T = b.tsize;
    LinK k;
    k.sy = b.sy;
    k.sx = b.sx;
    k.n0 = b.n[0]; k.n1 = b.n[1]; k.n2 = b.n[2];
    k.o0 = b.o[0]; k.o1 = b.o[1]; k.o2 = b.o[2];
    if (k.n0 <= 0 || k.n1 <= 0 || k.n2 <= 0) return B2_OK;
    k.ntaps = a->ntaps;
    int shifts[4], nshift = 0;
    for (int i = 0; i < a->ntaps; ++i) {
        const b2_tap &t = a->taps[i];
        // the slot rule: no level read may share the written slot modulo T, or a point would read a cell that
        // another point of the same launch is writing
        if (slot(t.tshift - a->wshift, T) == 0) {
            set_error("b2_linear_forward: tap %d reads level t%+d, the slot being written (t%+d modulo %d slots)", i,
                      t.tshift, a->wshift, T);
            return B2_ERR_INVALID;
        }
        int s = -1;
        for (int j = 0; j < nshift; ++j) if (shifts[j] == t.tshift) s = j;
        if (s < 0) {
            if (nshift == 4) { set_error("b2_linear_forward: more than 4 time levels read"); return B2_ERR_INVALID; }
            shifts[nshift] = t.tshift;
            s = nshift++;
        }
        k.sel[i] = s;
        long long delta = 0;
        for (int d = 0; d < nd; ++d) {
            const int di = 3 - nd + d, o = t.off[d];
            // the read must stay inside the allocated array
            if (b.o[di] + o < 0 || b.o[di] + b.n[di] - 1 + o >= b.a[di]) {
                set_error("b2_linear_forward: tap offset %d on dim %d leaves the allocated array", o, d);
                return B2_ERR_INVALID;
            }
            delta += (long long)o * (di == 0 ? k.sx : di == 1 ? k.sy : 1);
        }
        k.delta[i] = delta;
        k.coef[i] = t.coef;
    }
    if ((rc = loop_timer_start(a->timers))) return rc;
    dim3 block(64, 4, 1);
    dim3 grid((k.n2 + 63) / 64, (unsigned)std::min((k.n1 + 3) / 4, 65535), (unsigned)std::min(k.n0, 65535));
    float *base = (float *)f->d;
    // an update of `f.backward` (wshift = -1) runs from time_M down to time_m, like the reference's
    // backward-in-time loop (devito/ir/support/space.py: Backward direction)
    const int dirn = a->wshift;
    for (int time = dirn > 0 ? a->time_m : a->time_M; dirn > 0 ? time <= a->time_M : time >= a->time_m; time += dirn) {
        k.out = base + (size_t)slot(time + a->wshift, T) * b.slot_elems;
        for (int j = 0; j < nshift; ++j) k.lvl[j] = base + (size_t)slot(time + shifts[j], T) * b.slot_elems;
        for (int j = nshift; j < 4; ++j) k.lvl[j] = k.lvl[0];
        k_linear<<<grid, block, 0, stream()>>>(k);
        count_launch();
    }
    return loop_finish("b2_linear_forward", a->timers);
}

extern "C" int b2_linear_forward(const struct b2_linear_args *a) {
    if (!a || !a->f || !a->taps) { set_error("b2_linear_forward: NULL args"); return B2_ERR_INVALID; }
    if (a->ndim < 1 || a->ndim > 3) { set_error("b2_linear_forward: ndim must be 1..3"); return B2_ERR_INVALID; }
    if (a->ntaps < 1 || a->ntaps > B2_MAX_TAPS) {
        set_error("b2_linear_forward: %d taps (1..%d supported)", a->ntaps, B2_MAX_TAPS);
        return B2_ERR_INVALID;
    }
    if (a->wshift != 1 && a->wshift != -1) { set_error("b2_linear_forward: wshift must be +1 or -1"); return B2_ERR_INVALID; }
    if (a->time_M < a->time_m) return B2_OK;
    std::lock_guard<std::mutex> api_lock(api_mutex());
    if (int rc0 = use_device(a->deviceid)) return rc0;
    Staging st;
    return st.finish(linear_forward_body(a, st));
}
