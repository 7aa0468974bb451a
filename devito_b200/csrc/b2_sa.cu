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
//   sa_tma<R>    : the 2.5-D TMA sweep of the nested operator shared with the viscoacoustic update
//                  (k_nested_tma<R, SaEpi>, b2_nested.cuh; 3-D grids, R in {2, 4}) on u[t]. Its epilogue SaEpi reads C,
//                  w and u[t-dir] once with 16-byte loads and writes u[t+dir] with 16-byte stores.
//
// The host side is the nested operator's (b2_nested.cuh): nested_plan_init chooses the kernel, points b at the array
// or at g_sa_scratch[1] and encodes the maps of u and b; sa_plan_init adds C and runs k_sa_coef, and sa_step fills the
// epilogue or the SaK members of its own before launch_nested_tma / launch_nested_generic.
#include "b2_sa.cuh"
#include "b2_sa_point.cuh"
#include "b2_nested.cuh"
#include <algorithm>

namespace b2 {

__global__ void __launch_bounds__(256) k_sa_generic(SaK k) {
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (z >= k.n2 || y >= k.n1) return;
    for (int x = blockIdx.z; x < k.n0; x += gridDim.z) sa_point(k, x, y, z);
}

// the epilogue of k_nested_tma (b2_nested.cuh): the point body of b2_sa_point.cuh on four points
struct SaEpi {
    const float *um;                 // u[t - dir] slot
    float *u1;                       // u[t + dir] slot
    const float *C, *w;              // w may be null
    float dt;

    __device__ __forceinline__ void operator()(float4 acc, const float *U, int ucol, int, long long off,
                                               int zcnt) const {
        const float4 c = b2ptx::lds128(U + ucol);
        const float4 cv = ldg4(C + off);
        const float4 pv = ldg4(um + off);
        const float4 wv = w ? ldg4(w + off) : make_float4(0.f, 0.f, 0.f, 0.f);
        float4 o;
        o.x = fmaf(cv.x, acc.x, fmaf(2.f - dt * wv.x, c.x, (dt * wv.x - 1.f) * pv.x));
        o.y = fmaf(cv.y, acc.y, fmaf(2.f - dt * wv.y, c.y, (dt * wv.y - 1.f) * pv.y));
        o.z = fmaf(cv.z, acc.z, fmaf(2.f - dt * wv.z, c.z, (dt * wv.z - 1.f) * pv.z));
        o.w = fmaf(cv.w, acc.w, fmaf(2.f - dt * wv.w, c.w, (dt * wv.w - 1.f) * pv.w));
        float *dst = u1 + off;
        if (zcnt == 4) {
            *reinterpret_cast<float4 *>(dst) = o;
        } else {
            dst[0] = o.x;
            if (zcnt > 1) dst[1] = o.y;
            if (zcnt > 2) dst[2] = o.z;
        }
    }
};

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

// scratch cached across calls: C, and b expanded when it is a scalar
static ScratchSlot g_sa_scratch[2];

int sa_plan_init(SaPlan &p, int kernel) {
    int rc;
    if ((rc = nested_plan_init(p, kernel, "b2_sa_forward", g_sa_scratch[1], {p.u, p.w}, p.u, p.tsize))) return rc;
    if ((rc = cached_scratch(g_sa_scratch[0], p.slot_elems, &p.C))) return rc;
    const size_t n = p.slot_elems;
    const int blocks = (int)std::min<size_t>((n + 255) / 256, 65535);
    k_sa_coef<<<blocks, 256, 0, stream()>>>(p.C, p.b_arr ? nullptr : p.b, p.vp_arr, p.b_arr, p.vp_value, p.b_value,
                                            p.dt * p.dt, n);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

int sa_step(const SaPlan &p, int slot0, int slotm, int slot1) {
    if (p.use_tma) {
        const SaEpi e{p.u + (size_t)slotm * p.slot_elems, p.u + (size_t)slot1 * p.slot_elems, p.C, p.w, p.dt};
        return p.radius[2] == 2 ? launch_nested_tma<2>(p, slot0, e, "sa") : launch_nested_tma<4>(p, slot0, e, "sa");
    }
    SaK k;
    k.u0 = p.u + (size_t)slot0 * p.slot_elems;
    k.um = p.u + (size_t)slotm * p.slot_elems;
    k.u1 = p.u + (size_t)slot1 * p.slot_elems;
    k.b = p.b;
    k.C = p.C;
    k.w = p.w;
    k.dt = p.dt;
    return launch_nested_generic(k_sa_generic, k, p, "sa");
}

}  // namespace b2
