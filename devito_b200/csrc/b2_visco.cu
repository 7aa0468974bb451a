// Second-order SLS viscoacoustic update (the reference's `sls_2nd_order`, examples/seismic/viscoacoustic/
// operators.py:124-192). Scheme and tables: b2_visco_point.cuh.
//
//   k_visco_coef     : once per call, the tables Kd, Kg, Kt, W, Wm over the whole allocated slot into library scratch
//                      (from vp, b, qp, f0, dt and damp, each an array or a scalar), so that the sweeps have one form
//                      for scalar and array parameters; a scalar b is expanded into scratch too.
//   k_visco_adj_mix  : adjoint only, pointwise over the whole allocated slot, halo included: r[t-1] inside the box and
//                      s = ((1 + tt) p[t] + r[t-1]) / b everywhere, because the sweep reads s up to 2R-1 outside the
//                      box. L is linear, so the reference's two nested terms L((1+tt) rho p) + L(rho r[t-1]) are L(s).
//   k_visco_generic  : one thread per point, any even space order <= 16, 2-D and 3-D, any alignment. Its point body is
//                      b2_visco_point.cuh (run on the CPU by tests/support/emu_visco.cu, with the tables and the mix).
//   visco_tma<R>     : the 2.5-D TMA sweep of the nested operator shared with the self-adjoint update
//                      (k_nested_tma<R, ViscoEpi<ADJ>>, b2_nested.cuh; 3-D grids, R in {2, 4}) on p[t], or on s on the
//                      adjoint. Its epilogue ViscoEpi runs visco_update of b2_visco_point.cuh on four z points with
//                      16-byte loads and stores (DESIGN §3.3k).
//
// Algorithmic bytes per point and step (DESIGN §3.3k): forward 44 (p[t], b, p[t-1], r[t], five tables; writes r[t+1],
// p[t+1]); adjoint 64 (the mix reads p[t], r[t], Kd, Kg, Kt, b and writes r[t-1], s: 32; the sweep reads s, b, p[t],
// p[t+1], Kd, W, Wm and writes p[t-1]: 32).
//
// The host side is the nested operator's (b2_nested.cuh): nested_plan_init chooses the kernel, points b at the array
// or at g_visco_scratch[VK_NTAB] and encodes the maps of p (or s) and b; visco_plan_init adds s and the tables and runs
// k_visco_coef, and visco_step fills the epilogue or the ViscoK members of its own before launch_nested_tma /
// launch_nested_generic.
#include "b2_visco.cuh"
#include "b2_nested.cuh"
#include <algorithm>
#include <cmath>

namespace b2 {

__global__ void __launch_bounds__(256) k_visco_generic(ViscoK k) {
    const int z = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (z >= k.n2 || y >= k.n1) return;
    for (int x = blockIdx.z; x < k.n0; x += gridDim.z) visco_point(k, x, y, z);
}

__global__ void __launch_bounds__(256) k_visco_adj_mix(ViscoMixK k) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < k.n; i += (size_t)gridDim.x * blockDim.x)
        visco_mix_at(k, i);
}

#define VK_AT(v, c) ((c) == 0 ? (v).x : (c) == 1 ? (v).y : (c) == 2 ? (v).z : (v).w)

// the epilogue of k_nested_tma (b2_nested.cuh): visco_update of b2_visco_point.cuh on four points
template <bool ADJ> struct ViscoEpi {
    const float *p0, *pm;            // p[t], p[t - dir] slots (p[t] read on the adjoint only: the ring holds s)
    float *p1;                       // p[t + dir] slot
    const float *r0;                 // r[t] slot (forward)
    float *r1;                       // r[t+1] slot (forward)
    const float *K[VK_NTAB];

    __device__ __forceinline__ void operator()(float4 acc, const float *U, int ucol, int bcol, long long off,
                                               int zcnt) const {
        const float4 kd = ldg4(K[VK_D] + off), w = ldg4(K[VK_W] + off);
        const float4 wm = ldg4(K[VK_WM] + off);
        const float4 p0 = ADJ ? ldg4(this->p0 + off) : b2ptx::lds128(U + ucol);
        const float4 pm = ldg4(this->pm + off);
        float4 src = acc, rn = acc;
        if (!ADJ) {
            const float4 bc = b2ptx::lds128(U + bcol);
            const float4 kg = ldg4(K[VK_G] + off), kt = ldg4(K[VK_T] + off);
            const float4 r0 = ldg4(this->r0 + off);
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const float lb = VK_AT(acc, c) / VK_AT(bc, c);
                const float r = (VK_AT(kd, c) - VK_AT(kg, c)) * VK_AT(r0, c) + VK_AT(kg, c) * VK_AT(kt, c) * lb;
                const float sv = (1.f + VK_AT(kt, c)) * lb - r;
                if (c == 0) { rn.x = r; src.x = sv; }
                else if (c == 1) { rn.y = r; src.y = sv; }
                else if (c == 2) { rn.z = r; src.z = sv; }
                else { rn.w = r; src.w = sv; }
            }
        }
        float4 o;
        o.x = w.x * src.x + wm.x * (2.f * p0.x - pm.x) + (kd.x - wm.x) * p0.x;
        o.y = w.y * src.y + wm.y * (2.f * p0.y - pm.y) + (kd.y - wm.y) * p0.y;
        o.z = w.z * src.z + wm.z * (2.f * p0.z - pm.z) + (kd.z - wm.z) * p0.z;
        o.w = w.w * src.w + wm.w * (2.f * p0.w - pm.w) + (kd.w - wm.w) * p0.w;
        float *dp = p1 + off;
        float *dr = ADJ ? nullptr : r1 + off;
        if (zcnt == 4) {
            *reinterpret_cast<float4 *>(dp) = o;
            if (!ADJ) *reinterpret_cast<float4 *>(dr) = rn;
        } else {
            dp[0] = o.x;
            if (zcnt > 1) dp[1] = o.y;
            if (zcnt > 2) dp[2] = o.z;
            if (!ADJ) {
                dr[0] = rn.x;
                if (zcnt > 1) dr[1] = rn.y;
                if (zcnt > 2) dr[2] = rn.z;
            }
        }
    }
};

// one step of the TMA sweep (the ring streams slot t0 of p, or the single slot s on the adjoint)
template <bool ADJ>
static int visco_step_tma(const ViscoPlan &p, int t0, int t2, int t1) {
    auto at = [&](float *x, int t) { return x + (size_t)t * p.slot_elems; };
    ViscoEpi<ADJ> e;
    e.p0 = at(p.p, t0);
    e.pm = at(p.p, t2);
    e.p1 = at(p.p, t1);
    e.r0 = ADJ ? nullptr : at(p.r, t0);
    e.r1 = ADJ ? nullptr : at(p.r, t1);
    for (int i = 0; i < VK_NTAB; ++i) e.K[i] = p.K[i];
    const int slot0 = ADJ ? 0 : t0;
    return p.radius[2] == 2 ? launch_nested_tma<2>(p, slot0, e, "visco") : launch_nested_tma<4>(p, slot0, e, "visco");
}

// the tables of b2_visco_point.cuh over the slot (and bx = b when b is a scalar), evaluated in double
__global__ void __launch_bounds__(256) k_visco_coef(ViscoCoefK k) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < k.n; i += (size_t)gridDim.x * blockDim.x)
        visco_coef_point(k, i);
}

// scratch cached across calls: the tables, b, s
static ScratchSlot g_visco_scratch[VK_NTAB + 2];

int visco_plan_init(ViscoPlan &p, int kernel) {
    int rc;
    // the TMA sweep's ring streams p[t] forward (every slot of p, the slot a coordinate) and the single slot s on the
    // adjoint, so s comes before the maps
    if (p.adjoint && (rc = cached_scratch(g_visco_scratch[VK_NTAB + 1], p.slot_elems, &p.s))) return rc;
    if ((rc = nested_plan_init(p, kernel, "b2_visco_forward", g_visco_scratch[VK_NTAB], {p.p, p.r},
                               p.adjoint ? p.s : p.p, p.adjoint ? 1 : p.tsize)))
        return rc;
    for (int i = 0; i < VK_NTAB; ++i)
        if ((rc = cached_scratch(g_visco_scratch[i], p.slot_elems, &p.K[i]))) return rc;
    const size_t n = p.slot_elems;
    const int blocks = (int)std::min<size_t>((n + 255) / 256, 65535);
    ViscoCoefK ck;
    for (int i = 0; i < VK_NTAB; ++i) ck.K[i] = p.K[i];
    ck.bx = p.b_arr ? nullptr : p.b;
    ck.vp = p.vp_arr; ck.qp = p.qp_arr; ck.damp = p.damp;
    ck.vp_value = p.vp_value; ck.qp_value = p.qp_value; ck.b_value = p.b_value;
    ck.f0 = p.f0; ck.dt = p.dt;
    ck.n = n;
    k_visco_coef<<<blocks, 256, 0, stream()>>>(ck);
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

static int visco_mix(const ViscoPlan &p, int t0, int t2, int t1) {
    ViscoMixK k;
    for (int i = 0; i < VK_NTAB; ++i) k.K[i] = p.K[i];
    k.b = p.b;
    k.p0 = p.p + (size_t)t0 * p.slot_elems;
    k.r0 = p.r + (size_t)t0 * p.slot_elems;
    k.rw = p.r + (size_t)t1 * p.slot_elems;
    k.s = p.s;
    k.sx = p.sx;
    k.sy = p.sy;
    k.o0 = p.o[0]; k.o1 = p.o[1]; k.o2 = p.o[2];
    k.n0 = p.n[0]; k.n1 = p.n[1]; k.n2 = p.n[2];
    k.n = p.slot_elems;
    const int blocks = (int)std::min<size_t>((k.n + 255) / 256, 65535);
    timing_begin();
    k_visco_adj_mix<<<blocks, 256, 0, stream()>>>(k);
    timing_end();
    count_launch();
    B2_CUDA(cudaGetLastError(), B2_ERR_LAUNCH);
    return B2_OK;
}

int visco_step(const ViscoPlan &p, int t0, int t2, int t1) {
    int rc;
    if (p.adjoint && (rc = visco_mix(p, t0, t2, t1))) return rc;
    if (p.use_tma) return p.adjoint ? visco_step_tma<true>(p, t0, t2, t1) : visco_step_tma<false>(p, t0, t2, t1);
    auto at = [&](float *x, int t) { return x + (size_t)t * p.slot_elems; };
    ViscoK k;
    k.p0 = at(p.p, t0);
    k.pm = at(p.p, t2);
    k.p1 = at(p.p, t1);
    k.f = p.adjoint ? p.s : k.p0;
    k.r0 = p.adjoint ? nullptr : at(p.r, t0);
    k.r1 = p.adjoint ? nullptr : at(p.r, t1);
    k.b = p.b;
    for (int i = 0; i < VK_NTAB; ++i) k.K[i] = p.K[i];
    k.adjoint = p.adjoint ? 1 : 0;
    return launch_nested_generic(k_visco_generic, k, p, "visco");
}

}  // namespace b2
