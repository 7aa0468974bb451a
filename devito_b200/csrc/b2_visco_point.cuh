// One-point form of the second-order SLS viscoacoustic update (b2_visco_forward).
//
// `__host__ __device__`, like b2_sa_point.cuh, so that tests/support/emu_visco.cu can run the same code (the tables,
// the adjoint's mix and the point body) on the CPU and compare it with the float64 restatement without a GPU. The
// scheme is the reference's `sls_2nd_order` (examples/seismic/viscoacoustic/operators.py:124-192). With the nested
// operator of the self-adjoint update
//
//   F_d(q) = b(q) * sum_k c_k [f(q + k e_d) - f(q - (k-1) e_d)],   L(f)(p) = sum_d sum_k c_k [F_d(p + (k-1) e_d) - F_d(p - k e_d)]
//
// (b at the nodes, c_k = the half-node first-derivative weights divided by h_d), whose code both updates share
// (nested_div of b2_nested_point.cuh here, k_nested_tma of b2_nested.cuh in the TMA sweep), and the per-point tables of
// k_visco_coef (t_s, tt from qp and f0, m = 1/vp^2, damp the "mask" profile, e = (1 - damp) / dt):
//
//   Kd = damp,  Kg = dt damp / t_s,  Kt = tt,  W = damp / (m/dt^2 + e),  Wm = W m / dt^2
//
// forward (r.dt and p.dt are the reference's first-order forward differences (f[t+1] - f[t]) / dt, their transposes
// (f[t-1] - f[t]) / dt; solved for the level written, with W e = Kd - Wm):
//   r[t+1] = (Kd - Kg) r[t] + Kg Kt L(p[t]) / b
//   p[t+1] = W ((1 + Kt) L(p[t]) / b - r[t+1]) + Wm (2 p[t] - p[t-1]) + (Kd - Wm) p[t]
// adjoint (time reversed; `visco_mix_point` over the whole slot, then the sweep on s):
//   r[t-1] = (Kd - Kg) r[t] - Kg Kt p[t]                                         (inside the box)
//   s      = ((1 + Kt) p[t] + r[t-1]) / b                                        (everywhere)
//   p[t-1] = W L(s) + Wm (2 p[t] - p[t+1]) + (Kd - Wm) p[t]
#pragma once
#include "b2_nested_point.cuh"
#include <cmath>

namespace b2 {

// the per-point tables (k_visco_coef), each one allocated slot of library scratch
enum { VK_D = 0, VK_G, VK_T, VK_W, VK_WM, VK_NTAB };

struct ViscoK {
    const float *__restrict__ f;     // the field L is applied to: p[t] forward, s on the adjoint
    const float *__restrict__ p0;    // p[t]
    const float *__restrict__ pm;    // p[t - dir]
    float *__restrict__ p1;          // p[t + dir], written
    const float *__restrict__ r0;    // r[t]       (forward only)
    float *__restrict__ r1;          // r[t + 1], written (forward only)
    const float *__restrict__ b;     // buoyancy, p's space layout (a scalar b is expanded into scratch)
    const float *__restrict__ K[VK_NTAB];
    long long sx, sy;
    int n0, n1, n2;                  // extents of this launch
    int o0, o1, o2;                  // array index of the first point
    int r[3];                        // radius per internal dim (0 on the dummy dim of a 2-D grid)
    float c[3][B2_MAX_RADIUS];       // c[d][k-1] = c_k / h_d
    int adjoint;
};

#define B2_VISCO_HD __host__ __device__ __forceinline__

B2_VISCO_HD long long visco_index(const ViscoK &k, int x, int y, int z) {
    return (long long)(k.o0 + x) * k.sx + (long long)(k.o1 + y) * k.sy + (k.o2 + z);
}

// the epilogue shared by both sweeps: given L at the point, the tables and the levels read, write the point
B2_VISCO_HD void visco_update(const ViscoK &k, long long idx, float lap, float bc) {
    const float kd = k.K[VK_D][idx], w = k.K[VK_W][idx], wm = k.K[VK_WM][idx];
    const float p0 = k.p0[idx], pm = k.pm[idx];
    float src = lap;
    if (!k.adjoint) {
        const float kg = k.K[VK_G][idx], kt = k.K[VK_T][idx];
        const float lb = lap / bc;
        const float rn = (kd - kg) * k.r0[idx] + kg * kt * lb;
        k.r1[idx] = rn;
        src = (1.f + kt) * lb - rn;
    }
    k.p1[idx] = w * src + wm * (2.f * p0 - pm) + (kd - wm) * p0;
}

B2_VISCO_HD void visco_point(const ViscoK &k, int x, int y, int z) {
    const long long idx = visco_index(k, x, y, z);
    visco_update(k, idx, nested_div(k.f, k.b, k.sx, k.sy, k.r, k.c, idx), k.b[idx]);
}

// The adjoint's pointwise pass (k_visco_adj_mix) over the whole allocated slot.
struct ViscoMixK {
    const float *K[VK_NTAB];
    const float *b, *p0, *r0;        // b, p[t], r[t]
    float *rw, *s;                   // r[t-1] (written inside the box, read outside it), s
    long long sx, sy;
    int o0, o1, o2, n0, n1, n2;      // the box, as in ViscoK
    size_t n;                        // elements of the slot
};

// slot index i: r[t-1] inside the box, s = ((1 + Kt) p[t] + r[t-1]) / b everywhere
B2_VISCO_HD void visco_mix_at(const ViscoMixK &k, size_t i) {
    const long long x = (long long)i / k.sx, rem = (long long)i - x * k.sx;
    const long long y = rem / k.sy, z = rem - y * k.sy;
    const bool inside = x >= k.o0 && x < k.o0 + k.n0 && y >= k.o1 && y < k.o1 + k.n1 && z >= k.o2 &&
                        z < k.o2 + k.n2;
    const float kt = k.K[VK_T][i];
    float rn;
    if (inside) {
        const float kg = k.K[VK_G][i];
        rn = (k.K[VK_D][i] - kg) * k.r0[i] - kg * kt * k.p0[i];
        k.rw[i] = rn;
    } else {
        rn = k.rw[i];
    }
    k.s[i] = ((1.f + kt) * k.p0[i] + rn) / k.b[i];
}

// The tables (k_visco_coef): each parameter an array or, where its pointer is null, the scalar next to it (damp: 1).
struct ViscoCoefK {
    float *K[VK_NTAB];
    float *bx;                       // b expanded when b is a scalar, else null
    const float *vp, *qp, *damp;
    float vp_value, qp_value, b_value;
    double f0, dt;
    size_t n;
};

B2_VISCO_HD void visco_coef_point(const ViscoCoefK &k, size_t i) {
    const double v = k.vp ? k.vp[i] : k.vp_value;
    const double q = k.qp ? k.qp[i] : k.qp_value;
    const double d = k.damp ? k.damp[i] : 1.0;
    const double dt = k.dt, f0 = k.f0;
    const double t_s = (sqrt(1.0 + 1.0 / (q * q)) - 1.0 / q) / f0;
    const double t_ep = 1.0 / (f0 * f0 * t_s);
    const double m = 1.0 / (v * v);
    const double w = d / (m / (dt * dt) + (1.0 - d) / dt);
    k.K[VK_D][i] = (float)d;
    k.K[VK_G][i] = (float)(dt * d / t_s);
    k.K[VK_T][i] = (float)(t_ep / t_s - 1.0);
    k.K[VK_W][i] = (float)w;
    k.K[VK_WM][i] = (float)(w * m / (dt * dt));
    if (k.bx) k.bx[i] = k.b_value;
}

}  // namespace b2
