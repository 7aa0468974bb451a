// CPU emulation of the one-thread-per-point isotropic kernels — TEST INFRASTRUCTURE ONLY.
//
// devito_b200/csrc/b2_iso_point.cuh holds the bodies of k_iso_generic / k_ot4_w / k_iso_fs_fix as
// __host__ __device__ functions. This file loops them over the grid on the CPU (compiled by nvcc as
// host code, no GPU needed) so that tests/test_zz_emulation.py can compare exactly the code the GPU
// runs — index arithmetic, mirrored free-surface taps, the OT4 composition — with the oracle.
// It mirrors the launch sequence of b2::iso_step / b2::iso_fs_fix (b2_iso.cu).
#include "b2_iso_point.cuh"

using namespace b2;

static IsoGK make_args(float *u, const int *alloc /* 3 */, int so, int R, int ndim, const float *w0,
                       const float *w1, const float *w2, const float *damp, int param_kind,
                       const float *param, float vp, float dt, const int *lo, const int *hi, int t0,
                       int t2, int t1) {
    IsoGK k;
    const size_t slot = (size_t)alloc[0] * alloc[1] * alloc[2];
    k.u0 = u + (size_t)t0 * slot;
    k.um = u + (size_t)t2 * slot;
    k.u1 = u + (size_t)t1 * slot;
    k.damp = damp;
    k.param = param;
    k.sy = alloc[2];
    k.sx = (long long)alloc[1] * alloc[2];
    for (int d = 0; d < 3; ++d) {
        const int n = hi[d] - lo[d] + 1;
        const int o = (ndim == 2 && d == 0) ? 0 : lo[d] + so;
        const int r = (ndim == 2 && d == 0) ? 0 : R;
        if (d == 0) { k.n0 = n; k.o0 = o; k.r0 = r; }
        if (d == 1) { k.n1 = n; k.o1 = o; k.r1 = r; }
        if (d == 2) { k.n2 = n; k.o2 = o; k.r2 = r; }
    }
    k.param_kind = param_kind;
    k.inv_dt = 1.0f / dt;
    k.inv_dt2 = 1.0f / (dt * dt);
    k.m_dt2 = (1.0f / (vp * vp)) * k.inv_dt2;
    memset(k.w, 0, sizeof(k.w));
    const float *ws[3] = {w0, w1, w2};
    for (int d = 0; d < 3; ++d)
        if (ws[d]) for (int i = 0; i <= R; ++i) k.w[d][i] = ws[d][i];
    k.W = nullptr;
    k.ot4c = dt * dt / 12.0f;
    k.vp2 = vp * vp;
    k.U1 = nullptr;
    k.dm = nullptr;
    k.dsx = k.dsy = 0;
    k.dg0 = k.dg1 = k.dg2 = 0;
    return k;
}

extern "C" int emu_iso_step(float *u, const int *alloc /* 3 */, int so, int R, int ndim, const float *w0,
                            const float *w1, const float *w2, const float *damp, int param_kind,
                            const float *param, float vp, float dt, const int *lo, const int *hi, int t0,
                            int t2, int t1, int free_surface, int ot4, float *W) {
    IsoGK k = make_args(u, alloc, so, R, ndim, w0, w1, w2, damp, param_kind, param, vp, dt, lo, hi, t0, t2, t1);
    if (ot4) {
        IsoGK g = k;
        g.W = W;
        g.o0 -= g.r0; g.o1 -= g.r1; g.o2 -= g.r2;
        g.n0 += 2 * g.r0; g.n1 += 2 * g.r1; g.n2 += 2 * g.r2;
        for (int x = 0; x < g.n0; ++x)
            for (int y = 0; y < g.n1; ++y)
                for (int z = 0; z < g.n2; ++z) ot4_w_point(g, x, y, z);
        k.W = W;
    }
    for (int x = 0; x < k.n0; ++x)
        for (int y = 0; y < k.n1; ++y)
            for (int z = 0; z < k.n2; ++z) iso_point(k, x, y, z);
    if (free_surface)
        for (int x = 0; x < k.n0; ++x)
            for (int y = 0; y < k.n1; ++y)
                for (int z = 0; z <= k.r2; ++z) iso_fs_point(k, x, y, z);
    return 0;
}

// One Born step without sparse terms, in the order of b2_iso_forward: update u, update U with the same
// kernel, then the Born source (b2::iso_born_source).
extern "C" int emu_born_step(float *u, float *U, const float *dm, const int *dmalloc, int dmh,
                             const int *alloc, int so, int R, const float *w0, const float *w1,
                             const float *w2, const float *damp, int param_kind, const float *param,
                             float vp, float dt, const int *lo, const int *hi, int t0, int t2, int t1) {
    IsoGK ku = make_args(u, alloc, so, R, 3, w0, w1, w2, damp, param_kind, param, vp, dt, lo, hi, t0, t2, t1);
    IsoGK kU = make_args(U, alloc, so, R, 3, w0, w1, w2, damp, param_kind, param, vp, dt, lo, hi, t0, t2, t1);
    for (int x = 0; x < ku.n0; ++x)
        for (int y = 0; y < ku.n1; ++y)
            for (int z = 0; z < ku.n2; ++z) iso_point(ku, x, y, z);
    for (int x = 0; x < kU.n0; ++x)
        for (int y = 0; y < kU.n1; ++y)
            for (int z = 0; z < kU.n2; ++z) iso_point(kU, x, y, z);
    ku.U1 = kU.u1;
    ku.dm = dm;
    ku.dsx = (long long)dmalloc[1] * dmalloc[2];
    ku.dsy = dmalloc[2];
    ku.dg0 = lo[0] + dmh; ku.dg1 = lo[1] + dmh; ku.dg2 = lo[2] + dmh;
    for (int x = 0; x < ku.n0; ++x)
        for (int y = 0; y < ku.n1; ++y)
            for (int z = 0; z < ku.n2; ++z) born_src_point(ku, x, y, z);
    return 0;
}

// Snapshot copy of the iteration box (b2::iso_snapshot)
extern "C" int emu_snapshot(const float *slot, const int *alloc, int so, float *snap, const int *salloc, int sh,
                            const int *lo, const int *hi) {
    SnapK k;
    k.src = slot;
    k.dst = snap;
    k.sy = alloc[2];
    k.sx = (long long)alloc[1] * alloc[2];
    k.dsy = salloc[2];
    k.dsx = (long long)salloc[1] * salloc[2];
    k.n0 = hi[0] - lo[0] + 1; k.n1 = hi[1] - lo[1] + 1; k.n2 = hi[2] - lo[2] + 1;
    k.o0 = lo[0] + so; k.o1 = lo[1] + so; k.o2 = lo[2] + so;
    k.d0 = lo[0] + sh; k.d1 = lo[1] + sh; k.d2 = lo[2] + sh;
    for (int x = 0; x < k.n0; ++x)
        for (int y = 0; y < k.n1; ++y)
            for (int z = 0; z < k.n2; ++z) snapshot_point(k, x, y, z);
    return 0;
}

// Generic constant-coefficient update, same marshalling and loop direction as b2_linear_forward (b2_api_linear.cu)
extern "C" int emu_linear_steps(float *f, int tsize, int ndim, const int *size /* ndim */, int halo, int ntaps,
                                const int *tshift, const int *off /* ntaps x 3 */, const float *coef,
                                int wshift, const int *lo_in, const int *hi_in, int time_m, int time_M) {
    int alloc[3] = {1, 1, 1}, lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0}, hal[3] = {0, 0, 0};
    for (int d = 0; d < ndim; ++d) {
        const int di = 3 - ndim + d;
        alloc[di] = size[d]; lo[di] = lo_in[d]; hi[di] = hi_in[d]; hal[di] = halo;
    }
    LinK k;
    k.sy = alloc[2];
    k.sx = (long long)alloc[1] * alloc[2];
    const size_t slot = (size_t)alloc[0] * alloc[1] * alloc[2];
    k.n0 = hi[0] - lo[0] + 1; k.n1 = hi[1] - lo[1] + 1; k.n2 = hi[2] - lo[2] + 1;
    k.o0 = lo[0] + hal[0]; k.o1 = lo[1] + hal[1]; k.o2 = lo[2] + hal[2];
    k.ntaps = ntaps;
    int shifts[4], nshift = 0;
    for (int i = 0; i < ntaps; ++i) {
        int s = -1;
        for (int j = 0; j < nshift; ++j) if (shifts[j] == tshift[i]) s = j;
        if (s < 0) { shifts[nshift] = tshift[i]; s = nshift++; }
        k.sel[i] = s;
        long long delta = 0;
        for (int d = 0; d < ndim; ++d) {
            const int di = 3 - ndim + d;
            delta += (long long)off[3 * i + d] * (di == 0 ? k.sx : di == 1 ? k.sy : 1);
        }
        k.delta[i] = delta;
        k.coef[i] = coef[i];
    }
    // like b2_linear_forward: an update of `f.backward` (wshift = -1) runs from time_M down to time_m
    const int dirn = wshift;
    for (int time = dirn > 0 ? time_m : time_M; dirn > 0 ? time <= time_M : time >= time_m; time += dirn) {
        k.out = f + (size_t)((((time + wshift) % tsize) + tsize) % tsize) * slot;
        for (int j = 0; j < 4; ++j)
            k.lvl[j] = f + (size_t)((((time + shifts[j < nshift ? j : 0]) % tsize) + tsize) % tsize) * slot;
        for (int x = 0; x < k.n0; ++x)
            for (int y = 0; y < k.n1; ++y)
                for (int z = 0; z < k.n2; ++z) linear_point(k, x, y, z);
    }
    return 0;
}
