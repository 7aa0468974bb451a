// Internal interface of the isotropic-acoustic stencil kernels (b2_iso.cu).
#pragma once
#include "b2_common.cuh"

namespace b2 {

// The box: internal dims are always 3, for 2-D grids dim 0 is a dummy of extent 1 (radius 0).
struct IsoPlan : Box {
    int radius[3] = {0, 0, 0};
    float *u = nullptr;
    const float *damp = nullptr;
    const float *param = nullptr;
    int param_kind = B2_PARAM_SCALAR;
    float vp = 1.f, dt = 1.f;
    float w[3][B2_MAX_RADIUS + 1] = {};
    // TMA path
    bool use_tma = false;
    CUtensorMap tm_uh, tm_uc, tm_damp, tm_par;   // tm_damp/tm_par map coefA/coefB
    float *coefA = nullptr, *coefB = nullptr;    // tabulated update coefficients (library scratch)
    bool defer_coef = false;                     // plan init only allocates them (streamed loop: per chunk)
    // scalar parameter, whole table tabulated: one byte per allocated x-plane (library scratch, device), 1 where
    // damp on the plane equals damp on the pin plane o[0] + n[0]/2 bit for bit over the update box, so that A
    // does too. NULL otherwise: the sweep then streams every A tile.
    const unsigned char *coef_reuse = nullptr;
    int lx = 0;
    // OT4 (b2_iso_args.ot4): generic two-pass path, W = lap(u)/m in library scratch
    bool ot4 = false;
    float *ot4W = nullptr;
};

// x-slab decomposition: the halo step fused into the TMA sweep (b2_halo.cu fills it per step). The CTAs that
// produce the first / last `radius` owned planes also store them into the neighbour's halo through the
// CUDA-IPC mapped pointers; CTAs that read halo planes of u[t] acquire the neighbour's flag first.
struct IsoFuse {
    float *peer_lo = nullptr, *peer_hi = nullptr;     // neighbour field bases (all time slots); NULL = boundary
    long long slot_lo = 0, slot_hi = 0;               // elements of one time slot in the neighbour's array
    int n_lo = 0, n_hi = 0;                           // x-planes the neighbours own
    const int *flag_lo = nullptr, *flag_hi = nullptr; // local flags released by the neighbours
    int want = -1;                                    // flag value to acquire (< 0: halos already in place)
};

// Prepare the plan (decides generic vs TMA kernel, encodes tensor maps). `kernel`: 0 auto,
// 1 force generic, 2 force TMA (error if the layout does not qualify).
int iso_plan_init(IsoPlan &p, int kernel);

// (Re)tabulate the coefficient tables on the allocated x-planes [plane_lo, plane_hi).
int iso_coef_tabulate_planes(const IsoPlan &p, int plane_lo, int plane_hi);
// Tabulate the whole tables once damp and the parameter are on the device; with a scalar parameter also find
// the planes whose A repeats the pin plane's (p.coef_reuse).
int iso_coef_tabulate_all(IsoPlan &p);
// Planes of the last iso call whose A came from the pinned tile (reads the flags back: synchronises the stream).
int iso_coef_reuse_count();
int iso_coef_tabulate_rows(const IsoPlan &p, int x0, int x1, int y0, int y1);

// One time step over x in [xlo, xlo + xcount) (relative to the iteration origin):
// u[slot1] = update(u[slot0], u[slotm]).
int iso_step(const IsoPlan &p, int slot0, int slotm, int slot1, int xlo, int xcount);

// Same over the whole owned x-range with the fused halo step (TMA kernel only: p.use_tma).
int iso_step_fused(const IsoPlan &p, int slot0, int slotm, int slot1, const IsoFuse &f);

// Free surface at the low end of the last dimension: after iso_step, recompute the rows z < radius
// with mirrored vertical taps and clear the surface row (b2_iso_args.free_surface).
int iso_fs_fix(const IsoPlan &p, int slot0, int slotm, int slot1, int xlo, int xcount);

// ---- two-level pass (so = 8, scalar parameter): u[t] -> u[t+1] (its slot) and u[t+2] (a scratch slot) ----
// One source-injection entry of a step: cell (x, y, z) relative to the iteration origin, value added.
struct IsoInj {
    int x, y, z;
    float v;
};
constexpr int B2_ISO2_MAX_INJ = 64;                 // entries the pass takes; more: the one-step loop
// The plan qualifies for the pass (radius 4 on every axis, scalar parameter, TMA layout, 3 slots).
bool iso2_supported(const IsoPlan &p);
// Allocates the two scratch slots (u's slot layout, 2 x slot_elems floats, cached across calls); ok = false, with no
// error, when the device has no room for them.
int iso2_reserve(const IsoPlan &p, bool &ok);
// After iso2_reserve: zeroes the scratch slots outside the update box when the layout changed, encodes their
// tensor maps; `scratch[k]` is slot k's base.
int iso2_prepare(const IsoPlan &p, float *scratch[2]);
// flag |= 1 when any of u's 3 slots holds a non-zero outside the update box (device; the caller reads it back)
int iso2_halo_nonzero(const IsoPlan &p, int *flag);
// One pass: level 1 reads u[t] from slot `slot0` (src_scratch < 0) or scratch `src_scratch`, u[t-1] from slot
// `slotm`, writes u[t+1] to slot `slot1` with the entries `inj` (device, `ninj` of them) added, and u[t+2] to
// scratch `dst_scratch`.
int iso_step2(const IsoPlan &p, int slot0, int src_scratch, int slotm, int slot1, int dst_scratch, const IsoInj *inj,
              int ninj);

// Snapshot: copy the iteration box of time slot `slot` into one snapshot (own strides; (d0,d1,d2) = index
// of the first iterated point in the snapshot array)
int iso_snapshot(const IsoPlan &p, int slot, float *snap, long long dsx, long long dsy, int d0, int d1, int d2);

// Born: U1 += -dm * u.dt2 / (m/dt^2 + damp/dt) over the iteration box; `p` is u's plan (slots of u),
// U1 the new time level of the linearised field (same layout), dm with its own strides and the index
// (dg0, dg1, dg2) of the first iterated point.
int iso_born_source(const IsoPlan &p, int slot0, int slotm, int slot1, float *U1, const float *dm,
                    long long dsx, long long dsy, int dg0, int dg1, int dg2);

}  // namespace b2
