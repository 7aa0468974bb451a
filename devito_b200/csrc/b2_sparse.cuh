// Sparse source injection / receiver interpolation kernels (internal interface).
#pragma once
#include "b2_common.cuh"
#include "b2_iso.cuh"

namespace b2 {

struct SparseDev {
    bool present = false;
    const DevArray *data = nullptr, *gp = nullptr, *w[3] = {nullptr, nullptr, nullptr};   // held by a Staging
    int npoint_total = 0;   // second extent of data
    int nt = 0;
    int p_m = 0, p_M = -1;
    int r = 1;
    int ndim = 3;
};

// Field geometry the sparse kernels need (strides in the internal 3-dim convention of Box; bounds per grid dim)
struct FieldGeom {
    long long sx = 0, sy = 0;
    size_t slot_elems = 0;
    int so = 0;
    int ndim = 3;
    int lo[3] = {0, 0, 0};      // x_m, y_m, z_m
    int hi[3] = {0, 0, 0};      // x_M, y_M, z_M
    // x-slab decomposition: a neighbour owns the cells beyond x_m / x_M, so injection must not
    // touch them (the owner injects and its boundary planes are then exchanged)
    bool nb_lo = false, nb_hi = false;
    // streamed time loop (b2_api_iso.cu): [lo[0], hi[0]] is one x-range of a skewed sweep; interpolation then
    // samples only the cells of that range and ADDS its partial sum to the trace
    bool restrict_x = false;
    // ... or a range of dim 1 (the streamed loop under x-slab decomposition skews along y): [lo[1], hi[1]] is the
    // range, cut_lo1 / cut_hi1 say whether its ends are interior cuts (no reach beyond them)
    bool restrict_y = false, cut_lo1 = false, cut_hi1 = false;
    // fused halo step: cells injected into the first / last `pw` owned planes are mirrored into the
    // neighbour's halo copy (the sweep kernel stored those planes there before the injection)
    float *peer_lo = nullptr, *peer_hi = nullptr;
    long long off_lo = 0, off_hi = 0;        // element offset of "my plane 0" in the neighbour's array (slot included)
    int nown = 0, pw = 0;
};

// Checks the tables of `s` (radius, gp, the ndim weight tables, the point range against the traces) and only then
// stages them into `st`; `written`: the traces are copied back (receivers). `out.present` stays false without points.
int sparse_stage_in(Staging &st, const b2_sparse *s, int ndim, bool written, SparseDev &out);
// The sources and receivers (written back) of a wave call; the support of a point reaches r cells beyond the box, so
// an r beyond the halo `so` refuses the call (devito/operations/interpolators.py:28-37 `check_radius`).
int sparse_stage_pair(const char *who, Staging &st, const b2_sparse *src, const b2_sparse *rec, int ndim, int so,
                      SparseDev &src_out, SparseDev &rec_out);

// The geometry of box b on an `nd`-dim grid; under x-slab decomposition (`halo`) the cells beyond x_m / x_M
// belong to the neighbours.
FieldGeom field_geom(const Box &b, int nd, const b2_halo_ctx *halo = nullptr);

// Internal param_kind of launch_inject: the scale is a tabulated array in the field's layout, taken at the cell
// (the self-adjoint update's C = dt^2 vp^2 / b). Not part of the C ABI.
constexpr int B2_SCALE_TABLE = 3;

// u[cell] += w*w*w * src[time][p] * scale(cell) for up to two fields (TTI injects into u and v)
// scale(cell) = dt^2 * vp^2 | dt^2 * vp[cell]^2 | dt^2 / m[cell] | param[cell] (B2_SCALE_TABLE)
int launch_inject(const SparseDev &s, const FieldGeom &g, float *f0, float *f1, int time,
                  int param_kind, const float *param, float scalar_scale, float dt2);

// The (cell, value) entries launch_inject would add at `time` (3-D; inject_entry_count of them, skipped cells never
// match), written to `out` (device) when not null; `outside_flag` (device, may be null) |= 1 when a support cell lies
// outside the iteration box.
int inject_entry_count(const SparseDev &s);
int launch_inject_entries(const SparseDev &s, const FieldGeom &g, int time, int param_kind, const float *param,
                          float scalar_scale, float dt2, IsoInj *out, int *outside_flag);

// rec[time][p] = sum w*w*w * (f0[cell] (+ f1[cell]))
int launch_interp(const SparseDev &s, const FieldGeom &g, const float *f0, const float *f1, int time);

}  // namespace b2
