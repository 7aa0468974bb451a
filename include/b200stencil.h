/*
 * b200stencil.h — C ABI of the H100-native wave-propagation backend (libb200stencil.so).
 *
 * This is the drop-in boundary for the ONE hot path named in BASELINE.json: the time loop
 * that the reference's `Operator` emits for acoustic / TTI wave propagation.  In the
 * reference that loop is a JIT-generated C function
 *
 *     int Forward(struct dataobj *damp_vec, ..., struct dataobj *u_vec, const float vp,
 *                 const int x_M, const int x_m, ..., const int time_M, const int time_m,
 *                 ..., struct profiler *timers)
 *
 * looked up with `getattr(lib, name)` and called once per `Operator.apply`
 * (devito/operator/operator.py:857-869 `cfunction`, :1032 the FFI crossing; printed
 * samples of the generated code: examples/seismic/tutorials/08_snapshotting.ipynb:461-505).
 * The entry points below take exactly the same kinds of things — `struct dataobj`
 * descriptors, scalar spacings/dt, inclusive iteration bounds, a `struct profiler` — but
 * are pre-built for sm_90a instead of generated.  Only plain pointers, ints and floats
 * cross the boundary (no torch types).
 *
 * Conventions shared with the reference
 *   - arrays are C row-major `(time, x, y, z)`, z fastest, halo = space_order points per
 *     side on every space dimension (devito/types/dense.py:1256-1259), `time` has
 *     `size[0]` slots addressed `time % size[0]` (ModuloDimension t0/t1/t2,
 *     devito/ir/clusters/algorithms.py:321-427);
 *   - bounds `x_m..x_M`, `time_m..time_M`, `p_*_m..p_*_M` are INCLUSIVE
 *     (devito/types/dimension.py:279-331);
 *   - return value: 0 ok; 100 NaN/Inf in the wavefield; 200..203 device/launch failures
 *     (devito/passes/iet/errors.py:192-198).  We add 210 = invalid argument.
 *
 * Process model: one process per GPU (like the reference's device path: one MPI rank per GPU).
 * The library binds to the first `deviceid` it is given; a later call naming another device
 * returns 210.  b2_iso_forward / b2_tti_forward are blocking and serialised by an internal mutex,
 * so they may be called from several host threads (ctypes drops the GIL) but do not overlap.
 */
#ifndef B200STENCIL_H
#define B200STENCIL_H

#ifdef __cplusplus
extern "C" {
#endif

/* Identical to the reference's `struct dataobj` (devito/types/dense.py:737-746; printed in
 * examples/performance/01_gpu.ipynb:262-273).  `data` is the HOST array; `dmap` is the
 * device-resident mirror.  The reference fills `dmap` in C-land per call
 * (devito/passes/iet/languages/openacc.py:245-247); here:
 *    dmap == NULL : the callee allocates device memory, copies `data` H2D on entry, copies
 *                   written arrays D2H on exit and frees (== reference `devicerm=1`);
 *    dmap != NULL : the array is device-resident at `dmap` (same layout); no copies.
 * Written arrays are copied back when the call returns 0 or 100 (NaN); on any other return code
 * the host arrays are left untouched.  The device memory staged for a call is released on every
 * return path (b2_staging_outstanding counts what is still held).                        */
struct b2_dataobj {
    void *data;
    int *size;              /* allocated shape, ndim entries                               */
    unsigned long nbytes;
    unsigned long *npsize;  /* unused by this library (may be NULL)                        */
    unsigned long *dsize;   /* unused by this library (may be NULL)                        */
    int *hsize;             /* halo sizes  [d0_L, d0_R, d1_L, ...] (may be NULL)           */
    int *hofs;              /* halo offsets (may be NULL)                                  */
    int *oofs;              /* owned offsets (may be NULL)                                 */
    void *dmap;
};

/* Same role as the reference's `struct profiler` (devito/types/misc.py:41-68; printed
 * 01_gpu.ipynb cell 23): accumulated seconds per section.  section0 = stencil update,
 * section1 = source injection, section2 = receiver interpolation, haloupdate0 = exchange. */
struct b2_profiler {
    double section0;
    double section1;
    double section2;
    double haloupdate0;
};

/* One SparseTimeFunction with the host-tabulated tables the reference passes
 * (`*_gp`, `*_wx/wy/wz`; devito/operations/interpolators.py:390-421, 674-718). */
struct b2_sparse {
    struct b2_dataobj *data;      /* (nt, npoint) f32                                      */
    struct b2_dataobj *gp;        /* (npoint, ndim) i32 : base cell index                  */
    struct b2_dataobj *w[3];      /* (npoint, 2r) f32 per dim; unused dims NULL             */
    int p_m, p_M;                 /* inclusive point range                                  */
    int r;                        /* interpolation radius (linear: 1, sinc: 4)              */
};

/* What the sparse terms of the Operator look like (acoustic/operators.py:143-146,
 * tti/operators.py:475-477). */
enum { B2_PARAM_SCALAR = 0, B2_PARAM_VP = 1, B2_PARAM_M = 2 };

/* Halo-exchange context for slab decomposition along x (replaces `MPI_Comm comm, struct
 * neighborhood *nb` of the generated code, devito/mpi/distributed.py:822-902). Opaque. */
typedef struct b2_halo_ctx b2_halo_ctx;

/* ---- isotropic acoustic forward (replaces generated `Forward`,
 *      examples/seismic/acoustic/operators.py:71-150) -------------------------------------
 * u[t+1] = ( m (2u[t] - u[t-1])/dt^2 + damp u[t]/dt + sum_d sum_k w_d[k] u[t][.. +k ..] )
 *          / ( m/dt^2 + damp/dt ),   m = 1/vp^2
 * then  u[t+1][cell] += w.w.w * src[t][p] * dt^2 / m(cell)     (section1)
 * then  rec[t][p] = sum w.w.w * u[t + rec_toff][cell]           (section2)
 */
struct b2_iso_args {
    int ndim;                         /* 2 or 3                                             */
    int space_order;                  /* halo width of u/damp/param arrays                  */
    int radius;                       /* stencil radius (space_order/2)                     */
    const float *w[3];                /* per-dim FD weights incl. 1/h^2: w[d][0..radius]    *
                                       * (symmetric; w[d][0] is the centre weight)          */
    struct b2_dataobj *u;             /* (tsize, x+2so, y+2so, z+2so)                       */
    struct b2_dataobj *damp;          /* NULL -> no damping term                            */
    int param_kind;                   /* B2_PARAM_*                                         */
    struct b2_dataobj *param;         /* vp or m array when param_kind != SCALAR            */
    float vp;                         /* scalar velocity when param_kind == SCALAR          */
    float dt;
    int x_m, x_M, y_m, y_M, z_m, z_M; /* for ndim==2 the z entries are ignored              */
    int time_m, time_M;
    struct b2_sparse *src;            /* NULL -> no injection                               */
    struct b2_sparse *rec;            /* NULL -> no interpolation                           */
    int rec_toff;                     /* 0: rec reads u[t] (pre-update), 1: u[t+1]          */
    int errctl;                       /* !=0: NaN check every 100 steps -> return 100       */
    int deviceid;
    int kernel;                       /* 0 auto, 1 force generic kernel, 2 force TMA kernel */
    b2_halo_ctx *halo;                /* NULL -> single device                              */
    struct b2_profiler *timers;       /* may be NULL                                        */
    int adjoint;                      /* 0: forward in time. 1: the reference's `Adjoint`    *
                                       * operator (acoustic/operators.py:153-187): time runs *
                                       * from time_M down to time_m, u[t-1] is written from   *
                                       * u[t], u[t+1]; `src` is injected into u[t-1] (the     *
                                       * receiver data), `rec` samples u[t + rec_toff]        *
                                       * (rec_toff in {0,-1})                                 */
    /* imaging condition of the reference's `Gradient` operator (acoustic/operators.py:190-232):
     * after each (adjoint) step   grad -= usave[time] * (u[t+1] - 2 u[t] + u[t-1]) / dt^2.
     * `usave` is the forward wavefield saved with save=nt (same layout as u, nt time slots);
     * `grad` may have its own halo width (hsize). Both NULL -> no imaging condition.          */
    struct b2_dataobj *grad;
    struct b2_dataobj *usave;
    /* != 0: free surface on the low side of the LAST dimension (reference `freesurface`,
     * examples/seismic/acoustic/operators.py:5-47, models built with fs=True): vertical taps that fall
     * above the surface read sign(z-k) * u[|z-k|] (antisymmetric mirror), and u[t+1] is cleared on the
     * surface row z = 0 before the source is injected. Needs z_m (y_m in 2-D) == 0.               */
    int free_surface;
    /* != 0: the reference's 4th-order-in-time kernel (kernel='OT4', acoustic/operators.py:50-68):
     * the Laplacian is replaced by  lap(u) + dt^2/12 * lap( lap(u) / m ).  3-D/2-D, needs
     * space_order >= 2*radius; not combined with halo exchange, free surface or the imaging condition
     * in this version (-> 210).                                                                   */
    int ot4;
    /* Linearised (Born) modelling, the reference's `Born` operator (acoustic/operators.py:235-277):
     * both non-NULL -> `born_U` (same layout as u) is stepped next to u with the extra source
     * -born_dm * u.dt2 (u.dt2 taken after `src` was injected into u[t+1]); `rec` then samples born_U
     * instead of u. `born_dm` is a space array with its own halo width (hsize). Forward only; not
     * combined with halo exchange, free surface, OT4 or the imaging condition in this version.   */
    struct b2_dataobj *born_U;
    struct b2_dataobj *born_dm;
    /* Time-subsampled snapshots (reference: `Eq(usave, u)` with usave on a ConditionalDimension of
     * `factor`, examples/seismic/tutorials/08_snapshotting.ipynb:455-505): when snap != NULL, at every
     * time step with time % snap_factor == 0 the iteration box of u[time + snap_toff] is copied into
     * snap[time / snap_factor]. `snap` is (nsnaps, x, y, z) with its own halo width (hsize); the call
     * fails with 210 if a snapshot index would fall outside it.                                  */
    struct b2_dataobj *snap;
    int snap_factor;
    int snap_toff;
    /* != 0: `u` (and `damp` / `param` when they carry both pointers) come with a host array `data` AND the caller's
     * own device buffer `dmap`: the call copies data -> dmap before and dmap -> data (u only) after the time loop —
     * overlapped with a skewed sweep when the grid is large (streamed loop). Under x-slab decomposition this lets a
     * host-staged apply use the CUDA-IPC registered device allocations of the peer-memory halo path.          */
    int host_io;
};
int b2_iso_forward(const struct b2_iso_args *a);

/* ---- the acoustic gradient with binomial checkpointing (the reference's `jacobian_adjoint(checkpointing=True)`,
 *      examples/seismic/acoustic/wavesolver.py:196-210) ------------------------------------------------------------
 * Runs the Gradient operator `grad` (adjoint != 0, with `grad`; `src` = the receiver data injected into the adjoint
 * field grad->u) while the forward operator `fwd` (adjoint 0, `src`, u buffered with 3 time slots) recomputes the
 * forward wavefield from `ncheckpoints` device checkpoints instead of reading a saved (nt, x, y, z) array: grad->usave
 * must be fwd->u (the same struct, or one with the same data, dmap and nbytes). `actions` holds `nactions` triples
 * {kind, a, b}, in absolute time indices of the two operators:
 *   B2_REVOLVE_ADVANCE  {t0, t1}: forward steps time = t0 .. t1-1 (t0 = the current forward time; the sweeps, the two-
 *                                 level pass and the injection of b2_iso_forward)
 *   B2_REVOLVE_TAKESHOT {k, t}  : copy u[t] and u[t-1] (whole allocated slots, halo included) into checkpoint k
 *                                 (t = the current forward time)
 *   B2_REVOLVE_RESTORE  {k, -}  : copy them back; the current forward time becomes t
 *   B2_REVOLVE_REVERSE  {t, -}  : one adjoint step at time t with its injection, then grad -= u[t] * v.dt2, u[t] read
 *                                 from its slot of u (t = the current forward time or the one before)
 * The reverse steps name grad->time_M down to grad->time_m, once each. The forward state at entry is fwd->time_m
 * (levels time_m and time_m-1 in u). Every array is staged once, both plans are built once and the checkpoints
 * (2 slots each) are allocated for the call and freed on return. 3-D only; a halo context, OT4, a free surface, Born,
 * snapshots, host_io or receivers (`rec`) in either block, a usave that is not fwd's u, fwd and grad that differ in
 * space order, radius, dt, vp, damp, the parameter array or the iteration box, or a malformed action list return
 * 210. errctl checks u after every forward step at a time with (time - fwd->time_m) % 100 == 99 or at the last
 * forward time the schedule reaches (again when that time is recomputed), and v on the adjoint steps as
 * b2_iso_forward does. The loop time goes to grad->timers->section0.
 * b2_last_sweep_kernel then reports the forward sweeps that ran (space-separated, in order of first use), ';', the
 * adjoint one, e.g. "iso_tma2<4,scalar> iso_tma<4,scalar>;iso_tma<4,scalar>". */
enum { B2_REVOLVE_ADVANCE = 0, B2_REVOLVE_TAKESHOT = 1, B2_REVOLVE_RESTORE = 2, B2_REVOLVE_REVERSE = 3 };
int b2_iso_gradient_revolve(const struct b2_iso_args *fwd, const struct b2_iso_args *grad, const int *actions,
                            int nactions, int ncheckpoints);
/* Host only, no device needed: 0 when `actions` is a schedule b2_iso_gradient_revolve accepts for these time ranges,
 * else 210 with the first fault in b2_last_error (out-of-range times or checkpoints, a restore of an empty
 * checkpoint, a reverse step out of order or without its forward level live, steps left unreversed). */
int b2_revolve_check(const int *actions, int nactions, int ncheckpoints, int fwd_time_m, int fwd_time_M,
                     int grad_time_m, int grad_time_M);

/* ---- TTI centred forward (replaces generated `ForwardTTI`,
 *      examples/seismic/tti/operators.py:186-247, 431-480), 2-D and 3-D ----------------------- */
struct b2_tti_args {
    int space_order;                  /* halo width of u / v                                */
    int radius;                       /* space_order/2                                      */
    const float *w2[3];               /* 2nd-derivative weights incl 1/h^2, [0..radius]     */
    const float *w1[3];               /* half-node 1st-derivative weights incl 1/h:         *
                                       * `radius` entries for offsets (-r/2+1 .. r/2) about  *
                                       * x+h/2 (devito/finite_differences/tools.py:280-308)  */
    struct b2_dataobj *u, *v;
    struct b2_dataobj *damp;
    float vp, epsilon, delta, theta, phi;
    float dt;
    int x_m, x_M, y_m, y_M, z_m, z_M;
    int time_m, time_M;
    struct b2_sparse *src;            /* injected into both u and v                         */
    struct b2_sparse *rec;            /* samples u+v                                        */
    int rec_toff;
    int errctl;
    int deviceid;
    int kernel;
    b2_halo_ctx *halo;
    struct b2_profiler *timers;
    /* array-valued parameters (preset `layers-tti`, examples/seismic/preset_models.py:210-238):
     * each NULL -> the scalar above. Same allocated layout (halo = space_order) as u. The rotation
     * factors are sampled where the reference samples them: at the Gz point inside Gz, at the
     * shifted point in the outer derivative `(Gz*cos(theta)).dz(...)` (tti/operators.py:92-102). */
    struct b2_dataobj *vp_arr, *epsilon_arr, *delta_arr, *theta_arr, *phi_arr;
    /* Linearised (Born) modelling, the reference's `BornTTI` operator (tti/operators.py:532-586): all three NULL ->
     * the forward operator above. All three non-NULL -> after (u, v) is stepped and `src` injected into it, the pair
     * (born_du, born_dv) (same layout as u) is stepped with the same sweep and the extra sources
     * -born_dm * u.dt2 (into du) and -born_dm * v.dt2 (into dv), divided by m/dt^2 + damp/dt, with u.dt2 taken after
     * the injection; `rec` then samples born_du + born_dv instead of u + v. `born_dm` is a space array with its own
     * halo width (hsize). born_du and born_dv are written back to the host when staged, born_dm is not. Not combined
     * with halo exchange in this version; a missing member of the triple, a shape mismatch or a wrong born_dm
     * extent returns 210.                                                                                 */
    struct b2_dataobj *born_du, *born_dv, *born_dm;
    /* Adjoint modelling, the reference's `AdjointTTI` operator (tti/operators.py `AdjointOperator`,
     * `kernel_centered(..., forward=False)`): != 0 -> time runs from time_M down to time_m, (u, v) play (p, r) and
     * each step writes level time-1 from H0 = Gh(e2 p + sd r), Hz = Gzz(sd p + r) (e2 = 1+2 epsilon,
     * sd = sqrt(1+2 delta) sampled at every tap point), level time and level time+1 as the previous one; `src` is
     * injected with dt^2/m into both fields at the level written, `rec` samples p + r at level time. 0 -> the
     * forward operator. Not combined with halo exchange or the Born triple in this version (210).             */
    int adjoint;
    /* The gradient, the reference's `GradientTTI` operator (tti/operators.py `JacobianAdjOperator`): with
     * `adjoint`, after each step and its injection grad -= usave[time] * p.dt2 + vsave[time] * r.dt2 over the
     * iterated box. `usave` / `vsave` are saved forward wavefields (nt, x, y, z) with the space layout of u; `grad`
     * is a space array with its own halo width (hsize), written back when staged. All NULL -> no imaging. grad
     * without usave and vsave, grad without adjoint, or a saved field whose space layout differs from u's
     * returns 210.                                                                                          */
    struct b2_dataobj *grad, *usave, *vsave;
    /* 0 or 3: a 3-D grid. 2: a 2-D grid (x, z) (the reference's `Gzz_centered_2d`, tti/operators.py): u, v are
     * (tsize, x+2so, z+2so), every space array is (x, z) with its halo, w2 / w1 / x_m..y_M carry x and z in slots 0
     * and 1 (z_m / z_M ignored), and the rotation is (sin theta, cos theta) on (x, z). A 2-D call takes no azimuth:
     * phi != 0, phi_arr != NULL or halo != NULL returns 210. kernel 0 sweeps with the single-pass k_tti2d<R> when
     * the layout qualifies (radius 2 or 4, z extent and z start multiples of 4, 16-byte aligned arrays), else with
     * the two-pass kernels; kernel 2 on a layout that does not qualify returns 210. b2_last_sweep_kernel reports
     * "tti2d<R>" / "tti2d_arr<R>" (array parameters) or "tti_two_pass", with the suffixes of the 3-D calls.    */
    int ndim;
};
int b2_tti_forward(const struct b2_tti_args *a);

/* ---- self-adjoint variable-density visco-acoustic modelling (replaces the generated `IsoFwdOperator` /
 *      `IsoAdjOperator`, examples/seismic/self_adjoint/operators.py:4-160) ------------------------------------
 * With R = radius and c_d[k-1] (k = 1..R) the weights of a first derivative at the half node, offsets -R+1 .. R
 * about x + h/2, at offset +k (the weight at offset -k+1 is -c_d[k-1]), divided by h_d:
 *   F_d(q)  = b(q) sum_k c_d[k-1] (u[t](q + k e_d) - u[t](q - (k-1) e_d))
 *   u[t+1]  = dt^2 vp^2/b * sum_d sum_k c_d[k-1] (F_d(p + (k-1) e_d) - F_d(p - k e_d))
 *             + (2 - dt w) u[t] + (dt w - 1) u[t-1]
 * b sampled at the grid nodes q, vp, b and w = damp (w/Q) at p. Then u[t+1][cell] += w.w.w * src[t][p] * dt^2 vp^2/b
 * at the cell, and rec[t][p] samples u[t + rec_toff]. With `adjoint` the same formula writes u[t-1] from u[t] and
 * u[t+1], time runs from time_M down to time_m, `src` (the receiver data) is injected into u[t-1] with the same scale
 * and `rec` (the adjoint source) samples u[t] (rec_toff 0) or u[t-1] (rec_toff != 0).
 * Not combined with halo exchange or a free surface (210). kernel 0 runs the 2.5-D TMA sweep sa_tma<R> when the
 * layout qualifies (3-D, radius 2 or 4, z extent and z start multiples of 4, 16-byte aligned arrays), else the
 * one-thread-per-point kernel; kernel 2 on a layout that does not qualify returns 210.
 * b2_last_sweep_kernel reports "sa_tma<R>" or "sa_generic", with "+adj" on adjoint calls. */
struct b2_sa_args {
    int ndim;                         /* 2 or 3                                                      */
    int space_order;                  /* halo width of u / b / vp / damp                             */
    int radius;                       /* R <= space_order/2 (the nested stencil reaches 2R-1 points)  */
    const float *c[3];                /* per-dim weights incl. 1/h: c[d][0..radius-1]                */
    struct b2_dataobj *u;             /* (tsize, x+2so, y+2so[, z+2so]); tsize 3 or nt (save=True)   */
    struct b2_dataobj *b;             /* buoyancy array, or NULL -> b_value                          */
    float b_value;
    struct b2_dataobj *vp;            /* velocity array, or NULL -> vp_value                         */
    float vp_value;
    struct b2_dataobj *damp;          /* w/Q array, or NULL -> no attenuation                        */
    float dt;
    int x_m, x_M, y_m, y_M, z_m, z_M; /* for ndim==2 the z entries are ignored                       */
    int time_m, time_M;
    struct b2_sparse *src;            /* injected into the level written                             */
    struct b2_sparse *rec;            /* samples u[t] (rec_toff 0) or the level written              */
    int rec_toff;
    int adjoint;
    int errctl;                       /* !=0: NaN check every 100 steps -> return 100                */
    int deviceid;
    int kernel;                       /* 0 auto, 1 generic, 2 TMA (210 if the layout does not take it) */
    b2_halo_ctx *halo;                /* must be NULL                                                */
    int free_surface;                 /* must be 0                                                   */
    struct b2_profiler *timers;       /* may be NULL; section0 accumulates the loop time             */
};
int b2_sa_forward(const struct b2_sa_args *a);

/* ---- second-order SLS viscoacoustic modelling (replaces the generated `ForwardOperator` / `AdjointOperator` of
 *      examples/seismic/viscoacoustic at kernel='sls', time_order=2, operators.py:124-192) ------------------------
 * With L(f) = sum_d sum_k c_d[k-1] (F_d(p + (k-1) e_d) - F_d(p - k e_d)), F_d(q) = b(q) sum_k c_d[k-1] (f(q + k e_d) -
 * f(q - (k-1) e_d)) (the nested operator of b2_sa_forward, b at the nodes), t_s = (sqrt(1 + 1/qp^2) - 1/qp) / f0,
 * tt = 1/(f0^2 t_s^2) - 1, m = 1/vp^2, rho = 1/b and damp the "mask" profile (NULL: 1):
 *   r[t+1] = damp solve(r.dt - (tt/t_s) rho L(p) + r/t_s, r[t+1])
 *   p[t+1] = damp solve(m p.dt2 - rho (1+tt) L(p) + r[t+1] + (1-damp) p.dt, p[t+1])
 * with r.dt, p.dt the first-order forward differences (f[t+1] - f[t]) / dt and .dt.T = (f[t-1] - f[t]) / dt; then p[t+1][cell] += w.w.w * src[t][p] * dt^2 vp^2 and rec[t][p] samples p[t + rec_toff].
 * With `adjoint` time runs from time_M down to time_m:
 *   r[t-1] = damp solve(r.dt.T + (tt/t_s) p + r/t_s, r[t-1])
 *   p[t-1] = damp solve(m p.dt2 - L((1+tt) rho p) - L(rho r[t-1]) + (1-damp) p.dt.T, p[t-1])
 * `src` (the receiver data) is injected into p[t-1] with the same scale and `rec` (the adjoint source) samples p[t].
 * p (`u`) and r have the same layout. Not combined with halo exchange or a free surface (210). kernel 0 runs the
 * 2.5-D TMA sweep visco_tma<R> when the layout qualifies (3-D, radius 2 or 4, z extent and z start multiples of 4,
 * 16-byte aligned arrays), else the one-thread-per-point kernel; kernel 2 on a layout that does not qualify returns
 * 210. b2_last_sweep_kernel reports "visco_tma<R>" or "visco_generic", with "+adj" on adjoint calls. */
struct b2_visco_args {
    int ndim;                         /* 2 or 3                                                      */
    int space_order;                  /* halo width of p / r / b / vp / qp / damp                    */
    int radius;                       /* R <= space_order/2 (the nested stencil reaches 2R-1 points)  */
    const float *c[3];                /* per-dim weights incl. 1/h: c[d][0..radius-1]                */
    struct b2_dataobj *u;             /* p: (tsize, x+2so, y+2so[, z+2so]); tsize 3 or nt (save=True) */
    struct b2_dataobj *r;             /* the memory variable, p's layout                             */
    struct b2_dataobj *b;             /* buoyancy array, or NULL -> b_value                          */
    float b_value;
    struct b2_dataobj *vp;            /* velocity array, or NULL -> vp_value                         */
    float vp_value;
    struct b2_dataobj *qp;            /* quality-factor array, or NULL -> qp_value                   */
    float qp_value;
    struct b2_dataobj *damp;          /* mask profile, or NULL -> 1                                  */
    float f0;                         /* reference frequency of the relaxation times                 */
    float dt;
    int x_m, x_M, y_m, y_M, z_m, z_M; /* for ndim==2 the z entries are ignored                       */
    int time_m, time_M;
    struct b2_sparse *src;            /* injected into the level written                             */
    struct b2_sparse *rec;            /* samples p[t] (rec_toff 0) or the level written              */
    int rec_toff;
    int adjoint;
    int errctl;                       /* !=0: NaN check of p and r every 100 steps -> return 100      */
    int deviceid;
    int kernel;                       /* 0 auto, 1 generic, 2 TMA (210 if the layout does not take it) */
    b2_halo_ctx *halo;                /* must be NULL                                                */
    int free_surface;                 /* must be 0                                                   */
    struct b2_profiler *timers;       /* may be NULL; section0 accumulates the loop time             */
};
int b2_visco_forward(const struct b2_visco_args *a);

/* ---- generic explicit update with constant coefficients --------------------------------------
 * Any Operator whose single equation is  f[t + wshift][p] = sum_k coef_k * f[t + tshift_k][p + off_k]
 * with coefficients that do not depend on position (Constants, spacings, dt) — e.g. the reference's
 * 2-D diffusion example `Eq(u.dt, a*(u.dx2 + u.dy2))` solved for u.forward
 * (examples/cfd/example_diffusion.py:120-133, BASELINE config 1). Replaces the generated `Kernel`
 * function of such operators. Cells outside [x_m..x_M] x ... are not written (SubDomain semantics). */
struct b2_tap {
    int tshift;                       /* time level read: t + tshift                           */
    int off[3];                       /* space offsets (unused dims 0)                          */
    float coef;
};
#define B2_MAX_TAPS 64
struct b2_linear_args {
    int ndim;                         /* 1, 2 or 3                                              */
    struct b2_dataobj *f;             /* (tsize, x[, y[, z]]) with halo                         */
    int halo;                         /* halo width of f on every space dimension               */
    int ntaps;
    const struct b2_tap *taps;
    int wshift;                       /* +1: f.forward is written, -1: f.backward               */
    int x_m, x_M, y_m, y_M, z_m, z_M;
    int time_m, time_M;
    int deviceid;
    struct b2_profiler *timers;       /* may be NULL; section0 accumulates the loop time        */
};
int b2_linear_forward(const struct b2_linear_args *a);

/* ---- generic explicit linear SYSTEM (staggered-grid schemes: elastic, TTI first-order form ...) ----------
 * The time loops the reference generates for first-order systems on staggered grids
 * (examples/seismic/elastic/operators.py:26-65 `ForwardElastic`: v.forward = damp (v + dt b div tau),
 * tau.forward = damp (tau + dt (lam diag(div v.forward) + mu (grad v.forward + grad v.forward^T)));
 * examples/seismic/tti/operators.py:280-428 staggered TTI) have one shape: per time step a sequence of
 * STAGES, each writing one field as a linear combination of shifted reads of the fields,
 *     out[t + out_tshift][p] = sum_k coef_k * C_{cfield_k}[p] * F_{field_k}[t + tshift_k][p + off_k],
 * where C_j are coefficient arrays tabulated once per call (averaged / harmonically averaged material
 * parameters times the damping mask, evaluated at the output's staggered position) and off_k are ARRAY
 * offsets (the half-cell shifts of staggered fields are already folded in). Stages run in order, so a
 * later stage may read what an earlier one wrote at t+1 (tshift = 1). After the stages of a step:
 * injections (into up to 3 fields at once: the diagonal of the stress tensor) and interpolations
 * (of a field, or of a scratch field that an extra stage filled, e.g. div(v)).
 * All fields share the grid extents and the halo width `halo`; a field with 1 time slot is scratch.
 * A stage that reads shifted points of the level it writes is refused (every level of a 1-slot field is
 * the level it writes). A stage may widen its box by `ext` cells on every space axis: a scratch field
 * that receivers sample must also hold its values on the halo cells their support reaches (the
 * interpolation guard is d_m - r <= cell <= d_M + r); such a stage may not use coefficient arrays. */
struct b2_sys_tap {
    int field;                        /* index into `fields`                                    */
    int tshift;                       /* time level read: t + tshift (0 or 1)                   */
    int off[3];                       /* array offsets                                          */
    float coef;
    int cfield;                       /* index into `coefs`, or -1                              */
};
struct b2_sys_stage {
    int out_field;
    int out_tshift;                   /* +1 for an update, 0 for a scratch field                */
    int ntaps;
    const struct b2_sys_tap *taps;
    int ext;                          /* box widened by ext cells per side (0..halo; no cfield) */
};
struct b2_sys_inject {
    struct b2_sparse *s;
    int nfields;                      /* 1..3                                                    */
    int fields[3];
    int tshift;                       /* level deposited into (normally +1)                      */
    float scale;                      /* value = scale * src[time][p] * weights [* f(param)]     */
    int param_kind;                   /* 0: none; B2_PARAM_VP: * param[cell]^2; B2_PARAM_M: / param[cell] */
    struct b2_dataobj *param;         /* space array with the fields' allocated layout, or NULL  */
};
struct b2_sys_interp {
    struct b2_sparse *s;
    int field;
    int tshift;
};
#define B2_SYS_MAX_FIELDS 24
#define B2_SYS_MAX_COEFS 48
#define B2_SYS_MAX_TAPS 160
struct b2_system_args {
    int ndim;                         /* 2 or 3                                                  */
    int halo;                         /* halo width of every field on every space dimension      */
    int nfields;
    struct b2_dataobj **fields;       /* (tsize, x, y[, z]) each                                 */
    int ncoefs;
    struct b2_dataobj **coefs;        /* (x, y[, z]) each, NO halo (values at the output points) */
    int nstages;
    const struct b2_sys_stage *stages;
    int ninject, ninterp;
    const struct b2_sys_inject *inject;
    const struct b2_sys_interp *interp;
    int x_m, x_M, y_m, y_M, z_m, z_M;
    int time_m, time_M;
    int deviceid;
    struct b2_profiler *timers;       /* section0 = stages, section1 = injection, section2 = interpolation */
};
int b2_system_forward(const struct b2_system_args *a);

/* ---- halo exchange under x-slab decomposition (replaces `haloupdate0`/`sendrecv0`,
 *      devito/mpi/routines.py:285-552; printed examples/mpi/overview.ipynb:503-560) -------- */
/* NCCL bootstrap: rank 0 calls b2_nccl_unique_id, the 128 bytes are broadcast by the host
 * framework, every rank calls b2_halo_create. `nccl_lib` = path of libnccl.so.2 (or NULL). */
int  b2_nccl_unique_id(const char *nccl_lib, char id_out[128]);
b2_halo_ctx *b2_halo_create(const char *nccl_lib, const char id[128], int rank, int nranks,
                            int deviceid);
void b2_halo_destroy(b2_halo_ctx *ctx);
/* Exchange `width` yz-planes of time slot `slot` of field `f` (device-resident) with the
 * x-neighbours: owned planes -> neighbour halo. Blocking w.r.t. the library stream. */
int  b2_halo_update(b2_halo_ctx *ctx, struct b2_dataobj *f, int slot, int width);

/* Peer-memory halo path (one process per GPU, NVLink/NVSwitch): boundary planes are stored straight
 * into the neighbour's halo through CUDA-IPC-mapped peer pointers and ordered with device-side flags
 * (st.release.sys / ld.acquire.sys) — no NCCL call per time step. The host framework exchanges the
 * 64-byte IPC handles (torch.distributed), the library does the rest.
 *   b2_ipc_get_handle / b2_ipc_open / b2_ipc_close : cudaIpc{Get,Open,Close}MemHandle wrappers
 *   b2_halo_p2p_setup    : local flag buffer (2 ints: [from left, from right]) and the two remote
 *                          flag slots this rank signals (NULL at the physical boundary)
 *   b2_halo_p2p_register : for the field whose device base is `local_base`, the neighbours' mapped
 *                          bases and the number of x-planes they own                              */
int   b2_ipc_get_handle(void *devptr, char handle_out[64]);
void *b2_ipc_open(const char handle[64]);
int   b2_ipc_close(void *mapped);
int   b2_halo_p2p_setup(b2_halo_ctx *ctx, void *flags_local, void *flag_left_remote, void *flag_right_remote);
int   b2_halo_p2p_register(b2_halo_ctx *ctx, void *local_base, void *left_base, void *right_base,
                           int n_left, int n_right);

/* ---- utilities ---------------------------------------------------------------------------- */
int         b2_device_count(void);
/* PCI bus id ("0000:3b:00.0") of a device: the host side uses it to place its pinned buffers and threads
 * on the NUMA node next to the GPU (devito_b200/numa.py). */
int         b2_device_pci_bus_id(int deviceid, char *out, int len);
const char *b2_last_error(void);
const char *b2_version(void);
/* number of kernels launched by this library since load (for bench.py `gpu_launches`) */
unsigned long long b2_launch_count(void);
/* average device time (ms) of the stencil kernel launches since the last reset, measured
 * with CUDA events on the library stream; used for bench.py `roofline.achieved`. */
void   b2_kernel_timing_reset(void);
double b2_kernel_timing_ms(int *nlaunches);
void   b2_kernel_timing_enable(int on);
/* name of the sweep kernel variant the last b2_iso_forward / b2_tti_forward call on this process launched, e.g.
 * "iso_generic", "iso_tma<4,vp>" (template radius, parameter kind scalar|vp|m), "tti_two_pass",
 * "tti_fused<2>", "tti_ws<pf1>", "tti_arr_ct2<4>" (radius); "" if the call launched none. Several kernels are
 * selected at run time (layout checks, B2_* switches): this tells which one computed the answer. A TTI Born call
 * appends the path of its source term: "+born_v4" (float4 along z) or "+born_s" (one point per thread); a TTI
 * adjoint call appends "+adj" to the variant that ran its sweep. b2_sa_forward reports "sa_tma<R>" or "sa_generic", with "+adj" on
 * adjoint calls; b2_visco_forward "visco_tma<R>" or "visco_generic", with "+adj" on adjoint calls. */
const char *b2_last_sweep_kernel(void);
/* number of x-planes of the last b2_iso_forward call whose update coefficient A = 1/(m/dt^2 + damp/dt) the
 * TMA sweep took from the one tile it pins per CTA instead of streaming it: the planes of the update box whose
 * damp equals, bit for bit over the box, the damp of the centre plane x_m + (x_M - x_m + 1)/2 (scalar vp only,
 * whole table on the device before the time loop; 0 for the streamed loop, an array vp|m and the generic
 * kernel). Reads the flags back from the device: synchronises the library stream. -1 on a device error. */
int         b2_last_iso_coef_reuse(void);
/* device memory helpers for hosts that do not use torch */
void *b2_malloc_device(unsigned long nbytes, int deviceid);
void  b2_free_device(void *p, int deviceid);
int   b2_memcpy_h2d(void *dst, const void *src, unsigned long nbytes, int deviceid);
int   b2_memcpy_d2h(void *dst, const void *src, unsigned long nbytes, int deviceid);
int   b2_memset_device(void *dst, int value, unsigned long nbytes, int deviceid);
int   b2_synchronize(int deviceid);
/* make the library enqueue its work on an externally owned CUDA stream (cudaStream_t as
 * void*); NULL -> the library's own non-blocking stream. */
void  b2_set_stream(void *stream);
/* Host-staged applies recycle their device staging buffers across calls (up to B2_STAGING_CACHE_GB,
 * default 24): release what is cached. */
void  b2_staging_cache_release(void);
/* Staging buffers that entry-point calls allocated and have not released yet: 0 between calls. */
unsigned long long b2_staging_outstanding(void);
/* Phase times (ms) of the last b2_iso_forward call on this process: [0] host->device staging issued
 * before the time loop, [1] time loop, [2] write-back after the loop (device->host copies, snapshot drain,
 * release of the staging buffers), [3] whole call (host clock);
 * [4] = 1 when the call ran the streamed (skewed, copy-overlapped) time loop. */
void  b2_last_call_profile(double out[5]);

#ifdef __cplusplus
}
#endif
#endif /* B200STENCIL_H */
