/* Centred-TTI linearised (Born) modelling in the C oracle -- TEST INFRASTRUCTURE ONLY.
 *
 * The reference's `BornTTI` operator (examples/seismic/tti/operators.py:532-586) in the operation order of the code
 * it generates. It reuses the sparse-point helpers of oracle/oracle.c by including that file, and restates the TTI
 * step of `oracle_tti_forward` as a helper that can add the Born source term to the numerator. Compiled on demand by
 * tests/tti_born_ref.py into its own shared library.
 */
#include "../../oracle/oracle.c"

typedef struct {
    int R, so;
    const int *lo, *hi;
    size_t sx, sy, slot;
    const float *w2x, *w2y, *w2z, *w1x, *w1y, *w1z, *damp;
    const float *eps_a, *vp_a;
    int arrays;
    const float *tcx, *tcy, *tcz, *tsd;
    float r18s, czs, cys, cxs, e2s, r9s, r10, r11;
    float *gzu, *gzv;
    /* Born source (NULL: none): qu = -dm * u.dt2 of the background levels bu* into u, qv likewise into v */
    const float *bu1, *bu0, *bum, *bv1, *bv0, *bvm, *dm;
    size_t dsx, dsy;
    int dmhalo;
} tti_ctx;

static void tti_pair_step(const tti_ctx *c, const float *u0, const float *um, float *u1, const float *v0,
                          const float *vm, float *v1) {
    const int R = c->R, h = R / 2, so = c->so, arrays = c->arrays;
    const size_t sx = c->sx, sy = c->sy;
    const int *lo = c->lo, *hi = c->hi;
    const float *w1x = c->w1x, *w1y = c->w1y, *w1z = c->w1z, *w2x = c->w2x, *w2y = c->w2y, *w2z = c->w2z;
    const float *tcx = c->tcx, *tcy = c->tcy, *tcz = c->tcz, *tsd = c->tsd;
    const float czs = c->czs, cys = c->cys, cxs = c->cxs, r10 = c->r10, r11 = c->r11;
    float *gzu = c->gzu, *gzv = c->gzv;
#pragma omp parallel for collapse(2) schedule(static)
    for (int x = lo[0] - h; x <= hi[0] + h - 1; ++x)
        for (int y = lo[1] - h; y <= hi[1] + h - 1; ++y)
            for (int z = lo[2] - h; z <= hi[2] + h - 1; ++z) {
                const size_t i = IDX3(x + so, y + so, z + so);
                float dxu = 0, dyu = 0, dzu = 0, dxv = 0, dyv = 0, dzv = 0;
                for (int j = 0; j < R; ++j) {
                    const ptrdiff_t o = j - h + 1;
                    dxu += w1x[j] * u0[i + o * (ptrdiff_t)sx];
                    dyu += w1y[j] * u0[i + o * (ptrdiff_t)sy];
                    dzu += w1z[j] * u0[i + o];
                    dxv += w1x[j] * v0[i + o * (ptrdiff_t)sx];
                    dyv += w1y[j] * v0[i + o * (ptrdiff_t)sy];
                    dzv += w1z[j] * v0[i + o];
                }
                const float cx = arrays ? tcx[i] : cxs, cy = arrays ? tcy[i] : cys, cz = arrays ? tcz[i] : czs;
                gzu[i] = cz * dzu + cy * dyu + cx * dxu;
                gzv[i] = cz * dzv + cy * dyv + cx * dxv;
            }
#pragma omp parallel for collapse(2) schedule(static)
    for (int x = lo[0]; x <= hi[0]; ++x)
        for (int y = lo[1]; y <= hi[1]; ++y)
            for (int z = lo[2]; z <= hi[2]; ++z) {
                const size_t i = IDX3(x + so, y + so, z + so);
                float lap = (w2x[0] + w2y[0] + w2z[0]) * u0[i];
                for (int k = 1; k <= R; ++k)
                    lap += w2x[k] * (u0[i - k * sx] + u0[i + k * sx]) +
                           w2y[k] * (u0[i - k * sy] + u0[i + k * sy]) +
                           w2z[k] * (u0[i - k] + u0[i + k]);
                /* outer half-node derivatives of (r12,r13,r14) and (r15,r16,r17) */
                float H0 = 0, Hz = 0;
                const float r18 = arrays ? tsd[i] : c->r18s;
                const float e2 = c->eps_a ? 2 * c->eps_a[i] + 1 : c->e2s;
                const float r9 = c->vp_a ? 1.0f / (c->vp_a[i] * c->vp_a[i]) : c->r9s;
                for (int j = 0; j < R; ++j) {
                    const ptrdiff_t o = j - h;
                    const size_t iz = i + o, iy = i + o * (ptrdiff_t)sy, ix = i + o * (ptrdiff_t)sx;
                    const float cz = arrays ? tcz[iz] : czs, cy = arrays ? tcy[iy] : cys,
                                cx = arrays ? tcx[ix] : cxs;
                    H0 += w1z[j] * (gzv[iz] * (r18 * cz) - gzu[iz] * e2 * cz) +
                          w1x[j] * (gzv[ix] * (r18 * cx) - gzu[ix] * e2 * cx) +
                          w1y[j] * (gzv[iy] * (r18 * cy) - gzu[iy] * e2 * cy);
                    Hz += w1z[j] * (gzv[iz] * cz - gzu[iz] * (r18 * cz)) +
                          w1y[j] * (gzv[iy] * cy - gzu[iy] * (r18 * cy)) +
                          w1x[j] * (gzv[ix] * cx - gzu[ix] * (r18 * cx));
                }
                const float d = c->damp ? c->damp[i] : 0.0f;
                const float r26 = 1.0f / (r10 * r9 + r11 * d);
                if (c->dm) {
                    const size_t jd = (size_t)(x + c->dmhalo) * c->dsx + (size_t)(y + c->dmhalo) * c->dsy +
                                      (z + c->dmhalo);
                    const float qu = -c->dm[jd] * (r10 * c->bu1[i] - 2.0f * r10 * c->bu0[i] + r10 * c->bum[i]);
                    const float qv = -c->dm[jd] * (r10 * c->bv1[i] - 2.0f * r10 * c->bv0[i] + r10 * c->bvm[i]);
                    u1[i] = r26 * (e2 * lap + r10 * r9 * (2.0f * u0[i] - um[i]) + r11 * d * u0[i] + H0 + qu);
                    v1[i] = r26 * (r11 * d * v0[i] + r18 * lap - r9 * (-2.0f * r10 * v0[i] + r10 * vm[i]) + Hz + qv);
                } else {
                    u1[i] = r26 * (e2 * lap + r10 * r9 * (2.0f * u0[i] - um[i]) + r11 * d * u0[i] + H0);
                    v1[i] = r26 * (r11 * d * v0[i] + r18 * lap - r9 * (-2.0f * r10 * v0[i] + r10 * vm[i]) + Hz);
                }
            }
}

static int tti_ctx_init(tti_ctx *c, const int *alloc, int so, int radius, const float *w2x, const float *w2y,
                        const float *w2z, const float *w1x, const float *w1y, const float *w1z, const float *damp,
                        float vp, float epsilon, float delta, float theta, float phi, float dt, const int *lo,
                        const int *hi, const float *vp_a, const float *eps_a, const float *delta_a,
                        const float *theta_a, const float *phi_a) {
    /* *_a: array-valued parameters (NULL -> scalar), preset `layers-tti`. Rotation factors are
     * sampled at the Gz point inside Gz and at the shifted point in the outer derivative, exactly
     * like the reference's generated code (time-invariant tables r2..r5). */
    memset(c, 0, sizeof(*c));
    c->R = radius;
    c->so = so;
    c->lo = lo;
    c->hi = hi;
    c->sy = (size_t)alloc[2];
    c->sx = (size_t)alloc[1] * alloc[2];
    const size_t slot = c->slot = (size_t)alloc[0] * c->sx;
    c->w2x = w2x; c->w2y = w2y; c->w2z = w2z; c->w1x = w1x; c->w1y = w1y; c->w1z = w1z;
    c->damp = damp;
    c->eps_a = eps_a;
    c->vp_a = vp_a;
    c->gzu = (float *)calloc(slot, sizeof(float));
    c->gzv = (float *)calloc(slot, sizeof(float));
    if (!c->gzu || !c->gzv) return 202;
    c->arrays = vp_a || eps_a || delta_a || theta_a || phi_a;
    if (c->arrays) {
        float *tcx = (float *)malloc(slot * sizeof(float));
        float *tcy = (float *)malloc(slot * sizeof(float));
        float *tcz = (float *)malloc(slot * sizeof(float));
        float *tsd = (float *)malloc(slot * sizeof(float));
        for (size_t i = 0; i < slot; ++i) {
            const float th = theta_a ? theta_a[i] : theta, ph = phi_a ? phi_a[i] : phi;
            const float s_ = sinf(th);
            tcz[i] = cosf(th);
            tcy[i] = s_ * sinf(ph);
            tcx[i] = s_ * cosf(ph);
            tsd[i] = sqrtf(2 * (delta_a ? delta_a[i] : delta) + 1);
        }
        c->tcx = tcx; c->tcy = tcy; c->tcz = tcz; c->tsd = tsd;
    }
    c->r18s = sqrtf(2 * delta + 1);
    const float ct = cosf(theta), st = sinf(theta), sp = sinf(phi), cp = cosf(phi);
    c->czs = ct;
    c->cys = sp * st;
    c->cxs = st * cp;
    c->e2s = 2 * epsilon + 1;
    c->r9s = 1.0f / (vp * vp);
    c->r10 = 1.0f / (dt * dt);
    c->r11 = 1.0f / dt;
    return 0;
}

static void tti_ctx_free(tti_ctx *c) {
    free(c->gzu);
    free(c->gzv);
    free((void *)c->tcx); free((void *)c->tcy); free((void *)c->tcz); free((void *)c->tsd);
}


/* ------------------------------------------------------------------------------------------
 * Centred-TTI linearised (Born) modelling: the reference's `BornTTI` operator,
 * examples/seismic/tti/operators.py:532-586. Per time step, in the order of its equation list:
 *     (u, v)[t+1]   = update(u, v)                                         (eqn1)
 *     (u, v)[t+1]  += inject(src[time])                                    (source)
 *     (du, dv)[t+1] = update(du, dv) with qu = -dm * u.dt2, qv = -dm * v.dt2 in the numerators,
 *                     u.dt2 / v.dt2 taken with the levels t+1 just computed (eqn2)
 *     rec[time]     = interpolate(du[t] + dv[t])                            (receivers)
 * `dm` has its own halo width (the reference builds it with space_order 0).
 * ---------------------------------------------------------------------------------------- */
int oracle_tti_born_forward(float *u, float *v, float *du, float *dv, int tsize, const int *alloc, int so,
                            int radius, const float *w2x, const float *w2y, const float *w2z, const float *w1x,
                            const float *w1y, const float *w1z, const float *damp, float vp, float epsilon,
                            float delta, float theta, float phi, float dt, const int *lo, const int *hi, int time_m,
                            int time_M, osparse *src, osparse *rec, const float *vp_a, const float *eps_a,
                            const float *delta_a, const float *theta_a, const float *phi_a, const float *dm,
                            const int *dmalloc, int dmhalo) {
    tti_ctx c;
    if (tti_ctx_init(&c, alloc, so, radius, w2x, w2y, w2z, w1x, w1y, w1z, damp, vp, epsilon, delta, theta, phi, dt,
                     lo, hi, vp_a, eps_a, delta_a, theta_a, phi_a)) {
        tti_ctx_free(&c);
        return 202;
    }
    const size_t sx = c.sx, sy = c.sy, slot = c.slot;
    for (int time = time_m; time <= time_M; ++time) {
        const int t0 = ((time % tsize) + tsize) % tsize;
        const int t1 = (((time + 1) % tsize) + tsize) % tsize;
        const int t2 = (((time - 1) % tsize) + tsize) % tsize;
        float *u1 = u + (size_t)t1 * slot, *v1 = v + (size_t)t1 * slot;
        c.dm = NULL;
        tti_pair_step(&c, u + (size_t)t0 * slot, u + (size_t)t2 * slot, u1, v + (size_t)t0 * slot,
                      v + (size_t)t2 * slot, v1);
        inject(src, 3, u1, v1, sx, sy, so, lo, hi, time, vp_a ? 1 : 0, vp_a, vp, dt);
        c.dm = dm;
        c.dsy = (size_t)dmalloc[2];
        c.dsx = (size_t)dmalloc[1] * dmalloc[2];
        c.dmhalo = dmhalo;
        c.bu1 = u1; c.bu0 = u + (size_t)t0 * slot; c.bum = u + (size_t)t2 * slot;
        c.bv1 = v1; c.bv0 = v + (size_t)t0 * slot; c.bvm = v + (size_t)t2 * slot;
        tti_pair_step(&c, du + (size_t)t0 * slot, du + (size_t)t2 * slot, du + (size_t)t1 * slot,
                      dv + (size_t)t0 * slot, dv + (size_t)t2 * slot, dv + (size_t)t1 * slot);
        interp(rec, 3, du + (size_t)t0 * slot, dv + (size_t)t0 * slot, sx, sy, so, lo, hi, time);
    }
    tti_ctx_free(&c);
    return 0;
}
