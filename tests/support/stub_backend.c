/*
 * Test double for libb200stencil.so — TEST INFRASTRUCTURE ONLY (tests/test_zz_cinterface.py,
 * tests/test_entry_marshalling.py).
 *
 * It exports b2_iso_forward / b2_tti_forward / b2_sa_forward with the real signatures but computes NOTHING.
 * Each call keeps two records of the argument block it received:
 *  - `*_seen`: the block itself, pointers as the caller passed them (weights and sparse tables copied), so that
 *    a test can check WHICH of its objects the adapter written by `Operator.cinterface()` handed over;
 *  - `*_deep`: the block with every dataobj and sparse table copied BY VALUE (data, size, hsize, dmap), so that
 *    a test can compare what two callers passed after their own structs are gone.
 * Then, as a computed result would, it writes the call count into the first element of a host-staged `u`.
 */
#include <stdlib.h>
#include <string.h>
#include "b200stencil.h"

static struct b2_iso_args iso_seen, iso_deep;
static struct b2_tti_args tti_seen, tti_deep;
static struct b2_sa_args sa_seen, sa_deep;
static struct b2_sparse src_seen, rec_seen;
static float w_seen[6][16];
static int calls = 0;
static int next_rc = 0;

/* every allocation of the last deep record, released at the next call */
static void *owned[512];
static int nowned = 0;

static void *own(size_t n) {
    void *p = calloc(1, n ? n : 1);
    owned[nowned++] = p;
    return p;
}

static void release_owned(void) {
    for (int i = 0; i < nowned; ++i) free(owned[i]);
    nowned = 0;
}

static struct b2_dataobj *deep_obj(const struct b2_dataobj *o, int rank) {
    if (!o) return 0;
    struct b2_dataobj *c = own(sizeof(*c));
    c->nbytes = o->nbytes;
    c->dmap = o->dmap;
    /* zero-terminated: a reader finds the rank as the first 0 extent */
    c->size = own(sizeof(int) * 8);
    memcpy(c->size, o->size, sizeof(int) * rank);
    if (o->hsize) {
        c->hsize = own(sizeof(int) * 16);
        memcpy(c->hsize, o->hsize, sizeof(int) * 2 * rank);
    }
    if (o->data) {
        c->data = own(o->nbytes);
        memcpy(c->data, o->data, o->nbytes);
    }
    return c;
}

static struct b2_sparse *deep_sparse(const struct b2_sparse *s) {
    if (!s) return 0;
    struct b2_sparse *c = own(sizeof(*c));
    *c = *s;
    c->data = deep_obj(s->data, 2);
    c->gp = deep_obj(s->gp, 2);
    for (int d = 0; d < 3; ++d) c->w[d] = deep_obj(s->w[d], 2);
    return c;
}

/* weights by value: n entries of each of the k arrays */
static void deep_weights(const float **w, int k, int n) {
    for (int d = 0; d < k; ++d) {
        float *c = own(sizeof(float) * n);
        memcpy(c, w[d], sizeof(float) * n);
        w[d] = c;
    }
}

static void keep_sparse(struct b2_sparse **slot, struct b2_sparse *copy) {
    if (*slot) {
        *copy = **slot;
        *slot = copy;
    }
}

static void fill_timers(struct b2_profiler *t) {
    if (!t) return;
    t->section0 += 1.5;
    t->section1 += 0.25;
    t->section2 += 0.125;
}

static void mark_u(struct b2_dataobj *u) {
    if (u && u->data && !u->dmap) ((float *)u->data)[0] = (float)calls;
}

int b2_iso_forward(const struct b2_iso_args *a) {
    const int nd = a->ndim;
    release_owned();
    iso_deep = *a;
    deep_weights(iso_deep.w, nd, a->radius + 1);
    iso_deep.u = deep_obj(a->u, nd + 1);
    iso_deep.damp = deep_obj(a->damp, nd);
    iso_deep.param = deep_obj(a->param, nd);
    iso_deep.grad = deep_obj(a->grad, nd);
    iso_deep.usave = deep_obj(a->usave, nd + 1);
    iso_deep.born_U = deep_obj(a->born_U, nd + 1);
    iso_deep.born_dm = deep_obj(a->born_dm, nd);
    iso_deep.snap = deep_obj(a->snap, nd + 1);
    iso_deep.src = deep_sparse(a->src);
    iso_deep.rec = deep_sparse(a->rec);
    iso_deep.timers = 0;
    iso_seen = *a;
    for (int d = 0; d < nd; ++d) {
        memcpy(w_seen[d], a->w[d], sizeof(float) * (a->radius + 1));
        iso_seen.w[d] = w_seen[d];
    }
    keep_sparse(&iso_seen.src, &src_seen);
    keep_sparse(&iso_seen.rec, &rec_seen);
    fill_timers(a->timers);
    iso_seen.timers = 0;
    ++calls;
    mark_u(a->u);
    return next_rc;
}

int b2_tti_forward(const struct b2_tti_args *a) {
    release_owned();
    tti_deep = *a;
    deep_weights(tti_deep.w2, 3, a->radius + 1);
    deep_weights(tti_deep.w1, 3, a->radius);
    tti_deep.u = deep_obj(a->u, 4);
    tti_deep.v = deep_obj(a->v, 4);
    tti_deep.damp = deep_obj(a->damp, 3);
    tti_deep.vp_arr = deep_obj(a->vp_arr, 3);
    tti_deep.epsilon_arr = deep_obj(a->epsilon_arr, 3);
    tti_deep.delta_arr = deep_obj(a->delta_arr, 3);
    tti_deep.theta_arr = deep_obj(a->theta_arr, 3);
    tti_deep.phi_arr = deep_obj(a->phi_arr, 3);
    tti_deep.born_du = deep_obj(a->born_du, 4);
    tti_deep.born_dv = deep_obj(a->born_dv, 4);
    tti_deep.born_dm = deep_obj(a->born_dm, 3);
    tti_deep.grad = deep_obj(a->grad, 3);
    tti_deep.usave = deep_obj(a->usave, 4);
    tti_deep.vsave = deep_obj(a->vsave, 4);
    tti_deep.src = deep_sparse(a->src);
    tti_deep.rec = deep_sparse(a->rec);
    tti_deep.timers = 0;
    tti_seen = *a;
    for (int d = 0; d < 3; ++d) {
        memcpy(w_seen[d], a->w2[d], sizeof(float) * (a->radius + 1));
        memcpy(w_seen[3 + d], a->w1[d], sizeof(float) * a->radius);
        tti_seen.w2[d] = w_seen[d];
        tti_seen.w1[d] = w_seen[3 + d];
    }
    keep_sparse(&tti_seen.src, &src_seen);
    keep_sparse(&tti_seen.rec, &rec_seen);
    fill_timers(a->timers);
    tti_seen.timers = 0;
    ++calls;
    mark_u(a->u);
    return next_rc;
}

int b2_sa_forward(const struct b2_sa_args *a) {
    const int nd = a->ndim;
    release_owned();
    sa_deep = *a;
    deep_weights(sa_deep.c, nd, a->radius);
    sa_deep.u = deep_obj(a->u, nd + 1);
    sa_deep.b = deep_obj(a->b, nd);
    sa_deep.vp = deep_obj(a->vp, nd);
    sa_deep.damp = deep_obj(a->damp, nd);
    sa_deep.src = deep_sparse(a->src);
    sa_deep.rec = deep_sparse(a->rec);
    sa_deep.timers = 0;
    sa_seen = *a;
    for (int d = 0; d < nd; ++d) {
        memcpy(w_seen[d], a->c[d], sizeof(float) * a->radius);
        sa_seen.c[d] = w_seen[d];
    }
    keep_sparse(&sa_seen.src, &src_seen);
    keep_sparse(&sa_seen.rec, &rec_seen);
    fill_timers(a->timers);
    sa_seen.timers = 0;
    ++calls;
    mark_u(a->u);
    return next_rc;
}

const struct b2_iso_args *stub_iso_seen(void) { return &iso_seen; }
const struct b2_tti_args *stub_tti_seen(void) { return &tti_seen; }
const struct b2_sa_args *stub_sa_seen(void) { return &sa_seen; }
const struct b2_iso_args *stub_iso_deep(void) { return &iso_deep; }
const struct b2_tti_args *stub_tti_deep(void) { return &tti_deep; }
const struct b2_sa_args *stub_sa_deep(void) { return &sa_deep; }
int stub_calls(void) { return calls; }
void stub_set_rc(int rc) { next_rc = rc; }
