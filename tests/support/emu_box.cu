// The entry points' iteration box (make_box, check_reach in b2_common.cuh) as host code -- TEST INFRASTRUCTURE ONLY.
//
// Compiled by nvcc without a GPU; tests/test_entry_geometry.py checks the internal 3-dim convention and the reach
// rule of the wave entry points against numpy.
#include <cstdarg>
#include "b2_common.cuh"

namespace b2 {

thread_local std::string g_last_error;

void set_error(const char *fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_last_error = buf;
}

}  // namespace b2

using namespace b2;

struct BoxArgs {
    int x_m, x_M, y_m, y_M, z_m, z_M;
};

static Box box_of(const int *lo, const int *hi, int nd, const int *size, int halo) {
    const BoxArgs args = {lo[0], hi[0], lo[1], hi[1], lo[2], hi[2]};
    return make_box(&args, nd, size, halo);
}

// lo / hi: x_m, y_m, z_m / x_M, y_M, z_M (entries past nd ignored); size: time slots, then the nd space extents.
// out: a[3], n[3], o[3], sx, sy, slot_elems, tsize, so.
extern "C" void emu_make_box(const int *lo, const int *hi, int nd, const int *size, int halo, long long *out) {
    const Box b = box_of(lo, hi, nd, size, halo);
    for (int d = 0; d < 3; ++d) {
        out[d] = b.a[d];
        out[3 + d] = b.n[d];
        out[6 + d] = b.o[d];
    }
    out[9] = b.sx;
    out[10] = b.sy;
    out[11] = (long long)b.slot_elems;
    out[12] = b.tsize;
    out[13] = b.so;
}

// check_reach of that box: its return code; *empty = 1 when the call has nothing to do
extern "C" int emu_check_reach(const char *who, const int *lo, const int *hi, int nd, const int *size, int halo,
                               int reach, int *empty) {
    g_last_error.clear();
    bool e = false;
    const int rc = check_reach(who, box_of(lo, hi, nd, size, halo), nd, reach, e);
    *empty = e;
    return rc;
}

extern "C" const char *emu_last_error() { return g_last_error.c_str(); }
