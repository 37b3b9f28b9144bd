// Host build of the position fix, both solver modes (gypsum_b200/csrc/fix_core.cuh), for tests/fix_support.py, which the
// position-fix tests on the CPU and the GPU share.  Built with nvcc for the host only; no device code runs.
#include <cstddef>

#include "../../gypsum_b200/csrc/fix_core.cuh"
#include "../../include/gypsum_b200.h"

using namespace gb;

static_assert(sizeof(gb200_position_fix) == sizeof(FixRecord), "ABI and device position fixes must match");

namespace {
struct HostRows {  // fix_compute_lsq's rows: n rows of (tow, x, y, z)
    const double* p;
    int n;
    template <class F>
    GB_HD void operator()(F&& fn) const {
        for (int i = 0; i < n; ++i) fn(i, FixRow{p[4 * i], p[4 * i + 1], p[4 * i + 2], p[4 * i + 3]});
    }
};
}  // namespace

extern "C" {
// F_m: rows [n][4] of (tow, x, y, z), n >= 4, at receiver timestamp rx from the entering slide, as the device computes
// it (4 rows: fix_compute, in either solver mode; more: fix_compute_lsq).  Fills *out (slide_in, slide_out, the first
// four pseudoranges and the solution) and returns its status (1 solved, 2 the reference raises).
int fix_emu_compute_n(const double* rows, int n, double rx, double slide, FixRecord* out) {
    fix_record_clear(*out, rx);
    if (n == kFixRows) {
        FixRow r[kFixRows];
        for (int i = 0; i < kFixRows; ++i) r[i] = FixRow{rows[4 * i], rows[4 * i + 1], rows[4 * i + 2], rows[4 * i + 3]};
        out->status = fix_compute(r, rx, slide, *out);
    } else {
        out->status = fix_compute_lsq(HostRows{rows, n}, n, rx, slide, *out);
    }
    return out->status;
}
// offsets of gb200_position_fix's fields as the C++ compiler lays them out
void fix_emu_layout(long long* out /*[12]*/) {
    out[0] = offsetof(gb200_position_fix, receiver_timestamp);
    out[1] = offsetof(gb200_position_fix, slide_in);
    out[2] = offsetof(gb200_position_fix, slide_out);
    out[3] = offsetof(gb200_position_fix, clock_bias);
    out[4] = offsetof(gb200_position_fix, x);
    out[5] = offsetof(gb200_position_fix, y);
    out[6] = offsetof(gb200_position_fix, z);
    out[7] = offsetof(gb200_position_fix, pseudorange);
    out[8] = offsetof(gb200_position_fix, status);
    out[9] = offsetof(gb200_position_fix, n_ready);
    out[10] = offsetof(gb200_position_fix, channel);
    out[11] = sizeof(gb200_position_fix);
}
}
