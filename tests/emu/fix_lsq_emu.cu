// Host build of the position fix's least-squares mode (gypsum_b200/csrc/fix_core.cuh), for tests/test_fix_lsq_cpu.py and
// tests/test_gpu_fix_lsq.py.  Built with nvcc for the host only; no device code runs.
#include "../../gypsum_b200/csrc/fix_core.cuh"

using namespace gb;

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
// The fix of one millisecond in the least-squares mode: rows [n][4] of (tow, x, y, z), n >= 4, at receiver timestamp
// rx from the entering slide, as the device computes it (4 rows: fix_compute, more: fix_compute_lsq).  Fills *out
// (slide_in, slide_out, the first four pseudoranges and the solution) and returns its status (1 solved, 2 raised).
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
}
