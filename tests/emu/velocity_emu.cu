// Host build of the velocity fix (gypsum_b200/csrc/velocity_core.cuh) and the satellite velocity
// (orbit_core.cuh orbit_velocity), for tests/test_velocity_cpu.py and tests/test_gpu_velocity.py.  Built with nvcc for the
// host only; no device code runs.
#include <cstddef>

#include "../../gypsum_b200/csrc/velocity_core.cuh"
#include "../../include/gypsum_b200.h"

using namespace gb;

static_assert(sizeof(gb200_velocity_fix) == sizeof(VelocityRecord), "ABI and device velocity fixes must match");

namespace {
struct HostRows {  // velocity_compute's rows: n rows of (x, y, z, vx, vy, vz, drift, doppler)
    const double* p;
    int n;
    template <class F>
    GB_HD void operator()(F&& fn) const {
        for (int i = 0; i < n; ++i) {
            const double* r = p + 8 * i;
            fn(i, VelocityRow{r[0], r[1], r[2], r[3], r[4], r[5], r[6], r[7]});
        }
    }
};
}  // namespace

extern "C" {
// orbit_velocity: params[26] in OrbitalParameterType order at time of week tow -> out[4] = vx, vy, vz, drift.
void velocity_emu_satellite(const double* params, double tow, double* out) {
    orbit_velocity(params, tow, out[0], out[1], out[2], out[3]);
}
// The record of one millisecond whose fix is solved at (x, y, z), as k_velocity_fixes computes it from rows [n][8].
int velocity_emu_compute(const double* rows, int n, double rx, double x, double y, double z, VelocityRecord* out) {
    velocity_record_clear(*out, rx);
    velocity_compute(HostRows{rows, n}, n, x, y, z, *out);
    return out->status;
}
// velocity_geodetic: out[3] = latitude (degrees), longitude (degrees), height (m).
void velocity_emu_geodetic(double x, double y, double z, double* out) {
    double c, s, cl, sl;
    velocity_geodetic(x, y, z, out[0], out[1], out[2], c, s, cl, sl);
}
// offsets of gb200_velocity_fix's fields as the C++ compiler lays them out
void velocity_emu_layout(long long* out /*[18]*/) {
    out[0] = offsetof(gb200_velocity_fix, receiver_timestamp);
    out[1] = offsetof(gb200_velocity_fix, vx);
    out[2] = offsetof(gb200_velocity_fix, vy);
    out[3] = offsetof(gb200_velocity_fix, vz);
    out[4] = offsetof(gb200_velocity_fix, clock_drift);
    out[5] = offsetof(gb200_velocity_fix, latitude_deg);
    out[6] = offsetof(gb200_velocity_fix, longitude_deg);
    out[7] = offsetof(gb200_velocity_fix, height);
    out[8] = offsetof(gb200_velocity_fix, gdop);
    out[9] = offsetof(gb200_velocity_fix, pdop);
    out[10] = offsetof(gb200_velocity_fix, hdop);
    out[11] = offsetof(gb200_velocity_fix, vdop);
    out[12] = offsetof(gb200_velocity_fix, tdop);
    out[13] = offsetof(gb200_velocity_fix, residual_rms);
    out[14] = offsetof(gb200_velocity_fix, status);
    out[15] = offsetof(gb200_velocity_fix, n_rows);
    out[16] = offsetof(gb200_velocity_fix, reserved);
    out[17] = sizeof(gb200_velocity_fix);
}
}
