// The receiver's velocity and clock drift, its geodetic position and the dilution of precision of a solved position
// fix, from each row's tracker Doppler and its satellite's velocity and clock drift (orbit_velocity).  Host/device code:
// velocity.cu runs it on the device, tests/emu/velocity_emu.cu on the host.
//
// Row i of the velocity solve is the range-rate equation linearised at the fix position r: with the line of sight
// u_i = (s_i - r) / |s_i - r| and the measured range rate rho'_i = -(c / f_L1) f_i (the recordings are baseband and a
// positive Doppler is a closing satellite),
//     -u_i . v_r + c b' = rho'_i - u_i . v_s,i + c b'_sv,i,
// with unknowns the receiver's ECEF velocity v_r and its clock drift b' (s/s), solved as c b' in m/s so that the columns
// are alike in scale.  It is linear: one least-squares solve, by the streaming Givens triangle of the fix (fix_lsq_add /
// fix_lsq_solve, which also judges rank < 4 as np.linalg.lstsq does), over any number of rows >= 4.  The frame is the fix's:
// ECEF at the time of the fix, with no Sagnac term.  The rows [-u_i, 1] are those of the DOP matrix G, so
// Q = (G^T G)^-1 = R^-1 R^-T comes from the same triangle, rotated into east/north/up at the geodetic position.
//
// The arithmetic is written with o_add / o_sub / o_mul, IEEE sqrt and division, as fix_core.cuh is, so the host and
// device builds of the solve agree bit for bit; the satellite velocity (sin, cos, atan2) and the geodetic latitude and
// longitude (atan2) can round differently between the host's libm and the device's.
#pragma once
#include <math.h>

#include "fix_core.cuh"

namespace gb {

constexpr double kL1Hz = 1575.42e6;
constexpr double kWgs84A = 6378137.0;
constexpr double kWgs84F = 1.0 / 298.257223563;
constexpr double kWgs84B = kWgs84A * (1.0 - kWgs84F);
constexpr double kWgs84E2 = kWgs84F * (2.0 - kWgs84F);             // first eccentricity squared
constexpr double kWgs84Ep2 = kWgs84E2 / (1.0 - kWgs84E2);          // second eccentricity squared
constexpr double kRadToDeg = 57.295779513082320876798154814105;   // 180 / pi
constexpr int kGeodeticIterations = 4;

// gb200_velocity_fix.status
enum VelocityStatus {
    kVelNone = 0,        // no solved position fix at this millisecond: every number is NaN
    kVelSolved = 1,      // everything set (residual_rms only with more than four rows)
    kVelUnsolvable = 2,  // rank < 4, a non-finite row, or rows the fix call's order no longer gives: velocity and DOP
                         // are NaN, the geodetic position is set
};

struct VelocityRecord {  // mirrors include/gypsum_b200.h gb200_velocity_fix, 128 bytes
    double receiver_timestamp;
    double vx, vy, vz;  // ECEF m/s
    double clock_drift;  // s/s
    double latitude_deg, longitude_deg, height;  // WGS-84, degrees and metres
    double gdop, pdop, hdop, vdop, tdop;
    double residual_rms;  // m/s, more than four rows only
    int status;
    int n_rows;
    int reserved[2];
};
static_assert(sizeof(VelocityRecord) == 128, "velocity fix must stay 128 bytes");

// One row: the observation's satellite position, the satellite's velocity and clock drift at that time of week and the
// channel's tracker Doppler at that millisecond.
struct VelocityRow {
    double x, y, z;
    double vx, vy, vz, drift;
    double doppler;  // Hz
};

// A row takes part when its satellite is ready for the fix: flags 2 and 4, the predicate of k_fix_plan.
GB_HD GB_INLINE bool velocity_row_ready(int flags) {
    return (flags & (kObsComplete | kObsFixGate)) == (kObsComplete | kObsFixGate);
}

GB_HD inline void velocity_record_clear(VelocityRecord& v, double receiver_timestamp) {
    v.receiver_timestamp = receiver_timestamp;
    v.vx = v.vy = v.vz = v.clock_drift = NAN;
    v.latitude_deg = v.longitude_deg = v.height = NAN;
    v.gdop = v.pdop = v.hdop = v.vdop = v.tdop = v.residual_rms = NAN;
    v.status = kVelNone;
    v.n_rows = 0;
    v.reserved[0] = v.reserved[1] = 0;
}

// (x, y) / |(x, y)| without overflow or underflow; (1, 0) for the zero vector.
GB_HD GB_INLINE void velocity_unit(double x, double y, double& c, double& s) {
    const double m = fmax(fabs(x), fabs(y));
    if (!(m > 0.0)) {
        c = 1.0;
        s = 0.0;
        return;
    }
    const double xs = x / m, ys = y / m;
    const double h = sqrt(o_add(o_mul(xs, xs), o_mul(ys, ys)));
    c = xs / h;
    s = ys / h;
}

// ECEF -> WGS-84 geodetic, by Bowring's iteration on the parametric latitude beta (tan beta = (1 - f) tan phi), carried
// as unit vectors so that only the final angles need atan2.  Four iterations converge to rounding for heights from
// -10 km to +100 km.  Every finite point gives a finite result: on the axis (p = 0) the latitude is +-90 degrees, and
// inside the evolute near the centre (more than 6300 km below the surface) the latitude is clamped to the equator side.
// Also returns the latitude's and longitude's cosines and sines for the local east/north/up frame.
GB_HD inline void velocity_geodetic(double x, double y, double z, double& lat_deg, double& lon_deg, double& h, double& cphi,
                                    double& sphi, double& clam, double& slam) {
    velocity_unit(x, y, clam, slam);
    const double p = o_add(o_mul(x, clam), o_mul(y, slam));  // sqrt(x^2 + y^2), without overflow
    double cb, sb;
    velocity_unit(o_mul(1.0 - kWgs84F, p), z, cb, sb);
    double px = 0.0, pz = 0.0;
    for (int i = 0; i < kGeodeticIterations; ++i) {
        px = fmax(o_sub(p, o_mul(kWgs84E2 * kWgs84A, o_mul(o_mul(cb, cb), cb))), 0.0);
        pz = o_add(z, o_mul(kWgs84Ep2 * kWgs84B, o_mul(o_mul(sb, sb), sb)));
        velocity_unit(px, pz, cphi, sphi);
        velocity_unit(cphi, o_mul(1.0 - kWgs84F, sphi), cb, sb);
    }
    // h = p cos phi + z sin phi - a^2 / N, N = a / sqrt(1 - e^2 sin^2 phi) the prime-vertical radius: exact on the axis too
    const double w = sqrt(o_sub(1.0, o_mul(kWgs84E2, o_mul(sphi, sphi))));
    h = o_sub(o_add(o_mul(p, cphi), o_mul(z, sphi)), o_mul(kWgs84A, w));
    lat_deg = o_mul(atan2(sphi, cphi), kRadToDeg);
    lon_deg = o_mul(atan2(slam, clam), kRadToDeg);
}

// One row of the system at the fix position (rx, ry, rz): [-u, 1] and the right-hand side.  False where an input is
// not finite or the satellite sits on the fix position.
GB_HD GB_INLINE bool velocity_row(const VelocityRow& w, double rx, double ry, double rz, double a[kFixRows], double& b) {
    const double dx = o_sub(w.x, rx), dy = o_sub(w.y, ry), dz = o_sub(w.z, rz);
    const double d = sqrt(o_add(o_add(o_mul(dx, dx), o_mul(dy, dy)), o_mul(dz, dz)));
    const double ux = dx / d, uy = dy / d, uz = dz / d;
    const double rate = o_mul(-(kSpeedOfLight / kL1Hz), w.doppler);  // measured range rate, m/s
    const double usv = o_add(o_add(o_mul(ux, w.vx), o_mul(uy, w.vy)), o_mul(uz, w.vz));
    a[0] = -ux;
    a[1] = -uy;
    a[2] = -uz;
    a[3] = 1.0;
    b = o_add(o_sub(rate, usv), o_mul(kSpeedOfLight, w.drift));
    return isfinite(b) && isfinite(ux) && isfinite(uy) && isfinite(uz);
}

// The velocity record of one millisecond whose fix is solved at (rx, ry, rz), over n >= 4 rows.  rows(fn) calls
// fn(i, VelocityRow) for i = 0..n-1; it runs twice (the solve, then the residuals), so the rows are read again rather
// than kept.  Fills everything but receiver_timestamp.
template <class Rows>
GB_HD inline void velocity_compute(const Rows& rows, int n, double rx, double ry, double rz, VelocityRecord& v) {
    double cphi, sphi, clam, slam;
    velocity_geodetic(rx, ry, rz, v.latitude_deg, v.longitude_deg, v.height, cphi, sphi, clam, slam);
    v.n_rows = n;
    v.status = kVelUnsolvable;
    FixLsq s;
    fix_lsq_clear(s);
    bool finite = true;
    rows([&](int, const VelocityRow& w) {
        double a[kFixRows], b;
        finite = velocity_row(w, rx, ry, rz, a, b) && finite;
        fix_lsq_add(s, a, b);
    });
    double x[kFixRows];
    if (!finite || n < kFixRows || !fix_lsq_solve(s, n, x)) return;
    v.vx = x[0];
    v.vy = x[1];
    v.vz = x[2];
    v.clock_drift = x[3] / kSpeedOfLight;
    if (n > kFixRows) {
        double ss = 0.0;
        rows([&](int, const VelocityRow& w) {
            double a[kFixRows], b;
            velocity_row(w, rx, ry, rz, a, b);
            const double r = o_sub(b, o_add(o_add(o_add(o_mul(a[0], x[0]), o_mul(a[1], x[1])), o_mul(a[2], x[2])), x[3]));
            ss = o_add(ss, o_mul(r, r));
        });
        v.residual_rms = sqrt(ss / static_cast<double>(n));
    }
    // Q = R^-1 R^-T: t = R^-1 (upper triangular) by back-substitution, column by column
    double t[kFixRows][kFixRows];
#pragma unroll
    for (int j = 0; j < kFixRows; ++j) {
#pragma unroll
        for (int i = kFixRows - 1; i >= 0; --i) {
            if (i > j) {
                t[i][j] = 0.0;
                continue;
            }
            double acc = i == j ? 1.0 : 0.0;
#pragma unroll
            for (int k = i + 1; k <= j; ++k) acc = o_sub(acc, o_mul(s.r[i][k], t[k][j]));
            t[i][j] = acc / s.r[i][i];
        }
    }
    double q[kFixRows][kFixRows];
#pragma unroll
    for (int i = 0; i < kFixRows; ++i)
#pragma unroll
        for (int j = 0; j < kFixRows; ++j) {
            double acc = 0.0;
#pragma unroll
            for (int k = 0; k < kFixRows; ++k) acc = o_add(acc, o_mul(t[i][k], t[j][k]));
            q[i][j] = acc;
        }
    // the position block in east / north / up: d^T Q d for each unit direction d
    const double e[3] = {-slam, clam, 0.0};
    const double nn[3] = {-o_mul(sphi, clam), -o_mul(sphi, slam), cphi};
    const double u[3] = {o_mul(cphi, clam), o_mul(cphi, slam), sphi};
    auto quad = [&](const double* d) {
        double acc = 0.0;
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) acc = o_add(acc, o_mul(o_mul(d[i], q[i][j]), d[j]));
        return acc;
    };
    const double qe = quad(e), qn = quad(nn), qu = quad(u);
    const double qp = o_add(o_add(q[0][0], q[1][1]), q[2][2]);
    v.pdop = sqrt(qp);
    v.tdop = sqrt(q[3][3]);
    v.gdop = sqrt(o_add(qp, q[3][3]));
    v.hdop = sqrt(o_add(qe, qn));
    v.vdop = sqrt(qu);
    v.status = kVelSolved;
}

}  // namespace gb
