// The world model's position fix (reference gypsum/world_model.py:489-633, called every millisecond by receiver.py:137)
// from four satellites' times of week and ECEF positions (orbit_core.cuh).  Host/device code: fix.cu runs it on the
// device, tests/emu/fix_emu.cu on the host.
//
// _compute_position runs 5 rounds.  Each round takes the pseudorange (slide + receiver_timestamp) - tow of every row,
// runs 20 Newton iterations on the squared-range residuals from the guess the last round left, and then subtracts the
// guess's clock bias from the receiver's clock slide.  The arithmetic is written with o_add / o_sub / o_mul (no fused
// multiply-add contraction) in the reference's order of operations; np.linalg.solve is Gaussian elimination with partial
// pivoting, the kind of solve LAPACK's dgesv does, with IEEE division.  It cannot round as OpenBLAS does, so parity with
// the reference is a bound (DESIGN.md §6), while the host and device builds of this file agree bit for bit.
//
// The least-squares mode (gb200_tracker_set_fix_solver) solves where the reference raises, with five or more ready
// rows: the same rounds, iterations and squared-range system over all N rows, each step the least-squares solution of
// J v = -r (Gauss-Newton, what np.linalg.lstsq(J, -r) gives in place of solve).  Each row of [J | -r] is rotated into
// a 4x4 upper triangle and a 4-vector by Givens rotations as it is read, so the solve keeps no per-row storage, and
// back-substitution gives v.  The normal equations J^T J are no option: the clock column (2 c^2 dt) is about 1e8 times
// the position columns (2 dx), and J^T J would square a condition number already near 1e8-1e9.  numpy's lstsq is an
// SVD (LAPACK gelsd) and rounds differently, so parity with numpy is a bound here too (DESIGN.md §8c); the host and
// device builds agree bit for bit (o_add / o_mul, IEEE sqrt and division).  Exactly four rows take fix_compute.
#pragma once
#include <math.h>

#include "orbit_core.cuh"

namespace gb {

constexpr double kSpeedOfLight = 2.99792458e8;                 // constants.py:35
constexpr double kSpeedOfLight2 = kSpeedOfLight * kSpeedOfLight;  // math.pow(SPEED_OF_LIGHT, 2), correctly rounded
constexpr int kFixRounds = 5;                                   // world_model.py:606
constexpr int kFixIterations = 20;                              // :540
constexpr int kFixRows = 4;

// gb200_position_fix.status
enum FixStatus {
    kFixNone = 0,     // fewer than 4 satellites ready, or no clock slide yet
    kFixSolved = 1,   // the solution of _compute_position
    kFixRaised = 2,   // the reference raises here (5 or more ready, or an exactly singular system); in the
                      // least-squares mode: an exactly singular 4-row system or a rank-deficient one of 5 or more
    kFixStopped = 3,  // the receiver stopped at or before this millisecond
};

// gb200_tracker_set_fix_solver
enum FixSolver {
    kFixSolverReference = 0,     // the reference: 5 or more ready raises
    kFixSolverLeastSquares = 1,  // 5 or more ready: the least-squares fix (fix_compute_lsq)
};

struct FixRecord {  // mirrors include/gypsum_b200.h gb200_position_fix, 112 bytes
    double receiver_timestamp;
    double slide_in, slide_out;  // receiver_clock_slide entering _compute_position and after it
    double clock_bias, x, y, z;  // the ReceiverSolution
    double pseudorange[kFixRows];  // round 0's get_pseudorange_for_satellite of each row
    int status;
    int n_ready;
    int channel[kFixRows];  // the rows, in the world model's order; -1 where unused
};
static_assert(sizeof(FixRecord) == 112, "position fix must stay 112 bytes");

struct FixRow {
    double tow, x, y, z;  // gb200_sv_observation's time of week and position
};

// One receiver's state across calls (the first four fields), and what one call's kernels hand each other.
struct FixBank {
    double slide;  // receiver_clock_slide, when has_slide
    int has_slide;
    int stopped;       // the reference's receiver has raised: no fix any more
    int n_touched;     // satellites in the world model (ranked)
    int n_touched_before;  // of them, ranked before this call
    int first_raise;   // first status-2 millisecond of the call (n_ms: none)
    int last_fix;      // last status-1 / 2 millisecond (-1: none)
    int last_reset;    // last millisecond whose subframes reset the slide (-1: none)
    int stop_frozen;   // a decoder raise stopped the receiver in this call
    double reset_slide;  // the slide after last_reset (or entering the call)
    int reset_has;
    int first_miss;    // first millisecond whose fix broke the two passes' chain check (n_ms: none)
    long long n_repaired;  // fixes the serial repair recomputed, over all calls
};

// The chain check of the two passes: two slides agree to 4 units in the last place.  The slides a fix leaves from
// the two entering slides of the passes are measured to be identical (DESIGN.md §8c).
GB_HD GB_INLINE bool fix_same_slide(double a, double b) { return fabs(a - b) <= 4.0 * 0x1p-52 * fabs(b); }

GB_HD inline void fix_record_clear(FixRecord& f, double receiver_timestamp) {
    f.receiver_timestamp = receiver_timestamp;
    f.slide_in = f.slide_out = f.clock_bias = f.x = f.y = f.z = NAN;
    for (int i = 0; i < kFixRows; ++i) f.pseudorange[i] = NAN, f.channel[i] = -1;
    f.status = kFixNone;
    f.n_ready = 0;
}

// One row of the system at pseudorange t: its negated residual and its Jacobian row.
GB_HD GB_INLINE void fix_row(const FixRow& r, double t, double gx, double gy, double gz, double cb, double a[kFixRows],
                             double& rhs) {
    const double dx = o_sub(gx, r.x), dy = o_sub(gy, r.y), dz = o_sub(gz, r.z);
    const double dt = o_sub(t, cb);
    const double ct = o_mul(kSpeedOfLight, dt);
    rhs = -o_sub(o_add(o_add(o_mul(dx, dx), o_mul(dy, dy)), o_mul(dz, dz)), o_mul(ct, ct));
    a[0] = o_mul(2.0, dx);
    a[1] = o_mul(2.0, dy);
    a[2] = o_mul(2.0, dz);
    a[3] = o_mul(2.0, o_mul(kSpeedOfLight2, dt));
}

// _compute_solution_residuals (:489-507), negated as np.linalg.solve gets them, and _compute_jacobian_matrix (:509-526).
GB_HD GB_INLINE void fix_system(const FixRow* r, const double* t, double gx, double gy, double gz, double cb,
                                double a[kFixRows][kFixRows], double rhs[kFixRows]) {
#pragma unroll
    for (int i = 0; i < kFixRows; ++i) fix_row(r[i], t[i], gx, gy, gz, cb, a[i], rhs[i]);
}

// np.linalg.solve(a, b) for one 4x4 system, in place: Gaussian elimination with partial pivoting (the first largest
// magnitude, as LAPACK's idamax picks it).  Returns false on an exactly zero pivot, where numpy raises "Singular matrix".
// Rows swap by compile-time index only, so the system stays in registers.
GB_HD GB_INLINE bool fix_solve(double a[kFixRows][kFixRows], double b[kFixRows], double v[kFixRows]) {
#pragma unroll
    for (int k = 0; k < kFixRows; ++k) {
        int p = k;
        double best = fabs(a[k][k]);
#pragma unroll
        for (int i = k + 1; i < kFixRows; ++i)
            if (fabs(a[i][k]) > best) best = fabs(a[i][k]), p = i;
        if (best == 0.0) return false;
#pragma unroll
        for (int i = k + 1; i < kFixRows; ++i)
            if (i == p) {
#pragma unroll
                for (int j = k; j < kFixRows; ++j) {
                    const double s = a[k][j];
                    a[k][j] = a[i][j];
                    a[i][j] = s;
                }
                const double s = b[k];
                b[k] = b[i];
                b[i] = s;
            }
#pragma unroll
        for (int i = k + 1; i < kFixRows; ++i) {
            const double l = a[i][k] / a[k][k];
#pragma unroll
            for (int j = k + 1; j < kFixRows; ++j) a[i][j] = o_sub(a[i][j], o_mul(l, a[k][j]));
            b[i] = o_sub(b[i], o_mul(l, b[k]));
        }
    }
#pragma unroll
    for (int i = kFixRows - 1; i >= 0; --i) {
        double s = b[i];
#pragma unroll
        for (int j = i + 1; j < kFixRows; ++j) s = o_sub(s, o_mul(a[i][j], v[j]));
        v[i] = s / a[i][i];
    }
    return true;
}

// F_m: _compute_position (:591-633) for the rows r at receiver_timestamp rx from the entering slide.  Fills slide_in,
// slide_out, the pseudoranges and, when solved, the solution; returns kFixSolved, or kFixRaised where np.linalg.solve
// raises (slide_out is then the slide at that point and the solution stays NaN).
GB_HD inline int fix_compute(const FixRow* r, double rx, double slide, FixRecord& f) {
    f.slide_in = slide;
    double gx = 0.0, gy = 0.0, gz = 0.0, cb = 0.0;  // ReceiverSolution(clock_bias=0, EcefCoordinates.zero())
    for (int round = 0; round < kFixRounds; ++round) {
        const double now = o_add(slide, rx);  // get_pseudorange_for_satellite (:362-377)
        double t[kFixRows];
#pragma unroll
        for (int i = 0; i < kFixRows; ++i) t[i] = o_sub(now, r[i].tow);
        if (round == 0)
            for (int i = 0; i < kFixRows; ++i) f.pseudorange[i] = t[i];
        for (int it = 0; it < kFixIterations; ++it) {
            double a[kFixRows][kFixRows], b[kFixRows], v[kFixRows];
            fix_system(r, t, gx, gy, gz, cb, a, b);
            if (!fix_solve(a, b, v)) {
                f.slide_out = slide;
                return kFixRaised;
            }
            gx = o_add(gx, v[0]);
            gy = o_add(gy, v[1]);
            gz = o_add(gz, v[2]);
            cb = o_add(cb, v[3]);
        }
        slide = o_sub(slide, cb);  // self.receiver_clock_slide -= clock_bias
    }
    f.slide_out = slide;
    f.clock_bias = cb;
    f.x = gx;
    f.y = gy;
    f.z = gz;
    return kFixSolved;
}

// The streaming least-squares solve: the upper triangle R (r[i][j], j >= i) and Q^T b of the rows added so far.
struct FixLsq {
    double r[kFixRows][kFixRows];
    double q[kFixRows];
};

GB_HD GB_INLINE void fix_lsq_clear(FixLsq& s) {
#pragma unroll
    for (int i = 0; i < kFixRows; ++i) {
        s.q[i] = 0.0;
#pragma unroll
        for (int j = 0; j < kFixRows; ++j) s.r[i][j] = 0.0;
    }
}

// Rotates the row [a | b] into the triangle, column by column (a and b are consumed).  Each rotation zeroes a[k]
// against r[k][k] and leaves r[k][k] >= 0.
GB_HD GB_INLINE void fix_lsq_add(FixLsq& s, double a[kFixRows], double b) {
#pragma unroll
    for (int k = 0; k < kFixRows; ++k) {
        if (a[k] == 0.0) continue;
        const double h = sqrt(o_add(o_mul(s.r[k][k], s.r[k][k]), o_mul(a[k], a[k])));
        const double c = s.r[k][k] / h, sn = a[k] / h;
        s.r[k][k] = h;
#pragma unroll
        for (int j = k + 1; j < kFixRows; ++j) {
            const double u = s.r[k][j], w = a[j];
            s.r[k][j] = o_add(o_mul(c, u), o_mul(sn, w));
            a[j] = o_sub(o_mul(c, w), o_mul(sn, u));
        }
        const double u = s.q[k];
        s.q[k] = o_add(o_mul(c, u), o_mul(sn, b));
        b = o_sub(o_mul(c, b), o_mul(sn, u));
    }
}

// Back-substitution R v = Q^T b over n rows.  Returns false where the system has rank < 4 as np.linalg.lstsq judges it
// with its default rcond (machine epsilon * max(n, 4)), here on R's diagonal: |r_kk| <= eps * max(n, 4) * max |r_jj|.
GB_HD GB_INLINE bool fix_lsq_solve(const FixLsq& s, int n, double v[kFixRows]) {
    double top = 0.0;
#pragma unroll
    for (int k = 0; k < kFixRows; ++k) top = fmax(top, s.r[k][k]);
    const double tol = o_mul(o_mul(0x1p-52, static_cast<double>(n > kFixRows ? n : kFixRows)), top);
#pragma unroll
    for (int k = 0; k < kFixRows; ++k)
        if (!(s.r[k][k] > tol)) return false;
#pragma unroll
    for (int i = kFixRows - 1; i >= 0; --i) {
        double t = s.q[i];
#pragma unroll
        for (int j = i + 1; j < kFixRows; ++j) t = o_sub(t, o_mul(s.r[i][j], v[j]));
        v[i] = t / s.r[i][i];
    }
    return true;
}

// fix_compute over n >= 5 rows in the least-squares mode.  rows(fn) calls fn(i, FixRow) for the rows i = 0..n-1 in the
// world model's order; it runs once per iteration, so the rows are read again rather than kept.  pseudorange[] holds
// round 0's of the first four rows.  Returns kFixSolved, or kFixRaised where the system is rank-deficient (slide_out is
// then the slide at that point and the solution stays NaN).
template <class Rows>
GB_HD inline int fix_compute_lsq(const Rows& rows, int n, double rx, double slide, FixRecord& f) {
    f.slide_in = slide;
    double gx = 0.0, gy = 0.0, gz = 0.0, cb = 0.0;
    for (int round = 0; round < kFixRounds; ++round) {
        const double now = o_add(slide, rx);
        if (round == 0)
            rows([&](int i, const FixRow& r) {
#pragma unroll
                for (int j = 0; j < kFixRows; ++j)  // by compile-time index, so the record stays in registers
                    if (i == j) f.pseudorange[j] = o_sub(now, r.tow);
            });
        for (int it = 0; it < kFixIterations; ++it) {
            FixLsq s;
            fix_lsq_clear(s);
            rows([&](int, const FixRow& r) {
                double a[kFixRows], b;
                fix_row(r, o_sub(now, r.tow), gx, gy, gz, cb, a, b);
                fix_lsq_add(s, a, b);
            });
            double v[kFixRows];
            if (!fix_lsq_solve(s, n, v)) {
                f.slide_out = slide;
                return kFixRaised;
            }
            gx = o_add(gx, v[0]);
            gy = o_add(gy, v[1]);
            gz = o_add(gz, v[2]);
            cb = o_add(cb, v[3]);
        }
        slide = o_sub(slide, cb);
    }
    f.slide_out = slide;
    f.clock_bias = cb;
    f.x = gx;
    f.y = gy;
    f.z = gz;
    return kFixSolved;
}

// What a change-table entry (orbit_walk) after entry 0 records: a subframe the world model handled
// (handle_subframe_emitted: it counts again), a lost lock (handle_lost_satellite_lock: it stops counting) or the
// decoder's raise (frozen).
GB_HD GB_INLINE bool fix_change_is_subframe(const OrbitSnap& s) { return !s.frozen && s.counting; }
GB_HD GB_INLINE bool fix_change_is_drop(const OrbitSnap& s) { return !s.frozen && !s.counting; }

// The slide a subframe sets (handle_subframe_emitted, :749-752, whose `or True` makes every subframe reset it).
GB_HD GB_INLINE double fix_reset_slide(const OrbitSnap& s) {
    return o_sub(s.p[kTowAtLastTimestamp], s.p[kRxTimestampAtLastHow]);
}

}  // namespace gb
