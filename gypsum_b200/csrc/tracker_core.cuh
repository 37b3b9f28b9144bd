// Scalar half of the tracking loop (reference gypsum/tracker.py:157-203, :228-262, :297-303, :346-387): DLL / PLL
// updates, the `is_locked` heuristics and the periodic constellation check, all in float64 like the reference's
// Python floats.  Host/device code: the persistent tracking kernel runs it on one thread per channel, the lane
// emulator (tests/emu) runs it on the CPU against the reference's recorded trajectories.
#pragma once
#include <math.h>

#include "gb_common.cuh"

namespace gb {

constexpr int kLockWindow = 250;  // config.py:25 MILLISECONDS_TO_CONSIDER_FOR_TRACKER_LOCK_STATE
constexpr int kPeakRing = 1000;   // tracker.py:149 correlation_peaks_rolling_buffer maxlen
constexpr double kTau = 6.283185307179586476925286766559;

// Per-channel state that persists between calls.
struct TrackState {
    double doppler;         // tracker.py:123 current_doppler_shift
    double carrier_phase;   // :124 current_carrier_wave_phase_shift
    double phase_acc;       // :224 self.phase (float code-phase accumulator)
    double last_circ_time;  // :222 _time_since_last_constellation_circularity_induced_adjustment
    long long n_steps;      // milliseconds processed so far
    int code_phase;         // :125 current_prn_code_phase_shift (may leave [0, N): np.roll is modular)
    int prn;                // replica table row
    int lost;               // LostSatelliteLockError raised (tracker.py:378); the channel stops
    int err_count, err_head, peak_count, peak_head;
    // sliding sums over the last 250 phase errors / peaks (is_locked, tracker.py:169-190)
    double e_s1, e_s2;
    double n_sre, n_sim, n_sre2, p_sre, p_sre2;
    int n_cnt, p_cnt;
    double err_ring[kLockWindow];
    double peak_re[kPeakRing], peak_im[kPeakRing];
};

// One millisecond of one channel, as handed back to the host (112 bytes).
struct TrackMsRecord {
    double doppler, carrier_phase;  // current_* after this millisecond, INCLUDING the 6-second adjustment of tracker.py:380-387
    double error;                   // I*Q Costas discriminator (tracker.py:249)
    double disc;                    // (|E|^2 - |L|^2)/2 (tracker.py:297)
    double phase_acc;               // self.phase after the update
    double doppler_hist, carrier_phase_hist;  // what tracker.py:352-353 append to the histories: the loop state BEFORE that adjustment
    float peak_re, peak_im;         // coherent prompt peak (tracker.py:313)
    float strength;                 // tracker.py:311
    float early_re, early_im, late_re, late_im;
    int code_phase;                 // current_prn_code_phase_shift after the update (tracker.py:299)
    int symbol;                     // sign(Re peak) (tracker.py:316)
    int locked;                     // is_locked() as used by this millisecond's PLL bandwidth choice
    int lost;                       // 1: LostSatelliteLockError raised at this millisecond
    int peak_offset;                // argmax of the rolled prompt profile (tracker.py:310)
    int pad_[2];
};
static_assert(sizeof(TrackMsRecord) == 112, "track record must stay 112 bytes");

GB_HD GB_INLINE double pymod(double a, double m) {  // Python's float % for m > 0
    double r = fmod(a, m);
    if (r < 0.0) r += m;
    return r;
}
// The same value as pymod() without the fmod call when a lies in [-m, 2m) -- where a loop state that moved by one small
// step from [0, m) always lies: a - m is exact there (Sterbenz) and equals fmod(a, m); a + m for a negative a is exactly
// what Python's float % computes (fmod(a, m) = a, then + m).
GB_HD GB_INLINE double pymod_near(double a, double m) {
    if (a >= 0.0) {
        if (a < m) return a;
        if (a < 2.0 * m) return a - m;
    } else if (a >= -m) {
        return a + m;
    }
    return pymod(a, m);
}
GB_HD GB_INLINE double sign_of(double x) { return x > 0.0 ? 1.0 : (x < 0.0 ? -1.0 : 0.0); }

GB_HD inline void track_state_init(TrackState& st, int prn, double doppler, double carrier_phase, int code_phase) {
    st.doppler = doppler;
    st.carrier_phase = carrier_phase;
    st.phase_acc = static_cast<double>(code_phase);
    st.last_circ_time = 0.0;
    st.n_steps = 0;
    st.code_phase = code_phase;
    st.prn = prn;
    st.lost = 0;
    st.err_count = st.err_head = st.peak_count = st.peak_head = 0;
    st.e_s1 = st.e_s2 = 0.0;
    st.n_sre = st.n_sim = st.n_sre2 = st.p_sre = st.p_sre2 = 0.0;
    st.n_cnt = st.p_cnt = 0;
}

// tracker.py:191-197: the mean of the negative-pole cluster must lie within 6 degrees of the real axis (the reference
// writes abs() of a bool -- just the comparison).
GB_HD inline bool track_rot_ok(double mr, double mi) {
    const double angle = 180.0 - pymod((atan2(mi, mr) / kTau) * 360.0, 180.0);
    const double centered = angle < 90.0 ? angle : 180.0 - angle;
    return centered < 6.0;
}
// The same decision without the atan2 / fmod chain on almost every millisecond: |mi| against tan(6 deg) |mr| with a guard
// band of +-0.01 degree.  1 / 0 = decided, -1 = inside the band (or NaN / the origin): the reference arithmetic above decides.
GB_HD inline int track_rot_quick(double mr, double mi) {
    const double a = fabs(mi), b = fabs(mr);
    if (a < 0.10492777752783379 * b) return 1;   // tan(5.99 deg)
    if (a > 0.10528069947757225 * b) return 0;   // tan(6.01 deg)
    return -1;
}
// Equivalence with track_rot_ok is tested on the host over 36 k directions (tests/test_tracker_cpu.py).
GB_HD inline bool track_rot_ok_fast(double mr, double mi) {
    const int q = track_rot_quick(mr, mi);
    return q >= 0 ? q != 0 : track_rot_ok(mr, mi);
}

// Where the DLL accumulator wraps.  The reference hard-wires 2046 at every rate (tracker.py:301-303, :319; SURVEY F12);
// the tracker's "samples" code-phase mode wraps at N, the stream's samples per millisecond, so that every code phase in
// [0, N) stays on the signal.  At N = 2046 the two are the same computation.
constexpr double kReferenceCodeWrap = 2046.0;

// What _calculate_loop_filter_alpha_and_beta (tracker.py:228-244; lru-cached there as well) returns for the two loop
// bandwidths the tracker ever uses: [0] = 3 Hz (locked), [1] = 6 Hz (pull-in).  Same expressions, same evaluation order.
// wrap: the DLL accumulator's modulus (kReferenceCodeWrap or N).
struct TrackConsts {
    double alpha[2], beta[2];
    double wrap;
};
GB_HD inline TrackConsts track_consts(double fs, double wrap = kReferenceCodeWrap) {
    TrackConsts c;
    c.wrap = wrap;
    const double ts = 1.0 / fs;
    for (int i = 0; i < 2; ++i) {
        const double bw = i == 0 ? 3.0 : 6.0;
        c.alpha[i] = 4.0 * (1.0 / sqrt(2.0)) * bw * ts;
        c.beta[i] = 4.0 * (bw * bw) * ts;
    }
    return c;
}

// 1 / n for the window counts 1..250: from a table when the caller has one (the kernel keeps it in shared memory), else
// computed.  Only ever used inside guard bands (below), never for a value that is handed out.
GB_HD GB_INLINE double recip_count(const double* rtab, int n) { return rtab ? rtab[n] : 1.0 / n; }

// tracker.py:157-203.  Called after the current peak was pushed and before the current error is.
// The reference forms five means / variances with divisions every millisecond and compares them with fixed thresholds.
// Here each quantity is first formed with a reciprocal multiply (a few ulp off at most); only if it lands within a guard
// band of its threshold -- 1e-9 relative to the magnitudes it was subtracted from, seven orders above any possible
// difference -- is it recomputed with the reference's divisions.  The decisions are therefore the reference's, always; the
// divisions, the atan2 and the fmod run on a vanishing fraction of the milliseconds.  The three tests are independent and
// side-effect free, so a failed one ends the evaluation.
GB_HD inline bool track_is_locked(const TrackState& st, const double* rtab = nullptr) {
    if (st.err_count < kLockWindow) return false;
    {
        const double r = 1.0 / kLockWindow;  // compile-time constant
        double mean = st.e_s1 * r;
        const double a = st.e_s2 * r;
        double var = a - mean * mean;  // np.var (population)
        if (!(fabs(var - 900.0) > 1e-9 * (a + 900.0))) {
            mean = st.e_s1 / kLockWindow;
            var = st.e_s2 / kLockWindow - mean * mean;
        }
        if (!(var < 900.0)) return false;  // config.py:27
    }
    if (st.peak_count > 2) {
        double nv = 0.0, pv = 0.0, mr = 0.0, mi = 0.0, scale = 2.0;
        if (st.n_cnt >= 2) {
            const double rn = recip_count(rtab, st.n_cnt);
            mr = st.n_sre * rn;
            mi = st.n_sim * rn;
            const double a = st.n_sre2 * rn;
            nv = a - mr * mr;
            scale += a;
        }
        if (st.p_cnt >= 2) {
            const double rp = recip_count(rtab, st.p_cnt);
            const double pm = st.p_sre * rp, a = st.p_sre2 * rp;
            pv = a - pm * pm;
            scale += a;
        }
        double x = (nv + pv) / 2.0;
        if (!(fabs(x - 2.0) > 1e-9 * scale)) {
            nv = pv = 0.0;
            if (st.n_cnt >= 2) {
                const double m = st.n_sre / st.n_cnt;
                nv = st.n_sre2 / st.n_cnt - m * m;
            }
            if (st.p_cnt >= 2) {
                const double pm = st.p_sre / st.p_cnt;
                pv = st.p_sre2 / st.p_cnt - pm * pm;
            }
            x = (nv + pv) / 2.0;
        }
        if (!(x < 2.0)) return false;
        // 6-degree test: outside +-0.01 degree of the boundary the reciprocal-multiply means decide (their error is 1e-16
        // relative); inside, the reference's divisions, atan2 and modulo do
        const int q = track_rot_quick(mr, mi);
        if (q >= 0) return q != 0;
        if (st.n_cnt >= 2) {
            mr = st.n_sre / st.n_cnt;
            mi = st.n_sim / st.n_cnt;
        }
        return track_rot_ok(mr, mi);
    }
    return true;
}

GB_HD inline void track_push_peak(TrackState& st, double re, double im) {
    // the entry leaving the 250-window is the one pushed 250 steps ago
    if (st.peak_count >= kLockWindow) {
        const int old = (st.peak_head - kLockWindow + kPeakRing) % kPeakRing;
        const double ore = st.peak_re[old], oim = st.peak_im[old];
        if (ore < 0.0) {
            st.n_cnt--;
            st.n_sre -= ore;
            st.n_sim -= oim;
            st.n_sre2 -= ore * ore;
        } else {
            st.p_cnt--;
            st.p_sre -= ore;
            st.p_sre2 -= ore * ore;
        }
    }
    st.peak_re[st.peak_head] = re;
    st.peak_im[st.peak_head] = im;
    st.peak_head = (st.peak_head + 1) % kPeakRing;
    if (st.peak_count < kPeakRing) st.peak_count++;
    if (re < 0.0) {
        st.n_cnt++;
        st.n_sre += re;
        st.n_sim += im;
        st.n_sre2 += re * re;
    } else {
        st.p_cnt++;
        st.p_sre += re;
        st.p_sre2 += re * re;
    }
}

GB_HD inline void track_push_error(TrackState& st, double e) {
    if (st.err_count >= kLockWindow) {
        const double old = st.err_ring[st.err_head];
        st.e_s1 -= old;
        st.e_s2 -= old * old;
    } else {
        st.err_count++;
    }
    st.err_ring[st.err_head] = e;
    st.err_head = (st.err_head + 1) % kLockWindow;
    st.e_s1 += e;
    st.e_s2 += e * e;
}

// utils.py:119-144 over the whole peak ring (<= 1000 entries).  Returns false when there is nothing to do.
GB_HD inline bool track_constellation(const TrackState& st, double& circularity, bool& have_rot, double& rotation) {
    const int n = st.peak_count;
    if (n < 2) return false;
    double sr = 0.0, si = 0.0;
    for (int k = 0; k < n; ++k) {
        sr += st.peak_re[k];
        si += st.peak_im[k];
    }
    const double mr = sr / n, mi = si / n;
    double a = 0.0, b = 0.0, d = 0.0;
    for (int k = 0; k < n; ++k) {
        const double x = st.peak_re[k] - mr, y = st.peak_im[k] - mi;
        a += x * x;
        b += x * y;
        d += y * y;
    }
    a /= (n - 1);  // np.cov: ddof = 1
    b /= (n - 1);
    d /= (n - 1);
    const double half_tr = 0.5 * (a + d), rad = sqrt(0.25 * (a - d) * (a - d) + b * b);
    const double lmax = half_tr + rad, lmin = half_tr - rad;
    circularity = 1.0 - lmin / lmax;
    // rotation of the left pole (utils.py:119-131)
    int cnt = 0;
    double lr = 0.0, li = 0.0;
    for (int k = 0; k < n; ++k)
        if (st.peak_re[k] < 0.0) {
            lr += st.peak_re[k];
            li += st.peak_im[k];
            cnt++;
        }
    have_rot = cnt >= 2;
    if (have_rot) {
        const double angle = 180.0 - pymod((atan2(li / cnt, lr / cnt) / kTau) * 360.0, 180.0);
        rotation = angle > 90.0 ? angle - 180.0 : angle;
    }
    return true;
}

// tracker.py:319: a pseudosymbol is stamped with its chunk's start and end times delayed by code_phase / wrap ms, the
// delay rounded on its own and added to each time with its own rounding (the device adds with __dadd_rn, so that no
// multiply-add fused into one rounding moves a stamp by an ulp).  Division by a runtime 2046.0 rounds as by the literal.
GB_HD GB_INLINE double track_symbol_delay(int code_phase, double wrap) {
    return (static_cast<double>(code_phase) / wrap) * 0.001;
}

// The scalar part of GpsSatelliteTracker.process_samples for one millisecond.  E, L, peak come from the
// correlators (float32); everything after is float64.
GB_HD inline void track_update(TrackState& st, float2 E, float2 L, float2 peak, float strength, int peak_offset,
                               double start_time, const TrackConsts& tc, const double* rtab, TrackMsRecord& out) {
    // --- DLL, tracker.py:297-303 ---
    const double er = E.x, ei = E.y, lr = L.x, li = L.y;
    const double disc = ((er * er + ei * ei) - (lr * lr + li * li)) / 2.0;
    st.phase_acc += disc * 0.002;
    st.code_phase = static_cast<int>(st.phase_acc);  // int(): truncation toward zero
    st.phase_acc = pymod_near(st.phase_acc, tc.wrap);  // 2046 in the reference at every rate (SURVEY F12), or N
    // --- histories, tracker.py:346 ---
    const double pre = peak.x, pim = peak.y;
    track_push_peak(st, pre, pim);
    // --- PLL, tracker.py:246-262 ---
    const double error = pre * pim;
    const bool locked = track_is_locked(st, rtab);
    const double alpha = tc.alpha[locked ? 0 : 1], beta = tc.beta[locked ? 0 : 1];  // 3 Hz when locked, 6 Hz to pull in
    st.carrier_phase += error * alpha;
    st.carrier_phase = pymod_near(st.carrier_phase, kTau);
    st.doppler += error * beta;
    track_push_error(st, error);
    out.doppler_hist = st.doppler;  // tracker.py:352-353: appended to the histories before the check below
    out.carrier_phase_hist = st.carrier_phase;
    // --- periodic constellation check, tracker.py:370-387 ---
    int lost = 0;
    if (start_time - st.last_circ_time >= 6.0) {
        st.last_circ_time = start_time;
        double circ = 0.0, rot = 0.0;
        bool have_rot = false;
        if (track_constellation(st, circ, have_rot, rot)) {
            if (circ < 0.2) {
                lost = 1;
            } else if (circ < 0.93 && have_rot) {
                st.doppler += -sign_of(rot) * 5.0;
                st.carrier_phase += sign_of(rot) * (kTau / 4.0);
            }
        }
    }
    st.n_steps++;
    st.lost = lost;
    out.doppler = st.doppler;
    out.carrier_phase = st.carrier_phase;
    out.error = error;
    out.disc = disc;
    out.phase_acc = st.phase_acc;
    out.peak_re = peak.x;
    out.peak_im = peak.y;
    out.strength = strength;
    out.early_re = E.x;
    out.early_im = E.y;
    out.late_re = L.x;
    out.late_im = L.y;
    out.code_phase = st.code_phase;
    out.symbol = pre > 0.0 ? 1 : (pre < 0.0 ? -1 : 0);
    out.locked = locked ? 1 : 0;
    out.lost = lost;
    out.peak_offset = peak_offset;
    out.pad_[0] = out.pad_[1] = 0;
}

}  // namespace gb
