// Carrier-to-noise density (C/N0) and phase-lock indicator of every tracking channel, over windows of W consecutive
// milliseconds of its tracking records (DESIGN.md §8e).  Host/device code: signal.cu runs it on the device,
// tests/emu/signal_emu.cu on the host.
//
// The tracking record's prompt P_k is the coherent correlation at the argmax of the whole |prompt profile|, and its
// strength s_k is |P_k| over the mean of the other profile magnitudes, so every millisecond carries a noise estimate
// taken from about N lags: with Rayleigh-distributed noise magnitudes the noise power per lag is (4/pi) (|P_k| / s_k)^2.
// Over a window of n records
//     M2 = sum |P_k|^2 / n,   Pn = (4/pi) sum (|P_k| / s_k)^2 / n,   C/N0 = 10 log10((M2 - Pn) / (Pn * 1 ms)),
//     PLI = (sum I^2 - sum Q^2) / (sum I^2 + sum Q^2).
// For noise alone |P|^2 is the largest of N exponentials, whose mean over Pn is the harmonic number H_N, so the estimate
// has a known floor, 10 log10((H_N - 1) / 1 ms): 38.57 dB-Hz at N = 2046, 39.68 at N = 16368.  Status 1 (a signal)
// needs C/N0 >= floor + 1 dB.  The signal's own off-peak correlation raises Pn a little, so strong signals read slightly
// low (DESIGN.md §8e gives the measured bias).
//
// Every sum runs in millisecond order with o_add / o_mul and IEEE division, so a window's sums do not depend on where
// calls split the stream, and the host and device builds agree bit for bit up to the last log10.
#pragma once
#include <math.h>

#include "orbit_core.cuh"
#include "tracker_core.cuh"

namespace gb {

constexpr int kSignalMinMs = 20;        // the shortest window, and the fewest records a cut window is estimated from
constexpr int kSignalMaxMs = 60000;     // the longest window
constexpr double kSignalMarginDb = 1.0; // status 1 needs C/N0 >= floor + this
constexpr double kSignalFourOverPi = 4.0 / 3.14159265358979323846;  // a Rayleigh variable's power over its mean squared

// gb200_signal_window.status
enum SignalStatus {
    kSignalNone = 0,   // not estimated: fewer than kSignalMinMs records (a stop cut the window) or a sum is not finite
    kSignalFound = 1,  // C/N0 >= floor + 1 dB
    kSignalNoise = 2,  // C/N0 < floor + 1 dB, or M2 <= Pn (C/N0 NaN): nothing distinguishable from noise
};

struct SignalWindow {  // mirrors include/gypsum_b200.h gb200_signal_window, 64 bytes
    double receiver_timestamp;  // chunk start of the window's first millisecond
    double cn0_dbhz;
    double prompt_power;        // M2
    double noise_power;         // Pn
    double pll_lock;            // PLI
    long long first_ms;         // the window's first record, counted from the first one the channel's estimator consumed
    int ms_index;               // millisecond of the call holding the window's last counted record, -1 = an earlier call
    int n_ms;                   // records in the window: W, or fewer when a stop cut it
    int locked_ms;              // records whose `locked` flag is set
    int status;                 // SignalStatus
};
static_assert(sizeof(SignalWindow) == 64, "signal window must stay 64 bytes");

// A window's sums so far.
struct SignalSums {
    double i2, q2;  // sum I^2, sum Q^2 of the prompts
    double pn;      // sum |P|^2 / strength^2
    int n;          // records counted
    int locked;     // of them with `locked` set
};

// One channel's estimator, carried from call to call.
struct SignalState {
    SignalSums open;     // the window the last call left open (n < W)
    double t0;           // receiver timestamp of its first millisecond (when open.n > 0)
    long long consumed;  // records counted so far
    int stopped;         // the channel met a lost record: nothing further is counted
    int pad_;
};

GB_HD GB_INLINE void signal_sums_clear(SignalSums& s) {
    s.i2 = s.q2 = s.pn = 0.0;
    s.n = s.locked = 0;
}

GB_HD inline void signal_state_init(SignalState& st) {
    signal_sums_clear(st.open);
    st.t0 = 0.0;
    st.consumed = 0;
    st.stopped = 0;
    st.pad_ = 0;
}

// One millisecond's record: prompt I, Q, strength and the `locked` flag.
GB_HD GB_INLINE void signal_add(SignalSums& s, float peak_re, float peak_im, float strength, int locked) {
    const double i = peak_re, q = peak_im, st = strength;
    const double i2 = o_mul(i, i), q2 = o_mul(q, q);
    s.i2 = o_add(s.i2, i2);
    s.q2 = o_add(s.q2, q2);
    s.pn = o_add(s.pn, o_add(i2, q2) / o_mul(st, st));
    s.n += 1;
    s.locked += locked != 0 ? 1 : 0;
}

// The record of a window with sums s (s.n >= 1); floor_dbhz is signal_noise_floor_dbhz of the stream's N.
GB_HD inline SignalWindow signal_window(const SignalSums& s, double t0, long long first_ms, int ms_index, double floor_dbhz) {
    SignalWindow w;
    const double n = static_cast<double>(s.n);
    const double p = o_add(s.i2, s.q2);
    w.receiver_timestamp = t0;
    w.prompt_power = p / n;
    w.noise_power = o_mul(kSignalFourOverPi, s.pn / n);
    w.pll_lock = o_sub(s.i2, s.q2) / p;
    w.cn0_dbhz = NAN;
    w.first_ms = first_ms;
    w.ms_index = ms_index;
    w.n_ms = s.n;
    w.locked_ms = s.locked;
    if (s.n < kSignalMinMs || !isfinite(s.i2) || !isfinite(s.q2) || !isfinite(s.pn)) {
        w.status = kSignalNone;
    } else if (w.prompt_power > w.noise_power) {
        w.cn0_dbhz = o_mul(10.0, log10(o_sub(w.prompt_power, w.noise_power) / o_mul(w.noise_power, 1e-3)));
        w.status = w.cn0_dbhz >= o_add(floor_dbhz, kSignalMarginDb) ? kSignalFound : kSignalNoise;
    } else {
        w.status = kSignalNoise;
    }
    return w;
}

// An upper bound on the windows one call of n_ms milliseconds touches per channel: the carried one, then one every W.
GB_HD GB_INLINE int signal_max_segments(int n_ms, int window_ms) { return n_ms / window_ms + 2; }

// The estimate for noise alone at n samples per millisecond: 10 log10((H_n - 1) / 1 ms), H_n summed in order of k.
inline double signal_noise_floor_dbhz(int n) {
    double h = 0.0;
    for (int k = 1; k <= n; ++k) h += 1.0 / static_cast<double>(k);
    return 10.0 * log10((h - 1.0) / 1e-3);
}

}  // namespace gb
