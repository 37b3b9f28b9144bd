// Host build of the C/N0 and phase-lock estimator (gypsum_b200/csrc/signal_core.cuh), for tests/test_signal_cpu.py and
// tests/test_gpu_signal.py.  Built with nvcc for the host only; no device code runs.  It walks one channel's records
// one millisecond at a time, the plain statement of what k_signal_windows computes window by window in parallel.
#include <cstddef>

#include "../../gypsum_b200/csrc/signal_core.cuh"
#include "../../include/gypsum_b200.h"

using namespace gb;

static_assert(sizeof(gb200_signal_window) == sizeof(SignalWindow), "ABI and device signal windows must match");
static_assert(sizeof(gb200_track_record) == sizeof(TrackMsRecord), "ABI and device track records must match");

extern "C" {
void signal_emu_init(SignalState* st) { signal_state_init(*st); }
int signal_emu_state_bytes(void) { return static_cast<int>(sizeof(SignalState)); }
double signal_emu_floor(int n) { return signal_noise_floor_dbhz(n); }

// One call over one channel's n_ms records: windows to out (up to max_out), returns the number produced.
int signal_emu_run(SignalState* st, const TrackMsRecord* rec, const double* start_times, int n_ms, int window_ms,
                   double floor_dbhz, SignalWindow* out, int max_out) {
    int n_out = 0;
    if (st->stopped) return 0;
    for (int k = 0; k < n_ms; ++k) {
        if (rec[k].lost) {
            if (st->open.n > 0) {
                if (n_out < max_out) out[n_out] = signal_window(st->open, st->t0, st->consumed - st->open.n, k - 1, floor_dbhz);
                n_out++;
            }
            signal_sums_clear(st->open);
            st->t0 = 0.0;
            st->stopped = 1;
            break;
        }
        if (st->open.n == 0) st->t0 = start_times[k];
        signal_add(st->open, rec[k].peak_re, rec[k].peak_im, rec[k].strength, rec[k].locked);
        st->consumed++;
        if (st->open.n == window_ms) {
            if (n_out < max_out) out[n_out] = signal_window(st->open, st->t0, st->consumed - st->open.n, k, floor_dbhz);
            n_out++;
            signal_sums_clear(st->open);
            st->t0 = 0.0;
        }
    }
    return n_out;
}

// offsets of gb200_signal_window's fields as the C++ compiler lays them out
void signal_emu_layout(long long* out /*[11]*/) {
    out[0] = offsetof(gb200_signal_window, receiver_timestamp);
    out[1] = offsetof(gb200_signal_window, cn0_dbhz);
    out[2] = offsetof(gb200_signal_window, prompt_power);
    out[3] = offsetof(gb200_signal_window, noise_power);
    out[4] = offsetof(gb200_signal_window, pll_lock);
    out[5] = offsetof(gb200_signal_window, first_ms);
    out[6] = offsetof(gb200_signal_window, ms_index);
    out[7] = offsetof(gb200_signal_window, n_ms);
    out[8] = offsetof(gb200_signal_window, locked_ms);
    out[9] = offsetof(gb200_signal_window, status);
    out[10] = sizeof(gb200_signal_window);
}
}
