// Host build of the subframe decoder's state machine (gypsum_b200/csrc/nav_core.cuh) with its scalar preamble scan,
// for tests/test_nav_decoder_cpu.py and tests/test_nav_edges_cpu.py.  Built with nvcc for the host only; no device
// code runs.
#include <cstddef>
#include <cstring>

#include "../../gypsum_b200/csrc/nav_core.cuh"
#include "../../include/gypsum_b200.h"

using namespace gb;

static_assert(sizeof(gb200_subframe_event) == sizeof(SubframeEvent), "ABI and device subframe events must match");

extern "C" {
int nav_emu_state_size() { return (int)sizeof(NavState); }
void nav_emu_init(NavState* st) {
    memset(st, 0, sizeof(NavState));
    nav_state_init(st->h);
}
// n bit events of one channel (values 1 / 0 / -1); returns the number of events (may exceed max_events)
int nav_emu_run(NavState* st, int n, const int* bits, const double* t0, const double* t1, SubframeEvent* out, int max_events) {
    NavQueue q{st->val, st->known, st->qstart, st->qend};
    int n_out = 0;
    for (int k = 0; k < n; ++k) nav_step(st->h, q, bits[k], t0[k], t1[k], k, out, max_events, n_out);
    return n_out;
}
// nav_emu_run that also records, for every bit k, what nav_push chose and the queue the search saw:
// trace[4k .. 4k+3] = scan kind (NavPush), qhead and qlen after the push, phase after the bit (-1 = None)
int nav_emu_trace(NavState* st, int n, const int* bits, const double* t0, const double* t1, SubframeEvent* out,
                  int max_events, int* trace) {
    NavQueue q{st->val, st->known, st->qstart, st->qend};
    int n_out = 0;
    for (int k = 0; k < n; ++k) {
        const int n_at_bit = n_out;
        const int scan = nav_push(st->h, q, bits[k], t0[k], t1[k]);
        trace[4 * k] = scan;
        trace[4 * k + 1] = st->h.qhead;
        trace[4 * k + 2] = st->h.qlen;
        int up = -1, inv = -1;
        if (scan == kNavFullScan) {
            up = nav_first_pair(q, st->h.qhead, st->h.qlen, kPreambleUp);
            if (up < 0) inv = nav_first_pair(q, st->h.qhead, st->h.qlen, kPreambleInv);
        }
        nav_finish(st->h, q, scan, up, inv, k, out, max_events, n_out, n_at_bit);
        trace[4 * k + 3] = st->h.phase;
    }
    return n_out;
}
void nav_emu_summary(const NavState* st, long long* out /*[6]*/) {
    out[0] = st->h.phase;
    out[1] = st->h.emitted;
    out[2] = st->h.polarity;
    out[3] = st->h.qlen;
    out[4] = st->h.stopped;
    out[5] = st->h.bits;
}
// offsets of gb200_subframe_event's fields as the C++ compiler lays them out
void nav_emu_layout(long long* out /*[11]*/) {
    out[0] = offsetof(gb200_subframe_event, receiver_timestamp);
    out[1] = offsetof(gb200_subframe_event, trailing_edge_receiver_timestamp);
    out[2] = offsetof(gb200_subframe_event, words);
    out[3] = offsetof(gb200_subframe_event, kind);
    out[4] = offsetof(gb200_subframe_event, bit_index);
    out[5] = offsetof(gb200_subframe_event, subframe_id);
    out[6] = offsetof(gb200_subframe_event, tow);
    out[7] = offsetof(gb200_subframe_event, phase);
    out[8] = offsetof(gb200_subframe_event, polarity);
    out[9] = offsetof(gb200_subframe_event, parity_ok);
    out[10] = sizeof(gb200_subframe_event);
}
}
