// C ABI of the trackers (include/gypsum_b200.h): tracking, the receiver chain behind it and the signal windows.  The
// engine the trackers run on is in engine.cu.
#include <cmath>
#include <cstddef>

#include "host.cuh"
#include "bits_core.cuh"
#include "fix_core.cuh"
#include "velocity_core.cuh"
#include "signal_core.cuh"
#include "nav_core.cuh"
#include "orbit_core.cuh"

using namespace gb;
using namespace gb::capi;

// What a tracker's device memory holds for the next stage of its call chain process -> integrate_bits ->
// decode_subframes -> parse_subframes -> observations / position_fixes, and the one place that changes it.  A stage's
// output is on the chain when it came, stage by stage, from the records of one whole-bank process call: its n_ms is
// that call's milliseconds (0 = off the chain).  Each transition runs when its call has succeeded, except
// process_begin, which runs before the tracking launch of process and process_channels.
struct TrackerChain {
    struct Output {
        std::vector<int> counts;  // events per channel, `stride` apart on the device
        int stride = 0;
        int n_ms = 0;          // the chain it belongs to (0 = not on the chain)
        bool pending = false;  // the next stage's chain call has not consumed it yet
    };
    Output records;    // the last whole-bank process call's [channel][n_ms] records (n_ms only)
    Output bits;       // the last integrate call's bit events
    Output subframes;  // the last decode call's subframe events
    Output orbit;      // the change tables of the last parse call: stride and n_ms (0 = no parse call yet)
    bool fix_pending = false;  // the last parse call's fixes are not computed yet
    bool fix_gap = false;      // a parse call's fixes were skipped after the first fix call: for the tracker's lifetime
    bool parse_records = false;  // the last parse call came from the records still in d_out (their Dopplers)

    // the records are about to be rewritten: nothing behind them is on the chain any more; pending bits stay pending
    void process_begin() {
        records.n_ms = bits.n_ms = subframes.n_ms = 0;
        parse_records = false;
    }
    void processed(int n_ms) { records.n_ms = n_ms; }  // whole-bank calls only
    void integrated(const int* counts, int nc, int stride, bool own_records) {
        bits = {{counts, counts + nc}, stride, own_records ? records.n_ms : 0, true};
        subframes.n_ms = 0;
    }
    void decoded(const int* counts, int nc, int stride, bool own_bits) {
        subframes = {{counts, counts + nc}, stride, own_bits ? bits.n_ms : 0, true};
        if (own_bits) bits.pending = false;
    }
    // fixing_began: the receiver state exists (a fix call has run)
    void parsed(int n_ms, int change_stride, bool own_subframes, bool fixing_began) {
        if (own_subframes) subframes.pending = false;
        parse_records = own_subframes;
        orbit.n_ms = n_ms;
        orbit.stride = change_stride;
        if (fixing_began && fix_pending) fix_gap = true;
        fix_pending = true;
    }
    void fixed() { fix_pending = false; }
    bool subframes_on_chain() const { return subframes.n_ms && subframes.pending; }
};

struct gb200_tracker {
    gb200_engine* e = nullptr;
    int n_channels = 0;
    std::vector<char> seeded;     // pool slots that hold a channel (gb200_tracker_create seeds all)
    std::vector<char> undo_ok;    // shadow[c] holds channel c's state before its last keep_undo launch
    std::vector<int> sel_cache;   // what d_sel currently holds
    std::vector<int> prn;         // replica row per channel, -1 for a pool slot never seeded
    DevBuf<TrackState> states, shadow;
    DevBuf<int> d_sel;
    PinnedBuf<int> h_sel;
    DevBuf<TrackMsRecord> d_out;
    DevBuf<double> d_times;
    DevBuf<float> d_prof;
    PinnedBuf<TrackMsRecord> h_out;
    PinnedBuf<double> h_times;
    PinnedBuf<float> h_prof;
    TrackerChain chain;
    double code_wrap = kReferenceCodeWrap;  // gb200_tracker_set_code_phase_mode: the DLL's modulus and the symbol delay's
    bool tracked = false;                   // a tracking or bit-integration launch has used code_wrap
    // Each later stage's per-channel state (created by its first call) and scratch.
    struct {  // bits.cu
        DevBuf<BitState> states;
        DevBuf<BitEvent> d_events;
        DevBuf<int> d_counts;
        DevBuf<double> d_times;
        PinnedBuf<BitEvent> h_events;
        PinnedBuf<int> h_counts;
        PinnedBuf<double> h_times;
    } bits;
    struct {  // nav.cu
        DevBuf<NavState> states;
        DevBuf<SubframeEvent> d_events;
        DevBuf<int> d_counts, d_bit_counts;
        PinnedBuf<SubframeEvent> h_events;
        PinnedBuf<int> h_counts, h_bit_counts;
    } nav;
    struct {  // orbit.cu
        DevBuf<OrbitSnap> states, d_changes;
        DevBuf<SubframeFields> d_fields;
        DevBuf<int> d_field_counts, d_change_counts, d_event_ms, d_drop_ms, d_counts;
        PinnedBuf<int> h_field_counts, h_event_ms, h_drop_ms, h_counts;
        DevBuf<SvObservation> d_obs;
        PinnedBuf<SvObservation> h_obs;
    } orbit;
    struct {  // fix.cu: the receiver state is `bank` and `rank`
        int solver = kFixSolverReference;  // gb200_tracker_set_fix_solver
        DevBuf<FixBank> bank;
        DevBuf<int> rank, order, touch, prev;
        DevBuf<double> rx, reset, slide1;
        DevBuf<FixRecord> d_fixes;
        PinnedBuf<double> h_rx;
        PinnedBuf<FixRecord> h_fixes;
        bool kept = false;  // d_fixes holds the last fix call's records (gb200_tracker_position_fixes, not _device)
    } fix;
    struct {  // velocity.cu
        DevBuf<VelocityRecord> d_out;
        PinnedBuf<VelocityRecord> h_out;
    } vel;
    struct {  // signal.cu
        int window_ms = 0;  // W, fixed by the first call (0 = no call yet)
        double floor_dbhz = 0.0;  // signal_noise_floor_dbhz(N), from the first call on
        DevBuf<SignalState> states, carried;
        DevBuf<SignalWindow> d_out;
        DevBuf<int> d_stop, d_counts;
        DevBuf<double> d_times;
        PinnedBuf<SignalWindow> h_out;
        PinnedBuf<int> h_counts;
        PinnedBuf<double> h_times;
    } sig;
};

static_assert(sizeof(gb200_track_record) == sizeof(TrackMsRecord), "ABI track record and device record must match");
static_assert(sizeof(gb200_bit_event) == sizeof(BitEvent), "ABI bit event and device event must match");
static_assert(sizeof(gb200_subframe_event) == sizeof(SubframeEvent) && sizeof(SubframeEvent) == 96,
              "ABI subframe event and device event must match");
static_assert(sizeof(gb200_subframe_fields) == sizeof(SubframeFields) &&
                  offsetof(gb200_subframe_fields, tow_seconds) == offsetof(SubframeFields, tow_seconds) &&
                  offsetof(gb200_subframe_fields, bit_widths) == offsetof(SubframeFields, widths) &&
                  offsetof(gb200_subframe_fields, values) == offsetof(SubframeFields, values),
              "ABI subframe fields and device fields must match");
static_assert(sizeof(gb200_sv_observation) == sizeof(SvObservation) &&
                  offsetof(gb200_sv_observation, prn_count) == offsetof(SvObservation, prn_count) &&
                  offsetof(gb200_sv_observation, flags) == offsetof(SvObservation, flags),
              "ABI observation and device observation must match");
static_assert(GB200_CODE_PHASE_REFERENCE == 0 && GB200_CODE_PHASE_SAMPLES == 1, "code-phase modes are 0 and 1");
static_assert(GB200_FIX_SOLVER_REFERENCE == kFixSolverReference && GB200_FIX_SOLVER_LEAST_SQUARES == kFixSolverLeastSquares,
              "ABI and device fix solvers must match");
static_assert(sizeof(gb200_position_fix) == sizeof(FixRecord) &&
                  offsetof(gb200_position_fix, pseudorange) == offsetof(FixRecord, pseudorange) &&
                  offsetof(gb200_position_fix, status) == offsetof(FixRecord, status) &&
                  offsetof(gb200_position_fix, channel) == offsetof(FixRecord, channel),
              "ABI position fix and device fix must match");
static_assert(sizeof(gb200_velocity_fix) == sizeof(VelocityRecord) &&
                  offsetof(gb200_velocity_fix, residual_rms) == offsetof(VelocityRecord, residual_rms) &&
                  offsetof(gb200_velocity_fix, status) == offsetof(VelocityRecord, status) &&
                  offsetof(gb200_velocity_fix, n_rows) == offsetof(VelocityRecord, n_rows),
              "ABI velocity fix and device velocity fix must match");
static_assert(sizeof(gb200_signal_window) == sizeof(SignalWindow) &&
                  offsetof(gb200_signal_window, first_ms) == offsetof(SignalWindow, first_ms) &&
                  offsetof(gb200_signal_window, ms_index) == offsetof(SignalWindow, ms_index) &&
                  offsetof(gb200_signal_window, status) == offsetof(SignalWindow, status),
              "ABI signal window and device signal window must match");
static_assert(offsetof(TrackMsRecord, doppler) == 0 && sizeof(TrackMsRecord) % sizeof(double) == 0,
              "the velocity fix reads the tracking records' Doppler with a stride in doubles");
static_assert(offsetof(gb200_subframe_event, words) == offsetof(SubframeEvent, words) &&
                  offsetof(gb200_subframe_event, kind) == offsetof(SubframeEvent, kind) &&
                  offsetof(gb200_subframe_event, parity_ok) == offsetof(SubframeEvent, parity_ok),
              "ABI subframe event and device event must match");

namespace {

int check_channel(gb200_tracker* t, int channel) {
    if (channel < 0 || channel >= t->n_channels) GB_FAIL(t->e, GB200_EINVAL, "channel %d out of range", channel);
    return GB200_OK;
}

// A new tracker of n slots, none seeded yet, whose device states fill(t) writes; on failure nothing is left behind.
template <class Fill>
int new_tracker(gb200_engine* e, int n, gb200_tracker** out, Fill fill) {
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_CUDA(e, configure_track_kernel());
    gb200_tracker* t = new gb200_tracker;
    t->e = e;
    t->n_channels = n;
    t->seeded.assign(n, 0);
    t->undo_ok.assign(n, 0);
    t->prn.assign(n, -1);
    cudaError_t ce = t->states.ensure(n);
    if (ce == cudaSuccess) ce = fill(t);
    if (ce != cudaSuccess) {
        delete t;
        cudaGetLastError();
        GB_FAIL(e, GB200_ECUDA, "tracker state allocation failed: %s", cudaGetErrorString(ce));
    }
    *out = t;
    return GB200_OK;
}

// Seeds channels first .. first + k - 1 from the k acquisitions given, with one copy of their initial states.
cudaError_t seed_channels(gb200_tracker* t, int first, int k, const int32_t* prn_idx, const double* doppler_hz,
                          const double* carrier_phase, const int32_t* code_phase) {
    std::vector<TrackState> init(k);
    for (int c = 0; c < k; ++c) {
        memset(&init[c], 0, sizeof(TrackState));
        track_state_init(init[c], prn_idx[c], doppler_hz[c], carrier_phase[c], code_phase[c]);
    }
    const cudaError_t ce = cudaMemcpy(t->states.p + first, init.data(), sizeof(TrackState) * k, cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) {
        std::fill_n(&t->seeded[first], k, 1);
        std::fill_n(&t->undo_ok[first], k, 0);
        std::copy_n(prn_idx, k, &t->prn[first]);
    }
    return ce;
}

// A chain stage's per-channel device state, created by the stage's first call from init on zeroed host objects.
template <class T, class Init>
int ensure_state(gb200_engine* e, DevBuf<T>& state, int n, Init init) {
    if (state.p) return GB200_OK;
    std::vector<T> host(n);
    for (T& s : host) {
        memset(&s, 0, sizeof(T));
        init(s);
    }
    GB_CUDA(e, state.ensure(n));
    GB_CUDA(e, cudaMemcpy(state.p, host.data(), sizeof(T) * n, cudaMemcpyHostToDevice));
    return GB200_OK;
}

// A getter's copy of `bytes` of a stage's device state from state.p[i] on, once the work in flight is done.  Before the
// stage's first call the state does not exist and dst keeps the host default.
template <class T>
int read_state(gb200_engine* e, void* dst, const DevBuf<T>& state, int i = 0, size_t bytes = sizeof(T)) {
    if (!state.p) return GB200_OK;
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_CUDA(e, cudaStreamSynchronize(e->stream));
    GB_CUDA(e, cudaMemcpy(dst, state.p + i, bytes, cudaMemcpyDeviceToHost));
    return GB200_OK;
}
static_assert(offsetof(BitState, h) == 0 && offsetof(NavState, h) == 0, "the getters read a state's head at its start");

// Channel c's `count` events fit the `stride` they sit apart at; fmt formats (c, count, stride).
int check_fits(gb200_engine* e, const char* fmt, int c, int count, int stride) {
    if (count < 0 || count > stride) GB_FAIL(e, GB200_EINVAL, fmt, c, count, stride);
    return GB200_OK;
}

// A stage's per-channel output to the caller: the counts' copy is enqueued first, so that copy_events, which waits for
// the stream, waits for both; then the counts go to counts_out.  h_counts keeps them for the chain's record.
template <class CopyEvents>
int fetch_output(gb200_engine* e, int nc, const DevBuf<int>& d_counts, PinnedBuf<int>& h_counts, int32_t* counts_out,
                 CopyEvents copy_events) {
    GB_CUDA(e, cudaMemcpyAsync(h_counts.p, d_counts.p, nc * sizeof(int), cudaMemcpyDeviceToHost, e->stream));
    GB_TRY(copy_events());
    memcpy(counts_out, h_counts.p, nc * sizeof(int));
    return GB200_OK;
}

// The tracking records a stage reads: the caller's records_device, or else the [channel][n_ms] records the last
// whole-bank process call left in d_out, which must be n_ms long.  Then sets the device and waits for the stream, whose
// pinned staging may still be in flight.
int input_records(gb200_tracker* t, const void* records_device, int n_ms, const TrackMsRecord** records) {
    gb200_engine* e = t->e;
    if (!records_device && t->chain.records.n_ms != n_ms)
        GB_FAIL(e, GB200_ESTATE, "no records of %d ms on the device (last gb200_tracker_process call held %d)", n_ms,
                t->chain.records.n_ms);
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_CUDA(e, cudaStreamSynchronize(e->stream));
    *records = records_device ? static_cast<const TrackMsRecord*>(records_device) : t->d_out.p;
    return GB200_OK;
}

// The host form of a stage whose device form is launch(out_dev): n records into the scratch d_out, then to out_host.
template <class T, class Launch>
int launch_to_host(gb200_tracker* t, void* out_host, size_t n, DevBuf<T>& d_out, PinnedBuf<T>& h_out, Launch launch) {
    gb200_engine* e = t->e;
    if (!out_host) GB_FAIL(e, GB200_EINVAL, "null output");
    GB_CUDA(e, cudaSetDevice(e->device));
    if (n) GB_CUDA(e, d_out.ensure(n));
    GB_TRY(launch(d_out.p));
    return download(e, static_cast<T*>(out_host), d_out.p, n, h_out);
}

}  // namespace

extern "C" {

int gb200_tracker_create(gb200_engine* e, int n_channels, const int32_t* prn_idx, const double* doppler_hz,
                         const double* carrier_phase, const int32_t* code_phase, gb200_tracker** out) {
    if (!e) return GB200_EINVAL;
    if (!out) GB_FAIL(e, GB200_EINVAL, "null output");
    *out = nullptr;
    if (n_channels < 1 || !prn_idx || !doppler_hz || !carrier_phase || !code_phase) GB_FAIL(e, GB200_EINVAL, "no channels");
    GB_TRY(check_replicas(e));
    GB_TRY(check_prns(e, prn_idx, n_channels));
    return new_tracker(e, n_channels, out, [&](gb200_tracker* t) {
        return seed_channels(t, 0, n_channels, prn_idx, doppler_hz, carrier_phase, code_phase);
    });
}

int gb200_tracker_destroy(gb200_tracker* t) {
    if (!t) return GB200_OK;
    cudaSetDevice(t->e->device);
    cudaStreamSynchronize(t->e->stream);
    delete t;
    return GB200_OK;
}

// One launch of k_track_channels.  sel (host, may be null = every channel in order): the n_sel channels to advance; CTA i
// writes records out_dev[i * n_ms ...].  keep_undo: the kernel also stores every launched channel's previous state.
static int tracker_launch(gb200_tracker* t, int n_sel, const int32_t* sel, int n_ms, const double* start_times,
                          TrackMsRecord* out_dev, float* prof_dev, bool keep_undo) {
    gb200_engine* e = t->e;
    if (n_ms < 1 || !start_times) GB_FAIL(e, GB200_EINVAL, "need at least one whole millisecond of samples");
    GB_TRY(check_iq(e, n_ms));
    GB_TRY(check_samples(e, n_ms));
    // k_track_channels stages the chunks of an even S with 16-byte cp.async; at odd S, N is odd, every other millisecond of
    // a stream starts 8 bytes past a 16-byte boundary, and both tracking kernels read it in 8-byte pieces (a device ring's
    // odd slots are such addresses)
    const uintptr_t iq_align = e->s % 2 == 0 ? 16 : 8;
    if (reinterpret_cast<uintptr_t>(e->iq) % iq_align != 0)
        GB_FAIL(e, GB200_EINVAL, "IQ buffer must be %d-byte aligned for tracking at S = %d", static_cast<int>(iq_align), e->s);
    if (sel) {
        for (int i = 0; i < n_sel; ++i) {
            GB_TRY(check_channel(t, sel[i]));
            if (!t->seeded[sel[i]]) GB_FAIL(e, GB200_ESTATE, "channel %d was never seeded (gb200_tracker_reset_channel)", sel[i]);
            for (int j = 0; j < i; ++j)
                if (sel[j] == sel[i]) GB_FAIL(e, GB200_EINVAL, "channel %d listed twice", sel[i]);
        }
    } else {
        for (int c = 0; c < t->n_channels; ++c)
            if (!t->seeded[c]) GB_FAIL(e, GB200_ESTATE, "channel %d was never seeded (gb200_tracker_reset_channel)", c);
    }
    TrackArgs a{};
    if (n_ms == 1) {
        a.start_times = nullptr;  // a single millisecond's start time travels in the kernel arguments
        a.t0_single = start_times[0];
    } else {
        GB_CUDA(e, cudaStreamSynchronize(e->stream));  // h_times may still be in flight
        GB_CUDA(e, t->d_times.ensure(n_ms));
        GB_TRY(upload(e, t->d_times.p, start_times, n_ms, t->h_times));
        a.start_times = t->d_times.p;
    }
    if (sel) {
        const bool cached = static_cast<int>(t->sel_cache.size()) == n_sel && memcmp(t->sel_cache.data(), sel, sizeof(int) * n_sel) == 0;
        if (!cached) {  // the subset rarely changes between calls: upload it only when it did
            GB_CUDA(e, cudaStreamSynchronize(e->stream));
            GB_CUDA(e, t->d_sel.ensure(n_sel));
            GB_TRY(upload(e, t->d_sel.p, sel, n_sel, t->h_sel));
            t->sel_cache.assign(sel, sel + n_sel);
        }
        a.channel_idx = t->d_sel.p;
    }
    if (keep_undo) {
        GB_CUDA(e, t->shadow.ensure(t->n_channels));
        a.shadow = t->shadow.p;
    }
    a.iq = e->iq;
    a.states = t->states.p;
    a.out = out_dev;
    a.profiles = prof_dev;
    a.crep = e->crep.p;
    a.tw1 = e->tw1.p;
    a.tw2 = e->tw2.p;
    a.fs = static_cast<double>(e->fs);
    a.inv_fs = 1.0 / static_cast<double>(e->fs);
    a.N = e->N;
    a.s = e->s;
    a.n_ms = n_ms;
    a.n_channels = sel ? n_sel : t->n_channels;
    a.code_wrap = t->code_wrap;
    t->tracked = true;
    GB_LAUNCH(e, -1, launch_track_channels(a, e->stream));
    for (int i = 0; i < a.n_channels; ++i) t->undo_ok[sel ? sel[i] : i] = keep_undo ? 1 : 0;
    return GB200_OK;
}

int gb200_tracker_process_device(gb200_tracker* t, int n_ms, const double* start_times, void* out_device) {
    if (!t) return GB200_EINVAL;
    gb200_engine* e = t->e;
    if (!out_device) GB_FAIL(e, GB200_EINVAL, "null output");
    GB_CUDA(e, cudaSetDevice(e->device));
    return tracker_launch(t, t->n_channels, nullptr, n_ms, start_times, static_cast<TrackMsRecord*>(out_device), nullptr, false);
}

static int tracker_process_host(gb200_tracker* t, int n_sel, const int32_t* sel, int n_ms, const double* start_times,
                                bool keep_undo, gb200_track_record* out_host, float* profiles_host) {
    gb200_engine* e = t->e;
    if (!out_host) GB_FAIL(e, GB200_EINVAL, "null output");
    GB_CUDA(e, cudaSetDevice(e->device));
    if (n_ms < 1) GB_FAIL(e, GB200_EINVAL, "need at least one whole millisecond of samples");
    if (n_sel < 1) GB_FAIL(e, GB200_EINVAL, "no channels");
    const size_t n = static_cast<size_t>(n_sel) * n_ms;
    GB_CUDA(e, t->d_out.ensure(n));
    const size_t np = profiles_host ? n * e->N : 0;
    if (np) {
        GB_CUDA(e, t->d_prof.ensure(np));
        GB_CUDA(e, t->h_prof.ensure(np));
    }
    t->chain.process_begin();  // d_out is about to be rewritten
    GB_TRY(tracker_launch(t, n_sel, sel, n_ms, start_times, t->d_out.p, np ? t->d_prof.p : nullptr, keep_undo));
    if (!sel) t->chain.processed(n_ms);  // gb200_tracker_integrate_bits reads [channel][n_ms] of the whole bank
    // the profiles' copy is enqueued first, so the records' download waits for both
    if (np) GB_CUDA(e, cudaMemcpyAsync(t->h_prof.p, t->d_prof.p, np * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
    GB_TRY(download(e, reinterpret_cast<TrackMsRecord*>(out_host), t->d_out.p, n, t->h_out));
    if (np) memcpy(profiles_host, t->h_prof.p, np * sizeof(float));
    return GB200_OK;
}

int gb200_tracker_process(gb200_tracker* t, int n_ms, const double* start_times, gb200_track_record* out_host,
                          float* profiles_host) {
    if (!t) return GB200_EINVAL;
    return tracker_process_host(t, t->n_channels, nullptr, n_ms, start_times, false, out_host, profiles_host);
}

int gb200_tracker_process_channels(gb200_tracker* t, int n_sel, const int32_t* channels, int n_ms, const double* start_times,
                                   int keep_undo, gb200_track_record* out_host, float* profiles_host) {
    if (!t) return GB200_EINVAL;
    if (!channels) GB_FAIL(t->e, GB200_EINVAL, "null channel list");
    return tracker_process_host(t, n_sel, channels, n_ms, start_times, keep_undo != 0, out_host, profiles_host);
}

int gb200_tracker_undo_channel(gb200_tracker* t, int channel) {
    if (!t) return GB200_EINVAL;
    gb200_engine* e = t->e;
    GB_TRY(check_channel(t, channel));
    if (!t->undo_ok[channel]) GB_FAIL(e, GB200_ESTATE, "channel %d has no kept state to go back to", channel);
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_CUDA(e, cudaMemcpyAsync(t->states.p + channel, t->shadow.p + channel, sizeof(TrackState), cudaMemcpyDeviceToDevice, e->stream));
    t->undo_ok[channel] = 0;
    return GB200_OK;
}

int gb200_tracker_create_pool(gb200_engine* e, int capacity, gb200_tracker** out) {
    if (!e) return GB200_EINVAL;
    if (!out) GB_FAIL(e, GB200_EINVAL, "null output");
    *out = nullptr;
    if (capacity < 1) GB_FAIL(e, GB200_EINVAL, "no channels");
    return new_tracker(e, capacity, out,
                       [](gb200_tracker* t) { return cudaMemset(t->states.p, 0, sizeof(TrackState) * t->n_channels); });
}

int gb200_tracker_reset_channel(gb200_tracker* t, int channel, int32_t prn_idx, double doppler_hz, double carrier_phase,
                                int32_t code_phase) {
    if (!t) return GB200_EINVAL;
    gb200_engine* e = t->e;
    GB_TRY(check_channel(t, channel));
    GB_TRY(check_prns(e, &prn_idx, 1));
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_CUDA(e, cudaStreamSynchronize(e->stream));
    GB_CUDA(e, seed_channels(t, channel, 1, &prn_idx, &doppler_hz, &carrier_phase, &code_phase));
    return GB200_OK;
}

int gb200_tracker_get_state(gb200_tracker* t, int channel, double* doppler_hz, double* carrier_phase, double* phase_acc,
                            int32_t* code_phase, int32_t* lost) {
    if (!t) return GB200_EINVAL;
    gb200_engine* e = t->e;
    GB_TRY(check_channel(t, channel));
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_CUDA(e, cudaStreamSynchronize(e->stream));
    TrackState st;
    GB_CUDA(e, cudaMemcpy(&st, t->states.p + channel, offsetof(TrackState, err_ring), cudaMemcpyDeviceToHost));
    if (doppler_hz) *doppler_hz = st.doppler;
    if (carrier_phase) *carrier_phase = st.carrier_phase;
    if (phase_acc) *phase_acc = st.phase_acc;
    if (code_phase) *code_phase = st.code_phase;
    if (lost) *lost = st.lost;
    return GB200_OK;
}

int gb200_tracker_set_state(gb200_tracker* t, int channel, double doppler_hz, double carrier_phase, double phase_acc,
                            int32_t code_phase) {
    if (!t) return GB200_EINVAL;
    gb200_engine* e = t->e;
    GB_TRY(check_channel(t, channel));
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_CUDA(e, cudaStreamSynchronize(e->stream));
    TrackState st;
    const size_t head = offsetof(TrackState, err_ring);
    GB_CUDA(e, cudaMemcpy(&st, t->states.p + channel, head, cudaMemcpyDeviceToHost));
    st.doppler = doppler_hz;
    st.carrier_phase = carrier_phase;
    st.phase_acc = phase_acc;
    st.code_phase = code_phase;
    st.lost = 0;  // the reference tracker object keeps processing after it raised LostSatelliteLockError
    GB_CUDA(e, cudaMemcpy(t->states.p + channel, &st, head, cudaMemcpyHostToDevice));
    t->undo_ok[channel] = 0;
    return GB200_OK;
}

int gb200_tracker_integrate_bits(gb200_tracker* t, int n_ms, const double* start_times, const double* end_times,
                                 const void* records_device, gb200_bit_event* events_host, int32_t max_events,
                                 int32_t* counts_host) {
    if (!t) return GB200_EINVAL;
    gb200_engine* e = t->e;
    auto& s = t->bits;
    const int nc = t->n_channels;
    if (n_ms < 1 || !start_times || !end_times) GB_FAIL(e, GB200_EINVAL, "need at least one millisecond and its timestamps");
    if (!events_host || !counts_host || max_events < 1) GB_FAIL(e, GB200_EINVAL, "null / empty event buffer");
    BitArgs a{};
    GB_TRY(input_records(t, records_device, n_ms, &a.records));
    GB_TRY(ensure_state(e, s.states, nc, [](BitState& b) { bit_state_init(b); }));
    const size_t ne = static_cast<size_t>(nc) * max_events;
    GB_CUDA(e, s.d_events.ensure(ne));
    GB_CUDA(e, s.d_counts.ensure(nc));
    GB_CUDA(e, s.h_counts.ensure(nc));
    GB_CUDA(e, s.d_times.ensure(2 * static_cast<size_t>(n_ms)));
    GB_CUDA(e, s.h_times.ensure(2 * static_cast<size_t>(n_ms)));
    memcpy(s.h_times.p, start_times, sizeof(double) * n_ms);
    memcpy(s.h_times.p + n_ms, end_times, sizeof(double) * n_ms);
    GB_CUDA(e, cudaMemcpyAsync(s.d_times.p, s.h_times.p, 2 * sizeof(double) * n_ms, cudaMemcpyHostToDevice, e->stream));
    a.start_times = s.d_times.p;
    a.end_times = s.d_times.p + n_ms;
    a.states = s.states.p;
    a.events = s.d_events.p;
    a.counts = s.d_counts.p;
    a.n_ms = n_ms;
    a.n_channels = nc;
    a.max_events = max_events;
    a.code_wrap = t->code_wrap;
    t->tracked = true;
    GB_LAUNCH(e, -1, launch_integrate_bits(a, e->stream));
    GB_TRY(fetch_output(e, nc, s.d_counts, s.h_counts, counts_host, [&]() -> int {
        return download(e, reinterpret_cast<BitEvent*>(events_host), s.d_events.p, ne, s.h_events);
    }));
    t->chain.integrated(s.h_counts.p, nc, max_events, !records_device);
    return GB200_OK;
}

int gb200_tracker_signal_windows(gb200_tracker* t, int n_ms, const double* start_times, int32_t window_ms,
                                 const void* records_device, gb200_signal_window* out_host, int32_t max_windows,
                                 int32_t* counts_host) {
    if (!t) return GB200_EINVAL;
    gb200_engine* e = t->e;
    auto& s = t->sig;
    const int nc = t->n_channels;
    if (n_ms < 1 || !start_times) GB_FAIL(e, GB200_EINVAL, "need at least one millisecond and its start times");
    if (!out_host || !counts_host || max_windows < 1) GB_FAIL(e, GB200_EINVAL, "null / empty window buffer");
    if (window_ms < kSignalMinMs || window_ms > kSignalMaxMs)
        GB_FAIL(e, GB200_EINVAL, "window_ms must be between %d and %d, not %d", kSignalMinMs, kSignalMaxMs, window_ms);
    if (s.window_ms && window_ms != s.window_ms)
        GB_FAIL(e, GB200_ESTATE, "the open windows were formed with window_ms = %d, not %d", s.window_ms, window_ms);
    SignalArgs a{};
    GB_TRY(input_records(t, records_device, n_ms, &a.records));
    GB_TRY(ensure_state(e, s.states, nc, [](SignalState& st) { signal_state_init(st); }));
    if (!s.window_ms) s.floor_dbhz = signal_noise_floor_dbhz(e->N);
    s.window_ms = window_ms;
    const size_t nw = static_cast<size_t>(nc) * max_windows;
    GB_CUDA(e, s.carried.ensure(nc));
    GB_CUDA(e, s.d_stop.ensure(nc));
    GB_CUDA(e, s.d_counts.ensure(nc));
    GB_CUDA(e, s.h_counts.ensure(nc));
    GB_CUDA(e, s.d_out.ensure(nw));
    GB_CUDA(e, s.d_times.ensure(n_ms));
    GB_TRY(upload(e, s.d_times.p, start_times, n_ms, s.h_times));
    a.start_times = s.d_times.p;
    a.states = s.states.p;
    a.carried = s.carried.p;
    a.stop = s.d_stop.p;
    a.out = s.d_out.p;
    a.counts = s.d_counts.p;
    a.floor_dbhz = s.floor_dbhz;
    a.n_ms = n_ms;
    a.n_channels = nc;
    a.window_ms = window_ms;
    a.max_windows = max_windows;
    GB_LAUNCH(e, -1, launch_signal_windows(a, e->stream));
    e->launches++;  // the stop scan and the windows
    return fetch_output(e, nc, s.d_counts, s.h_counts, counts_host, [&]() -> int {
        return download(e, reinterpret_cast<SignalWindow*>(out_host), s.d_out.p, nw, s.h_out);
    });
}

int gb200_tracker_bit_state(gb200_tracker* t, int channel, int64_t out[8]) {
    if (!t) return GB200_EINVAL;
    GB_TRY(check_channel(t, channel));
    if (!out) GB_FAIL(t->e, GB200_EINVAL, "null output");
    BitState st;
    memset(&st, 0, sizeof(st));
    bit_state_init(st);
    GB_TRY(read_state(t->e, &st, t->bits.states, channel, sizeof(BitHead)));
    const BitHead& h = st.h;
    const int64_t v[8] = {h.emitted, h.failed, h.processed, h.slide, h.determined, h.prev_decision, h.cursor, h.stopped};
    memcpy(out, v, sizeof(v));
    return GB200_OK;
}

int gb200_tracker_decode_subframes(gb200_tracker* t, const void* bits_device, const int32_t* bit_counts_host,
                                   int32_t bits_stride, gb200_subframe_event* events_host, int32_t max_events,
                                   int32_t* counts_host) {
    if (!t) return GB200_EINVAL;
    gb200_engine* e = t->e;
    auto& s = t->nav;
    const TrackerChain::Output& bits = t->chain.bits;
    const int nc = t->n_channels;
    if (!events_host || !counts_host || max_events < 1) GB_FAIL(e, GB200_EINVAL, "null / empty event buffer");
    const int* counts = bit_counts_host;
    int stride = bits_stride;
    if (bits_device) {
        if (!bit_counts_host || bits_stride < 1) GB_FAIL(e, GB200_EINVAL, "bit events need their counts and a stride >= 1");
        for (int c = 0; c < nc; ++c)
            GB_TRY(check_fits(e, "channel %d: %d bit events do not fit a stride of %d", c, counts[c], stride));
    } else {
        if (!bits.pending) GB_FAIL(e, GB200_ESTATE, "no undecoded bit events on the device (call gb200_tracker_integrate_bits first)");
        counts = bits.counts.data();
        stride = bits.stride;
        for (int c = 0; c < nc; ++c)
            GB_TRY(check_fits(e, "channel %d: the last integrate call produced %d bit events but kept %d", c, counts[c], stride));
    }
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_CUDA(e, cudaStreamSynchronize(e->stream));  // pinned staging may still be in flight
    GB_TRY(ensure_state(e, s.states, nc, [](NavState& n) { nav_state_init(n.h); }));
    const size_t ne = static_cast<size_t>(nc) * max_events;
    GB_CUDA(e, s.d_events.ensure(ne));
    GB_CUDA(e, s.d_counts.ensure(nc));
    GB_CUDA(e, s.h_counts.ensure(nc));
    GB_CUDA(e, s.d_bit_counts.ensure(nc));
    GB_TRY(upload(e, s.d_bit_counts.p, counts, nc, s.h_bit_counts));
    NavArgs a{};
    a.bits = bits_device ? static_cast<const BitEvent*>(bits_device) : t->bits.d_events.p;
    a.counts = s.d_bit_counts.p;
    a.bit_states = bits_device ? nullptr : t->bits.states.p;
    a.states = s.states.p;
    a.events = s.d_events.p;
    a.event_counts = s.d_counts.p;
    a.stride = stride;
    a.n_channels = nc;
    a.max_events = max_events;
    GB_LAUNCH(e, -1, launch_decode_subframes(a, e->stream));
    GB_TRY(fetch_output(e, nc, s.d_counts, s.h_counts, counts_host, [&]() -> int {
        return download(e, reinterpret_cast<SubframeEvent*>(events_host), s.d_events.p, ne, s.h_events);
    }));
    t->chain.decoded(s.h_counts.p, nc, max_events, !bits_device);
    return GB200_OK;
}

int gb200_tracker_subframe_state(gb200_tracker* t, int channel, int64_t out[6]) {
    if (!t) return GB200_EINVAL;
    GB_TRY(check_channel(t, channel));
    if (!out) GB_FAIL(t->e, GB200_EINVAL, "null output");
    NavHead h;
    nav_state_init(h);
    GB_TRY(read_state(t->e, &h, t->nav.states, channel, sizeof(NavHead)));
    const int64_t v[6] = {h.phase, h.emitted, h.polarity, h.qlen, h.stopped, h.bits};
    memcpy(out, v, sizeof(v));
    return GB200_OK;
}

int gb200_tracker_parse_subframes(gb200_tracker* t, const void* events_device, const int32_t* counts_host, int32_t stride,
                                  const int32_t* event_ms_host, const int32_t* drop_ms_host, int32_t n_ms,
                                  gb200_subframe_fields* fields_host, int32_t max_fields, int32_t* field_counts_host) {
    if (!t) return GB200_EINVAL;
    gb200_engine* e = t->e;
    auto& s = t->orbit;
    const TrackerChain::Output& sub = t->chain.subframes;
    const int nc = t->n_channels;
    if (!fields_host || !field_counts_host || max_fields < 1) GB_FAIL(e, GB200_EINVAL, "null / empty field buffer");
    for (int c = 0; c < nc; ++c)
        for (int d = 0; d < c; ++d)
            if (t->prn[c] >= 0 && t->prn[c] == t->prn[d])
                GB_FAIL(e, GB200_EINVAL, "channels %d and %d track the same replica row %d (the world model is keyed by satellite)",
                        d, c, t->prn[c]);
    const int* counts = counts_host;
    if (events_device) {
        if (!counts_host || !event_ms_host || !drop_ms_host || stride < 1 || n_ms < 1)
            GB_FAIL(e, GB200_EINVAL, "subframe events need their counts, milliseconds, drops, a stride >= 1 and n_ms >= 1");
        for (int c = 0; c < nc; ++c) {
            GB_TRY(check_fits(e, "channel %d: %d events do not fit a stride of %d", c, counts[c], stride));
            if (drop_ms_host[c] < -1 || drop_ms_host[c] >= n_ms)
                GB_FAIL(e, GB200_EINVAL, "channel %d: drop millisecond %d outside [-1, %d)", c, drop_ms_host[c], n_ms);
            for (int j = 0; j < counts[c]; ++j) {
                const int m = event_ms_host[static_cast<size_t>(c) * stride + j];
                const int prev = j ? event_ms_host[static_cast<size_t>(c) * stride + j - 1] : 0;
                if (m < prev || m >= n_ms)
                    GB_FAIL(e, GB200_EINVAL, "channel %d: event %d's millisecond %d is out of order or outside [0, %d)", c, j, m, n_ms);
            }
        }
    } else {
        if (!t->chain.subframes_on_chain())
            GB_FAIL(e, GB200_ESTATE, "no unparsed subframe events of a process -> integrate_bits -> decode_subframes chain on the device");
        counts = sub.counts.data();
        stride = sub.stride;
        n_ms = sub.n_ms;
        for (int c = 0; c < nc; ++c)
            GB_TRY(check_fits(e, "channel %d: the last decode call produced %d events but kept %d", c, counts[c], stride));
    }
    GB_CUDA(e, cudaSetDevice(e->device));
    GB_CUDA(e, cudaStreamSynchronize(e->stream));  // pinned staging may still be in flight
    GB_TRY(ensure_state(e, s.states, nc, [](OrbitSnap& o) { orbit_state_init(o); }));
    const size_t nf = static_cast<size_t>(nc) * stride;
    GB_CUDA(e, s.d_fields.ensure(nf));
    GB_CUDA(e, s.d_changes.ensure(static_cast<size_t>(nc) * (stride + 2)));
    GB_CUDA(e, s.d_field_counts.ensure(nc));
    GB_CUDA(e, s.d_change_counts.ensure(nc));
    GB_CUDA(e, s.h_field_counts.ensure(nc));
    GB_CUDA(e, s.d_counts.ensure(nc));
    GB_TRY(upload(e, s.d_counts.p, counts, nc, s.h_counts));
    OrbitArgs a{};
    if (events_device) {
        GB_CUDA(e, s.d_event_ms.ensure(nf));
        GB_CUDA(e, s.d_drop_ms.ensure(nc));
        GB_TRY(upload(e, s.d_event_ms.p, event_ms_host, nf, s.h_event_ms));
        GB_TRY(upload(e, s.d_drop_ms.p, drop_ms_host, nc, s.h_drop_ms));
        a.events = static_cast<const SubframeEvent*>(events_device);
        a.event_ms = s.d_event_ms.p;
        a.drop_ms = s.d_drop_ms.p;
    } else {
        a.events = t->nav.d_events.p;
        a.bits = t->bits.d_events.p;
        a.bit_stride = t->chain.bits.stride;
        a.records = t->d_out.p;
    }
    a.counts = s.d_counts.p;
    a.states = s.states.p;
    a.fields = s.d_fields.p;
    a.field_counts = s.d_field_counts.p;
    a.changes = s.d_changes.p;
    a.change_counts = s.d_change_counts.p;
    a.stride = stride;
    a.n_ms = n_ms;
    a.n_channels = nc;
    GB_LAUNCH(e, -1, launch_parse_subframes(a, e->stream));
    // the fields are [channel][stride] on the device and [channel][max_fields] for the caller
    const int keep = std::min<int>(stride, max_fields);
    GB_TRY(fetch_output(e, nc, s.d_field_counts, s.h_field_counts, field_counts_host, [&]() -> int {
        GB_CUDA(e, cudaStreamSynchronize(e->stream));
        GB_CUDA(e, cudaMemcpy2DAsync(fields_host, sizeof(SubframeFields) * max_fields, s.d_fields.p, sizeof(SubframeFields) * stride,
                                     sizeof(SubframeFields) * keep, nc, cudaMemcpyDeviceToHost, e->stream));
        GB_CUDA(e, cudaStreamSynchronize(e->stream));
        return GB200_OK;
    }));
    t->chain.parsed(n_ms, stride + 2, !events_device, t->fix.bank.p != nullptr);
    return GB200_OK;
}

int gb200_tracker_orbit_state(gb200_tracker* t, int channel, double params[26], uint32_t* set_mask, int64_t* prn_count,
                              int32_t* counting) {
    if (!t) return GB200_EINVAL;
    GB_TRY(check_channel(t, channel));
    OrbitSnap s;
    orbit_state_init(s);
    GB_TRY(read_state(t->e, &s, t->orbit.states, channel));
    if (params) memcpy(params, s.p, sizeof(s.p));
    if (set_mask) *set_mask = s.set;
    if (prn_count) *prn_count = s.count;
    if (counting) *counting = s.counting;
    return GB200_OK;
}

int gb200_tracker_chain_sizes(const gb200_tracker* t, int32_t out[3]) {
    if (!t) return GB200_EINVAL;
    if (!out) GB_FAIL(t->e, GB200_EINVAL, "null output");
    out[0] = t->chain.bits.stride;
    out[1] = t->chain.subframes.stride;
    out[2] = t->chain.orbit.n_ms;
    return GB200_OK;
}

static int observations_launch(gb200_tracker* t, SvObservation* out_dev) {
    gb200_engine* e = t->e;
    const TrackerChain::Output& orbit = t->chain.orbit;
    if (!orbit.n_ms) GB_FAIL(e, GB200_ESTATE, "no gb200_tracker_parse_subframes call yet");
    GB_LAUNCH(e, -1, launch_sv_observations(t->orbit.d_changes.p, t->orbit.d_change_counts.p, orbit.stride, t->n_channels,
                                            orbit.n_ms, out_dev, e->stream));
    return GB200_OK;
}

int gb200_tracker_observations_device(gb200_tracker* t, void* out_device) {
    if (!t) return GB200_EINVAL;
    if (!out_device) GB_FAIL(t->e, GB200_EINVAL, "null output");
    GB_CUDA(t->e, cudaSetDevice(t->e->device));
    return observations_launch(t, static_cast<SvObservation*>(out_device));
}

int gb200_tracker_observations(gb200_tracker* t, gb200_sv_observation* out_host) {
    if (!t) return GB200_EINVAL;
    const size_t n = static_cast<size_t>(t->n_channels) * t->chain.orbit.n_ms;
    return launch_to_host(t, out_host, n, t->orbit.d_obs, t->orbit.h_obs,
                          [&](SvObservation* out_dev) { return observations_launch(t, out_dev); });
}

// The observations of the last parse call and the fixes over them (fix.cu), enqueued into out_dev.
static int fixes_launch(gb200_tracker* t, const double* rx_host, FixRecord* out_dev) {
    gb200_engine* e = t->e;
    auto& s = t->fix;
    if (!rx_host) GB_FAIL(e, GB200_EINVAL, "null receiver timestamps");
    if (!t->chain.orbit.n_ms) GB_FAIL(e, GB200_ESTATE, "no gb200_tracker_parse_subframes call yet");
    if (t->chain.fix_gap)
        GB_FAIL(e, GB200_ESTATE, "the fixes of an earlier parse call were skipped: the receiver's clock slide chain has a gap");
    if (!t->chain.fix_pending) GB_FAIL(e, GB200_ESTATE, "the fixes of the last parse call were already computed");
    const int nc = t->n_channels, n_ms = t->chain.orbit.n_ms;
    GB_CUDA(e, cudaStreamSynchronize(e->stream));  // pinned staging may still be in flight
    GB_TRY(ensure_state(e, s.bank, 1, [](FixBank& b) { b.slide = NAN; }));
    GB_TRY(ensure_state(e, s.rank, nc, [](int& r) { r = -1; }));
    GB_CUDA(e, t->orbit.d_obs.ensure(static_cast<size_t>(nc) * n_ms));
    GB_CUDA(e, s.order.ensure(nc));
    GB_CUDA(e, s.touch.ensure(nc));
    GB_CUDA(e, s.prev.ensure(n_ms));
    GB_CUDA(e, s.rx.ensure(n_ms));
    GB_CUDA(e, s.reset.ensure(n_ms));
    GB_CUDA(e, s.slide1.ensure(n_ms));
    GB_TRY(upload(e, s.rx.p, rx_host, n_ms, s.h_rx));
    GB_TRY(observations_launch(t, t->orbit.d_obs.p));
    FixArgs a{};
    a.changes = t->orbit.d_changes.p;
    a.change_counts = t->orbit.d_change_counts.p;
    a.change_stride = t->chain.orbit.stride;
    a.obs = t->orbit.d_obs.p;
    a.rx = s.rx.p;
    a.bank = s.bank.p;
    a.rank = s.rank.p;
    a.order = s.order.p;
    a.touch_ms = s.touch.p;
    a.reset = s.reset.p;
    a.prev = s.prev.p;
    a.slide1 = s.slide1.p;
    a.out = out_dev;
    a.n_channels = nc;
    a.n_ms = n_ms;
    a.solver = s.solver;
    GB_LAUNCH(e, -1, launch_position_fixes(a, e->stream));
    e->launches += 4;  // plan, two passes, repair and finish
    t->chain.fixed();
    return GB200_OK;
}

int gb200_tracker_position_fixes_device(gb200_tracker* t, const double* receiver_timestamps_host, void* out_device) {
    if (!t) return GB200_EINVAL;
    if (!out_device) GB_FAIL(t->e, GB200_EINVAL, "null output");
    GB_CUDA(t->e, cudaSetDevice(t->e->device));
    GB_TRY(fixes_launch(t, receiver_timestamps_host, static_cast<FixRecord*>(out_device)));
    t->fix.kept = false;
    return GB200_OK;
}

int gb200_tracker_position_fixes(gb200_tracker* t, const double* receiver_timestamps_host, gb200_position_fix* out_host) {
    if (!t) return GB200_EINVAL;
    auto& s = t->fix;
    return launch_to_host(t, out_host, t->chain.orbit.n_ms, s.d_fixes, s.h_fixes, [&](FixRecord* out_dev) -> int {
        GB_TRY(fixes_launch(t, receiver_timestamps_host, out_dev));
        s.kept = true;
        return GB200_OK;
    });
}

// The velocity fixes of the last parse call (velocity.cu), enqueued into out_dev.  Reads what the fix call left on the
// device and changes nothing.
static int velocity_launch(gb200_tracker* t, const double* doppler_dev, const void* fixes_dev, VelocityRecord* out_dev) {
    gb200_engine* e = t->e;
    const int n_ms = t->chain.orbit.n_ms;
    if (!n_ms) GB_FAIL(e, GB200_ESTATE, "no gb200_tracker_parse_subframes call yet");
    if (t->chain.fix_pending)
        GB_FAIL(e, GB200_ESTATE, "the position fixes of the last parse call are not computed yet (call gb200_tracker_position_fixes)");
    if (!fixes_dev && !t->fix.kept)
        GB_FAIL(e, GB200_ESTATE, "the last fix call wrote its records to caller memory (gb200_tracker_position_fixes_device): "
                                 "pass that buffer as fixes_device");
    if (!doppler_dev && !t->chain.parse_records)
        GB_FAIL(e, GB200_ESTATE, "the tracking records behind the last parse call are not on the device (it was fed a "
                                 "caller's events, or a later process call replaced them): pass doppler_device");
    VelocityArgs a{};
    a.fixes = fixes_dev ? static_cast<const FixRecord*>(fixes_dev) : t->fix.d_fixes.p;
    a.obs = t->orbit.d_obs.p;
    a.changes = t->orbit.d_changes.p;
    a.change_counts = t->orbit.d_change_counts.p;
    a.change_stride = t->chain.orbit.stride;
    if (doppler_dev) {
        a.doppler = doppler_dev;
        a.doppler_channel_stride = n_ms;
        a.doppler_ms_stride = 1;
    } else {  // TrackMsRecord::doppler of [channel][n_ms] records
        constexpr int kRecordDoubles = sizeof(TrackMsRecord) / sizeof(double);
        a.doppler = &t->d_out.p[0].doppler;
        a.doppler_channel_stride = static_cast<long long>(kRecordDoubles) * n_ms;
        a.doppler_ms_stride = kRecordDoubles;
    }
    a.order = t->fix.order.p;
    a.bank = t->fix.bank.p;
    a.out = out_dev;
    a.n_ms = n_ms;
    GB_LAUNCH(e, -1, launch_velocity_fixes(a, e->stream));
    return GB200_OK;
}

int gb200_tracker_velocity_fixes_device(gb200_tracker* t, const double* doppler_device, const void* fixes_device,
                                        void* out_device) {
    if (!t) return GB200_EINVAL;
    if (!out_device) GB_FAIL(t->e, GB200_EINVAL, "null output");
    GB_CUDA(t->e, cudaSetDevice(t->e->device));
    return velocity_launch(t, doppler_device, fixes_device, static_cast<VelocityRecord*>(out_device));
}

int gb200_tracker_velocity_fixes(gb200_tracker* t, const double* doppler_device, const void* fixes_device,
                                 gb200_velocity_fix* out_host) {
    if (!t) return GB200_EINVAL;
    return launch_to_host(t, out_host, t->chain.orbit.n_ms, t->vel.d_out, t->vel.h_out, [&](VelocityRecord* out_dev) {
        return velocity_launch(t, doppler_device, fixes_device, out_dev);
    });
}

int gb200_tracker_set_fix_solver(gb200_tracker* t, int solver) {
    if (!t) return GB200_EINVAL;
    if (solver != GB200_FIX_SOLVER_REFERENCE && solver != GB200_FIX_SOLVER_LEAST_SQUARES)
        GB_FAIL(t->e, GB200_EINVAL, "unknown fix solver %d", solver);
    // the receiver's stop and slide so far came from the mode they were computed in
    if (t->fix.bank.p) GB_FAIL(t->e, GB200_ESTATE, "the fix solver cannot change after the tracker's first fix call");
    t->fix.solver = solver;
    return GB200_OK;
}

int gb200_tracker_set_code_phase_mode(gb200_tracker* t, int mode) {
    if (!t) return GB200_EINVAL;
    if (mode != GB200_CODE_PHASE_REFERENCE && mode != GB200_CODE_PHASE_SAMPLES)
        GB_FAIL(t->e, GB200_EINVAL, "unknown code-phase mode %d", mode);
    // the channels' accumulators and the integrators' queued stamps already hold the modulus they were computed with
    if (t->tracked) GB_FAIL(t->e, GB200_ESTATE, "the code-phase mode cannot change after the tracker's first tracking call");
    t->code_wrap = mode == GB200_CODE_PHASE_SAMPLES ? static_cast<double>(t->e->N) : kReferenceCodeWrap;
    return GB200_OK;
}

int gb200_tracker_fix_repairs(gb200_tracker* t, int64_t* n) {
    if (!t) return GB200_EINVAL;
    if (!n) GB_FAIL(t->e, GB200_EINVAL, "null output");
    FixBank b{};
    GB_TRY(read_state(t->e, &b, t->fix.bank));
    *n = b.n_repaired;
    return GB200_OK;
}

int gb200_tracker_receiver_state(gb200_tracker* t, double* slide, int32_t* stopped, int32_t* order) {
    if (!t) return GB200_EINVAL;
    gb200_engine* e = t->e;
    const int nc = t->n_channels;
    FixBank b{};
    b.slide = NAN;
    std::vector<int> rank(nc, -1);
    GB_TRY(read_state(e, &b, t->fix.bank));
    // the rank is made after the bank, so read_state has waited for the stream if it exists
    if (t->fix.rank.p) GB_CUDA(e, cudaMemcpy(rank.data(), t->fix.rank.p, sizeof(int) * nc, cudaMemcpyDeviceToHost));
    if (slide) *slide = b.has_slide ? b.slide : NAN;
    if (stopped) *stopped = b.stopped;
    if (order) {
        for (int k = 0; k < nc; ++k) order[k] = -1;
        for (int c = 0; c < nc; ++c)
            if (rank[c] >= 0 && rank[c] < nc) order[rank[c]] = c;
    }
    return GB200_OK;
}

}  // extern "C"
