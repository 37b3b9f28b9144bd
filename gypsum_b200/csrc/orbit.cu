// Subframe fields, the world model's per-satellite state and the per-millisecond satellite time and position on the
// device (orbit_core.cuh), the consumers of the subframe events k_decode_subframes leaves in device memory.
//
// k_parse_subframes: one warp per channel.  The lanes look for the millisecond the channel is dropped at (the first
// tracking record that says `lost`, or the first CannotDetermine event), then lane 0 walks the channel's events in order:
// it parses every subframe, advances the channel's state and writes the state after every change to the change table.
//
// k_sv_observations: one thread per (channel, millisecond), in float64.  It takes the last change at or before its
// millisecond and runs the clock loop (10 iterations of 7 Kepler iterations) and the position: about 90 double-precision
// sin / cos per thread, so it is bound by FP64 issue.
#include "kernels.cuh"
#include "orbit_core.cuh"

namespace gb {

constexpr int kOrbitWarps = 4;
constexpr int kObsThreads = 128;
constexpr unsigned kOrbitFull = 0xffffffffu;

__global__ void __launch_bounds__(kOrbitWarps * 32) k_parse_subframes(const OrbitArgs a) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int ch = blockIdx.x * kOrbitWarps + w;
    if (ch >= a.n_channels) return;  // whole warps only
    const SubframeEvent* ev = a.events + static_cast<size_t>(ch) * a.stride;
    const BitEvent* bits = a.bits ? a.bits + static_cast<size_t>(ch) * a.bit_stride : nullptr;
    const int n = a.counts[ch];
    int drop = -1;
    if (a.drop_ms) {
        drop = a.drop_ms[ch];
    } else {
        // receiver.py:244-255: LostSatelliteLockError from the tracker (tracker.py:378) ...
        const TrackMsRecord* rec = a.records + static_cast<size_t>(ch) * a.n_ms;
        for (int m0 = 0; m0 < a.n_ms; m0 += 32) {
            const int m = m0 + lane;
            const unsigned hit = __ballot_sync(kOrbitFull, m < a.n_ms && rec[m].lost != 0);
            if (hit) {
                drop = m0 + __ffs(hit) - 1;
                break;
            }
        }
        // ... or from the decoder's CannotDetermine (satellite_signal_processing_pipeline.py:142-147)
        for (int j0 = 0; j0 < n; j0 += 32) {
            const int j = j0 + lane;
            const unsigned hit = __ballot_sync(kOrbitFull, j < n && ev[j].kind == kNavCannotDetermine);
            if (hit) {
                const int m = bits[ev[j0 + __ffs(hit) - 1].bit_index].ms_index;
                if (drop < 0 || m < drop) drop = m;
                break;
            }
        }
    }
    if (lane != 0) return;
    OrbitSnap s = a.states[ch];
    const int* ems = a.event_ms ? a.event_ms + static_cast<size_t>(ch) * a.stride : nullptr;
    int n_fields, n_chg;
    orbit_walk(s, ev, n, [&](int j, const SubframeEvent& e) { return ems ? ems[j] : bits[e.bit_index].ms_index; }, drop, a.n_ms,
               a.fields + static_cast<size_t>(ch) * a.stride, n_fields, a.changes + static_cast<size_t>(ch) * (a.stride + 2), n_chg);
    a.change_counts[ch] = n_chg;
    a.field_counts[ch] = n_fields;
    a.states[ch] = s;
}

__global__ void __launch_bounds__(kObsThreads) k_sv_observations(const OrbitSnap* __restrict__ changes,
                                                                   const int* __restrict__ change_counts, int change_stride,
                                                                   int n_ms, SvObservation* __restrict__ out) {
    const int ch = blockIdx.y;
    const int m = blockIdx.x * kObsThreads + threadIdx.x;
    if (m >= n_ms) return;
    SvObservation o;
    orbit_observe(orbit_change_at(changes + static_cast<size_t>(ch) * change_stride, change_counts[ch], m), m, o);
    out[static_cast<size_t>(ch) * n_ms + m] = o;
}

cudaError_t launch_parse_subframes(const OrbitArgs& a, cudaStream_t st) {
    k_parse_subframes<<<(a.n_channels + kOrbitWarps - 1) / kOrbitWarps, kOrbitWarps * 32, 0, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_sv_observations(const OrbitSnap* changes, const int* change_counts, int change_stride, int n_channels,
                                   int n_ms, SvObservation* out, cudaStream_t st) {
    const dim3 grid((n_ms + kObsThreads - 1) / kObsThreads, n_channels);
    k_sv_observations<<<grid, kObsThreads, 0, st>>>(changes, change_counts, change_stride, n_ms, out);
    return cudaGetLastError();
}

}  // namespace gb
