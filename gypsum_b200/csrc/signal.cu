// C/N0 and phase-lock windows of every tracking channel (signal_core.cuh), from the tracking records the tracking kernel
// left in device memory.
//
// k_signal_stop: the warps of a channel each scan one stretch of its records, 32 per ballot, for the first record with
// `lost` set (the channel stops there: that record is not counted), and keep the smallest with atomicMin; the first
// one snapshots the channel's carried state.  k_signal_windows: one thread per
// (channel, window of this call).  Window j of a call covers the call's milliseconds [start_j, end_j): window 0 continues
// the window the last call left open with open.n records, so it ends after r = W - open.n of them, and window j > 0 is
// [r + (j-1) W, r + j W).  Each thread walks its milliseconds in order, up to the stop, so its sums are those a walk
// over the whole stream would form; the one window that holds the stop (or the end of the call) writes the channel's
// state back.  The windows a call emits are those it closes, then possibly one a stop cut, so window j goes to output
// slot j.
#include "kernels.cuh"
#include "signal_core.cuh"

namespace gb {

constexpr int kSignalStopWarps = 4;
constexpr int kSignalStopSpan = 1024;  // records one warp of k_signal_stop scans
constexpr int kSignalThreads = 128;
constexpr int kSignalBatch = 8;  // records fetched before they are summed, for memory-level parallelism

__global__ void __launch_bounds__(kSignalStopWarps * 32) k_signal_stop(const SignalArgs a) {
    const int lane = threadIdx.x & 31;
    const int ch = blockIdx.x;
    const int span = blockIdx.y * kSignalStopWarps + (threadIdx.x >> 5);
    const int k_begin = span * kSignalStopSpan;
    if (k_begin >= a.n_ms) return;
    if (span == 0 && lane == 0) a.carried[ch] = a.states[ch];
    if (a.states[ch].stopped) return;
    const int k_end = min(a.n_ms, k_begin + kSignalStopSpan);
    const TrackMsRecord* __restrict__ rec = a.records + static_cast<size_t>(ch) * a.n_ms;
    for (int k0 = k_begin; k0 < k_end; k0 += 32) {
        const int k = k0 + lane;
        const unsigned lost = __ballot_sync(0xffffffffu, k < k_end && __ldg(&rec[k].lost) != 0);
        if (lost) {
            if (lane == 0) atomicMin(a.stop + ch, k0 + __ffs(lost) - 1);
            break;
        }
    }
}

__device__ __forceinline__ void signal_load(const TrackMsRecord* __restrict__ r, float& re, float& im, float& s, int& locked) {
    const float2 p = __ldg(reinterpret_cast<const float2*>(&r->peak_re));
    re = p.x;
    im = p.y;
    s = __ldg(&r->strength);
    locked = __ldg(&r->locked);
}

__global__ void __launch_bounds__(kSignalThreads) k_signal_windows(const SignalArgs a) {
    const int ch = blockIdx.x;
    const int j = blockIdx.y * kSignalThreads + threadIdx.x;
    const SignalState c = a.carried[ch];
    if (c.stopped) {
        if (j == 0) a.counts[ch] = 0;
        return;
    }
    const int W = a.window_ms, n_ms = a.n_ms, stop = min(a.stop[ch], n_ms);
    const int r = W - c.open.n;  // 1..W
    const int start = j == 0 ? 0 : r + (j - 1) * W;
    if (start > stop) return;
    const int end = r + j * W;
    SignalSums s;
    if (j == 0) {
        s = c.open;
    } else {
        signal_sums_clear(s);
    }
    const TrackMsRecord* __restrict__ rec = a.records + static_cast<size_t>(ch) * n_ms;
    const int last = min(end, stop);
    int k = start;
    for (; k + kSignalBatch <= last; k += kSignalBatch) {
        float re[kSignalBatch], im[kSignalBatch], st[kSignalBatch];
        int lk[kSignalBatch];
#pragma unroll
        for (int u = 0; u < kSignalBatch; ++u) signal_load(rec + k + u, re[u], im[u], st[u], lk[u]);
#pragma unroll
        for (int u = 0; u < kSignalBatch; ++u) signal_add(s, re[u], im[u], st[u], lk[u]);
    }
    for (; k < last; ++k) {
        float re, im, st;
        int lk;
        signal_load(rec + k, re, im, st, lk);
        signal_add(s, re, im, st, lk);
    }
    const bool carried = j == 0 && c.open.n > 0;
    const double t0 = carried ? c.t0 : (start < n_ms ? a.start_times[start] : 0.0);
    const long long first = c.consumed + start - (j == 0 ? c.open.n : 0);
    SignalWindow* out = a.out + static_cast<size_t>(ch) * a.max_windows;
    if (end <= stop) {  // closed: W records
        if (j < a.max_windows) out[j] = signal_window(s, t0, first, end - 1, a.floor_dbhz);
        return;
    }
    // this window holds the stop or the end of the call: the channel's state goes back
    SignalState next;
    signal_state_init(next);
    if (stop < n_ms) {  // cut by a stop: emitted if it holds a record; its last one is the stop's predecessor
        const int emitted = s.n > 0 ? 1 : 0;
        if (emitted && j < a.max_windows) out[j] = signal_window(s, t0, first, stop - 1, a.floor_dbhz);
        a.counts[ch] = j + emitted;
        next.consumed = c.consumed + stop;
        next.stopped = 1;
    } else {
        a.counts[ch] = j;
        next.open = s;
        next.t0 = s.n > 0 ? t0 : 0.0;
        next.consumed = c.consumed + n_ms;
    }
    a.states[ch] = next;
}

cudaError_t launch_signal_windows(const SignalArgs& a, cudaStream_t st) {
    // no lost record: the stop stays above every millisecond (0x7f7f7f7f)
    cudaError_t e = cudaMemsetAsync(a.stop, 0x7f, sizeof(int) * a.n_channels, st);
    if (e != cudaSuccess) return e;
    const int spans = (a.n_ms + kSignalStopSpan - 1) / kSignalStopSpan;
    k_signal_stop<<<dim3(a.n_channels, (spans + kSignalStopWarps - 1) / kSignalStopWarps), kSignalStopWarps * 32, 0, st>>>(a);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const dim3 grid(a.n_channels, (signal_max_segments(a.n_ms, a.window_ms) + kSignalThreads - 1) / kSignalThreads);
    k_signal_windows<<<grid, kSignalThreads, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace gb
