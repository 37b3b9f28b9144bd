// Navigation-message subframe decoding on the device (reference gypsum/navigation_message_decoder.py:173-196), the
// consumer of the bit events k_integrate_bits leaves in device memory: one warp per channel.  The lanes fetch 32 bit
// events at a time and lane 0 runs the sequential state machine of nav_core.cuh on them, with the queue's bit planes in
// shared memory.  A full preamble scan -- when the search (re)starts on a queue that changed by more than one append --
// is warp-parallel: each lane builds the candidate masks of 32 queue positions at a time from funnel shifts of the
// packed planes, and the first candidate with a partner 300 bits later comes from a ballot and __ffs.
#include "kernels.cuh"
#include "nav_core.cuh"

namespace gb {

constexpr int kNavWarps = 4;
constexpr unsigned kFull = 0xffffffffu;

// nav_first_pair over the whole queue with the warp; `scratch` holds one candidate mask per 32 queue positions.
__device__ int warp_first_pair(const NavQueue& q, uint32_t* scratch, int qhead, int qlen, uint32_t pattern, int lane) {
    const int n_chunks = ((qlen - 8) >> 5) + 1;  // candidate positions 0 .. qlen - 8
    for (int k = lane; k < n_chunks; k += 32) {
        const int p0 = (qhead + 32 * k) & (kNavQueueCap - 1);
        const int p1 = (p0 + 32) & (kNavQueueCap - 1);
        const uint32_t w0 = nav_ring_bits(q.val, p0), w1 = nav_ring_bits(q.val, p1);
        const uint32_t k0 = nav_ring_bits(q.known, p0), k1 = nav_ring_bits(q.known, p1);
        uint32_t m = kFull;
#pragma unroll
        for (int t = 0; t < 8; ++t) {
            const uint32_t s = __funnelshift_r(w0, w1, t);  // bit j: queued bit 32k + j + t
            m &= ((pattern >> t) & 1u ? s : ~s) & __funnelshift_r(k0, k1, t);
        }
        const int last = qlen - 8 - 32 * k;  // last valid offset in this chunk
        if (last < 31) m &= (2u << last) - 1u;
        scratch[k] = m;
    }
    __syncwarp();
    int found = -1;
    for (int base = 0; base < n_chunks && found < 0; base += 32) {
        const int k = base + lane;
        uint32_t pair = 0;
        if (k < n_chunks) {
            const uint32_t a = scratch[k];
            const uint32_t b = k + 9 < n_chunks ? scratch[k + 9] : 0u;
            const uint32_t c = k + 10 < n_chunks ? scratch[k + 10] : 0u;
            pair = a & __funnelshift_r(b, c, kSubframeBits - 9 * 32);  // bit j: candidate at 32k + j + 300
        }
        const unsigned hit = __ballot_sync(kFull, pair != 0);
        if (hit) {
            const int first = __ffs(hit) - 1;
            const uint32_t pf = __shfl_sync(kFull, pair, first);
            found = 32 * (base + first) + __ffs(pf) - 1;
        }
    }
    __syncwarp();  // scratch is rewritten by the next scan
    return found;
}

__global__ void __launch_bounds__(kNavWarps * 32) k_decode_subframes(const NavArgs a) {
    __shared__ uint32_t s_val[kNavWarps][kNavQueueWords];
    __shared__ uint32_t s_known[kNavWarps][kNavQueueWords];
    __shared__ uint32_t s_scratch[kNavWarps][kNavQueueWords];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int ch = blockIdx.x * kNavWarps + w;
    if (ch >= a.n_channels) return;  // whole warps only: nothing below synchronises the block
    NavState& st = a.states[ch];
    for (int i = lane; i < kNavQueueWords; i += 32) {
        s_val[w][i] = st.val[i];
        s_known[w][i] = st.known[i];
    }
    __syncwarp();
    const NavQueue q{s_val[w], s_known[w], st.qstart, st.qend};
    NavHead h = st.h;  // lane 0's copy is the decoder; the others only ever read qhead / qlen through shuffles
    const BitEvent* __restrict__ bits = a.bits + static_cast<size_t>(ch) * a.stride;
    SubframeEvent* out = a.events + static_cast<size_t>(ch) * a.max_events;
    const int n = a.counts[ch];
    int n_out = 0;
    for (int k0 = 0; k0 < n; k0 += 32) {
        if (__shfl_sync(kFull, h.stopped, 0)) break;
        const int k = k0 + lane;
        int bv = 0;
        double t0 = 0.0, t1 = 0.0;
        if (k < n) {
            bv = bits[k].bit_value;
            t0 = bits[k].receiver_timestamp;
            t1 = bits[k].trailing_edge_receiver_timestamp;
        }
        const int m = min(32, n - k0);
        for (int j = 0; j < m; ++j) {
            const int bj = __shfl_sync(kFull, bv, j);
            const double t0j = __shfl_sync(kFull, t0, j);
            const double t1j = __shfl_sync(kFull, t1, j);
            const int n_at_bit = n_out;
            int scan = kNavSkip;
            if (lane == 0) scan = nav_push(h, q, bj, t0j, t1j);
            scan = __shfl_sync(kFull, scan, 0);
            int up = -1, inv = -1;
            if (scan == kNavFullScan) {
                const int qhead = __shfl_sync(kFull, h.qhead, 0), qlen = __shfl_sync(kFull, h.qlen, 0);
                __syncwarp();  // lane 0's queue writes
                up = warp_first_pair(q, s_scratch[w], qhead, qlen, kPreambleUp, lane);
                if (up < 0) inv = warp_first_pair(q, s_scratch[w], qhead, qlen, kPreambleInv, lane);
            }
            if (lane == 0) nav_finish(h, q, scan, up, inv, k0 + j, out, a.max_events, n_out, n_at_bit);
        }
    }
    __syncwarp();
    for (int i = lane; i < kNavQueueWords; i += 32) {
        st.val[i] = s_val[w][i];
        st.known[i] = s_known[w][i];
    }
    if (lane == 0) {
        // the tracking channel lost lock (bits_core.cuh `stopped`): no bit will follow the ones decoded here
        if (a.bit_states && a.bit_states[ch].h.stopped && h.stopped == kNavRunning) h.stopped = kNavStopLostLock;
        st.h = h;
        a.event_counts[ch] = n_out;
    }
}

cudaError_t launch_decode_subframes(const NavArgs& a, cudaStream_t st) {
    k_decode_subframes<<<(a.n_channels + kNavWarps - 1) / kNavWarps, kNavWarps * 32, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace gb
