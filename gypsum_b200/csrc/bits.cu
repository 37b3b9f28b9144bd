// Navigation-bit integration on the device (reference gypsum/navigation_bit_intergrator.py:278-288; SURVEY.md 8f N4):
// one warp per tracking channel walks that channel's millisecond records where the tracking kernel left them in HBM.
// The lanes fetch 32 records at a time (symbol, code phase, lost flag + the chunk timestamps) so the sequential state
// machine of bits_core.cuh, which lane 0 runs, pays one memory round trip per 32 symbols; what comes back to the host
// is 50 bit events per channel-second instead of 1000 records.
#include "bits_core.cuh"
#include "kernels.cuh"

namespace gb {

constexpr int kBitWarps = 4;

__global__ void __launch_bounds__(kBitWarps * 32) k_integrate_bits(const BitArgs a) {
    const int lane = threadIdx.x & 31;
    const int ch = blockIdx.x * kBitWarps + (threadIdx.x >> 5);
    if (ch >= a.n_channels) return;
    BitState& st = a.states[ch];
    BitHead h = st.h;  // scalars in registers; the symbol / queue rings stay in global memory behind L1
    const TrackMsRecord* __restrict__ rec = a.records + static_cast<size_t>(ch) * a.n_ms;
    BitEvent* out = a.events + static_cast<size_t>(ch) * a.max_events;
    int n_out = 0;
    int stopped = h.stopped;
    for (int k0 = 0; k0 < a.n_ms; k0 += 32) {
        const int k = k0 + lane;
        int sym = 0, lost = 0;
        double t0 = 0.0, ts = 0.0, te = 0.0;
        if (k < a.n_ms) {
            sym = rec[k].symbol;
            lost = rec[k].lost;
            // tracker.py:319-325: the symbol is stamped with the chunk times delayed by the code phase.  The sums are
            // rounded on their own, as the reference rounds them: a multiply-add fused into one rounding would move
            // some stamps by an ulp.
            const double delay = (static_cast<double>(rec[k].code_phase) / 2046.0) * 0.001;
            t0 = a.start_times[k];
            ts = __dadd_rn(t0, delay);
            te = __dadd_rn(a.end_times[k], delay);
        }
        const int m = min(32, a.n_ms - k0);
        for (int j = 0; j < m; ++j) {
            const int sj = __shfl_sync(0xffffffffu, sym, j);
            const int lj = __shfl_sync(0xffffffffu, lost, j);
            const double t0j = __shfl_sync(0xffffffffu, t0, j);
            const double tsj = __shfl_sync(0xffffffffu, ts, j);
            const double tej = __shfl_sync(0xffffffffu, te, j);
            if (lane == 0 && !stopped) {
                if (lj) stopped = 1;  // LostSatelliteLockError (tracker.py:378): this ms emitted no pseudosymbol
                else bit_step(h, st, sj, t0j, tsj, tej, k0 + j, out, a.max_events, n_out);
            }
        }
    }
    if (lane == 0) {
        h.stopped = stopped;
        st.h = h;
        a.counts[ch] = n_out;
    }
}

cudaError_t launch_integrate_bits(const BitArgs& a, cudaStream_t st) {
    k_integrate_bits<<<(a.n_channels + kBitWarps - 1) / kBitWarps, kBitWarps * 32, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace gb
