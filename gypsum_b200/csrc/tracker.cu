// Persistent per-channel tracking kernel (reference gypsum/tracker.py:264-389).
//
// One CTA per channel walks the stream one millisecond at a time: the next 1-ms IQ chunk is prefetched into a
// second shared buffer with cp.async while the current one is processed (double buffering); the carrier is wiped
// off with the channel's current (Doppler, phase); the polyphase forward warp FFTs, the product with the PRN's
// replica spectrum and the inverse warp FFTs run back to back in registers (nothing goes to global memory);
// the early / late correlations of tracker.py:293-295 are just lags p-1 / p+1 of that same circular correlation,
// and the prompt profile of :307-313 is the correlation rolled by p; one thread then runs the float64 loop
// filters (tracker_core.cuh) and the next millisecond starts.  Feedback makes time strictly sequential per
// channel; channels are independent (SURVEY.md 8e).
#include "kernels.cuh"
#include "ptx_helpers.cuh"
#include "tracker_core.cuh"
#include "warp_fft.cuh"

namespace gb {

constexpr int kTrackThreads = 256;

struct TrackPartial {
    float mx;
    int key;  // index in the rolled prompt profile
    int cnt;
    float sum;
    float re, im;
    int pad[2];
};

__device__ __forceinline__ int pymod_int(int a, int m) {
    int r = a % m;
    return r < 0 ? r + m : r;
}

// The float64 loop filters run on one thread; keeping them out of line keeps the per-millisecond instruction
// footprint of the other warps small (the loop body otherwise overflows the instruction cache).
__device__ __noinline__ void track_update_device(TrackState* st, float2 E, float2 L, float2 peak, float strength, int key,
                                                 double t0, const TrackConsts* tc, const double* rtab, TrackMsRecord* out) {
    TrackMsRecord rec;
    track_update(*st, E, L, peak, strength, key, t0, *tc, rtab, rec);
    *out = rec;
}

// Loads the channel state into shared memory (keeping a copy for a later rollback when asked to), the loop constants and
// rtab[n] = 1 / n for the lock-window counts.  The caller's barrier publishes them.
__device__ __forceinline__ void track_prologue(const TrackArgs& a, int ch, TrackState* st, TrackConsts* tc, double* rtab, int tid) {
    const int* src = reinterpret_cast<const int*>(a.states + ch);
    int* dst = reinterpret_cast<int*>(st);
    int* shd = a.shadow ? reinterpret_cast<int*>(a.shadow + ch) : nullptr;
    for (int i = tid; i < static_cast<int>(sizeof(TrackState) / 4); i += kTrackThreads) {
        const int v = src[i];
        dst[i] = v;
        if (shd) shd[i] = v;
    }
    if (tid == 0) *tc = track_consts(a.fs, a.code_wrap);
    rtab[tid] = tid ? 1.0 / static_cast<double>(tid) : 0.0;  // kTrackThreads == 256 entries
}
__device__ __forceinline__ void store_state(const TrackState* st, TrackState* gst, int tid) {
    const int* src = reinterpret_cast<const int*>(st);
    int* dst = reinterpret_cast<int*>(gst);
    for (int i = tid; i < static_cast<int>(sizeof(TrackState) / 4); i += kTrackThreads) dst[i] = src[i];
}

// tracker.py:378: once the channel has stopped, later milliseconds are not processed; each gets this record.
__device__ __forceinline__ void stopped_record(const TrackState* st, TrackMsRecord* out) {
    TrackMsRecord rec = {};
    rec.lost = 2;
    rec.doppler = rec.doppler_hist = st->doppler;
    rec.carrier_phase = rec.carrier_phase_hist = st->carrier_phase;
    rec.code_phase = st->code_phase;
    *out = rec;
}

// Millisecond k's loop parameters from the channel state.
struct MsParams {
    double t0;       // chunk start time
    int pm, kE, kL;  // prompt code phase mod N; early and late lags
    float2 fine;     // this thread's fine carrier factor
};
// Also writes the coarse carrier table: the wipe-off (tracker.py:278-281) exp(-j(2 pi f (n/fs + t0) + phi)) of sample n is
// coarse[n / 256] * fine[n % 256], each factor from a float64-reduced phase.  The caller's barrier publishes the table.
__device__ __forceinline__ MsParams ms_params(const TrackArgs& a, const TrackState* st, int k, int tid, float2* coarse) {
    MsParams ms;
    const double f = st->doppler, phi_cycles = st->carrier_phase * (1.0 / kTau);
    ms.t0 = a.start_times ? a.start_times[k] : a.t0_single;
    const int p = st->code_phase;
    ms.pm = pymod_int(p, a.N);
    ms.kE = pymod_int(p - 1, a.N);
    ms.kL = pymod_int(p + 1, a.N);
    if (tid < (a.N + kTrackThreads - 1) / kTrackThreads)
        coarse[tid] = wipeoff(make_float2(1.f, 0.f), f * (static_cast<double>(tid * kTrackThreads) * a.inv_fs + ms.t0) + phi_cycles);
    ms.fine = carrier_at(f, static_cast<double>(tid), a.inv_fs);
    return ms;
}

// One (branch, parity h) warp's share of the circular correlation of its polyphase row x: forward transform, product with
// the replica half-spectrum, inverse transform, exchange with the other warp of pair `pair` through the tiles, and
// recombination into 16 lags per lane.  tw1, tw2 and crep may be in shared or global memory.
__device__ __forceinline__ void track_correlate(float2 (&x)[32], int lane, int h, int pair, const float2* tw1, const float2* tw2,
                                                const float2* crep, float2* tile, const float2* ptile, float2 (&out16)[16]) {
    if (h) mul_tw2(x, lane, tw2);
    wfft_phase1<false>(x, lane, tw1, tile);
    __syncwarp();
    wfft_phase2<false>(x, lane, tile);
    __syncwarp();
    mul_vec(x, lane, crep + h * kFft);
    wfft_phase1<true>(x, lane, tw1, tile);
    __syncwarp();
    wfft_phase2<true>(x, lane, tile);
    __syncwarp();
    exchange_store(x, lane, h, tile);
    pair_barrier(pair);
    if (h == 0) combine_even(x, lane, tw2, ptile, out16);
    else combine_odd(x, lane, tw2, ptile, out16);
}

// One (branch r, parity h) warp's 16 finished lags per lane: prompt profile statistics in rolled order
// (tracker.py:308-313) into *part, the early / late taps into el, the optional |prompt| profile.
template <int S>
__device__ __forceinline__ void prompt_stats(const float2 (&out16)[16], int lane, int h, int r, int pm, int kE, int kL,
                                             const TrackArgs& a, int slot, int k, float2* el, TrackPartial* part) {
    float mx = -1.f, sum = 0.f, bre = 0.f, bim = 0.f;
    int key = 0x7fffffff, cnt = 0;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
        const int q = lane + 32 * (16 * h + jj);
        if (q < kChips) {
            const int n = S * q + r;
            const float v = gb_mag(out16[jj]);
            int kk = n - pm;
            kk = kk < 0 ? kk + a.N : kk;
            if (v > mx || (v == mx && kk < key)) {
                cnt = v > mx ? 1 : cnt + 1;
                mx = v;
                key = kk;
                bre = out16[jj].x;
                bim = out16[jj].y;
            } else if (v == mx) {
                cnt++;
            }
            sum += v;
            if (n == kE) el[0] = out16[jj];
            if (n == kL) el[1] = out16[jj];
            if (a.profiles) a.profiles[(static_cast<size_t>(slot) * a.n_ms + k) * a.N + kk] = v;
        }
    }
    const int bits = __float_as_int(mx);
    const int mb = __reduce_max_sync(0xffffffffu, bits);
    const bool is = bits == mb;
    const int kmin = __reduce_min_sync(0xffffffffu, is ? key : 0x7fffffff);
    const int ctot = __reduce_add_sync(0xffffffffu, is ? cnt : 0);
    const unsigned owner = __ballot_sync(0xffffffffu, is && key == kmin);
    const int src = __ffs(owner) - 1;
    bre = __shfl_sync(0xffffffffu, bre, src);
    bim = __shfl_sync(0xffffffffu, bim, src);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
    if (lane == 0) {
        TrackPartial pp;
        pp.mx = __int_as_float(mb);
        pp.key = kmin;
        pp.cnt = ctot;
        pp.sum = sum;
        pp.re = bre;
        pp.im = bim;
        pp.pad[0] = pp.pad[1] = 0;
        *part = pp;
    }
}

// Merges the n_parts warp statistics in task order (first index of the maximum wins, as np.argmax), forms the peak
// strength and runs the scalar loop update.
__device__ __forceinline__ void finish_ms(const TrackPartial* partial, int n_parts, int N, TrackState* st, const float2* el,
                                          double t0, const TrackConsts* tc, const double* rtab, TrackMsRecord* out) {
    float mx = -1.f, pre = 0.f, pim = 0.f;
    int key = 0x7fffffff, cnt = 0;
    double sum = 0.0;
    for (int w = 0; w < n_parts; ++w) {
        const TrackPartial pp = partial[w];
        if (pp.mx > mx || (pp.mx == mx && pp.key < key)) {
            cnt = pp.mx > mx ? pp.cnt : cnt + pp.cnt;
            mx = pp.mx;
            key = pp.key;
            pre = pp.re;
            pim = pp.im;
        } else if (pp.mx == mx) {
            cnt += pp.cnt;
        }
        sum += static_cast<double>(pp.sum);
    }
    const float strength = static_cast<float>(record_strength(mx, sum, cnt, N));
    track_update_device(st, el[0], el[1], make_float2(pre, pim), strength, key, t0, tc, rtab, out);
}

template <int S>
__global__ void __launch_bounds__(kTrackThreads, 1) k_track_channels(const TrackArgs a) {
    extern __shared__ __align__(16) float2 smem[];
    constexpr int n_fft_warps = 2 * S;
    float2* iqbuf = smem;                 // [2][N]
    float2* ypoly = iqbuf + 2 * a.N;      // [S][1024]
    float2* crep_s = ypoly + S * kFft;    // [2][1024]
    float2* tw1_s = crep_s + 2 * kFft;
    float2* tw2_s = tw1_s + kFft;
    float2* tiles = tw2_s + kFft;                            // [2s][kTileF2]
    TrackState* st = reinterpret_cast<TrackState*>(tiles + static_cast<size_t>(n_fft_warps) * kTileF2);
    TrackPartial* partial = reinterpret_cast<TrackPartial*>(st + 1);  // [8]
    float2* el = reinterpret_cast<float2*>(partial + 8);              // [2] early, late
    float2* coarse = el + 2;                                          // [16] carrier at samples 0, 256, ... (+ phase)
    uint64_t* mbar = reinterpret_cast<uint64_t*>(coarse + 16);
    double* rtab = reinterpret_cast<double*>(mbar + 2);               // [256] 1 / n for the lock-window counts
    TrackConsts* tc = reinterpret_cast<TrackConsts*>(rtab + 256);

    const int slot = blockIdx.x;                                     // where this CTA's records go
    const int ch = a.channel_idx ? a.channel_idx[slot] : slot;       // which channel's state it advances
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    TrackState* gst = a.states + ch;

    // ---- load the channel state, the twiddles and this PRN's replica spectrum ----
    track_prologue(a, ch, st, tc, rtab, tid);
    if (tid == 0) mbar_init(mbar, 1);
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(mbar, 4 * kFft * sizeof(float2));
        bulk_g2s(tw1_s, a.tw1, kFft * sizeof(float2), mbar);
        bulk_g2s(tw2_s, a.tw2, kFft * sizeof(float2), mbar);
        bulk_g2s(crep_s, a.crep + static_cast<size_t>(st->prn) * 2 * kFft, 2 * kFft * sizeof(float2), mbar);
    }
    mbar_wait(mbar, 0);

    const int chunk16 = a.N / 2;  // 16-byte pieces per 1-ms chunk when N is even
    auto prefetch = [&](int k) {
        const float2* src = a.iq + static_cast<size_t>(k) * a.N;
        float2* dst = iqbuf + (k & 1) * a.N;
        if constexpr (S % 2 == 0) {
            for (int i = tid; i < chunk16; i += kTrackThreads) cp_async16(dst + 2 * i, src + 2 * i);
        } else {  // N = 1023 S is odd: every other millisecond starts 8 bytes past a 16-byte boundary
            for (int i = tid; i < a.N; i += kTrackThreads) cp_async8(dst + i, src + i);
        }
        cp_async_commit();
    };
    if (a.n_ms > 0) prefetch(0);

    const int r = warp >> 1, h = warp & 1;
    float2* tile = tiles + warp * kTileF2;
    const float2* ptile = tiles + (warp ^ 1) * kTileF2;
    TrackMsRecord* out = a.out + static_cast<size_t>(slot) * a.n_ms;

    for (int k = 0; k < a.n_ms; ++k) {
        if (k + 1 < a.n_ms) {
            prefetch(k + 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();  // chunk k landed; the previous millisecond's loop-filter update is visible
        if (st->lost) {
            if (tid == 0) stopped_record(st, &out[k]);
            continue;
        }
        const MsParams ms = ms_params(a, st, k, tid, coarse);
        __syncthreads();
        // ---- carrier wipe-off, polyphase de-interleave ----
        const float2* buf = iqbuf + (k & 1) * a.N;
        for (int kk = 0, n = tid; n < a.N; ++kk, n += kTrackThreads)
            ypoly[(n % S) * kFft + n / S] = cmul(buf[n], cmul(coarse[kk], ms.fine));
        __syncthreads();
        if (tid < S) ypoly[tid * kFft + (kFft - 1)] = ypoly[tid * kFft];
        __syncthreads();

        if (warp < n_fft_warps) {
            float2 x[32], out16[16];
            build_z(x, lane, r, S, ypoly);
            track_correlate(x, lane, h, r, tw1_s, tw2_s, crep_s, tile, ptile, out16);
            prompt_stats<S>(out16, lane, h, r, ms.pm, ms.kE, ms.kL, a, slot, k, el, partial + warp);
        }
        __syncthreads();
        if (tid == 0) finish_ms(partial, n_fft_warps, a.N, st, el, ms.t0, tc, rtab, &out[k]);
        // the __syncthreads at the top of the next millisecond publishes st / frees el, partial
    }
    __syncthreads();
    store_state(st, gst, tid);
}

// ---------------------------------------------------------------------------------------------------------------------
// S >= 5 (5.115 to 16.368 Msps).  The layout above keeps two whole chunks, S rows and 2S tiles at once: 263 KB at S = 5,
// 725 KB at S = 16.  This kernel holds only the S polyphase rows, one tile per warp and the state (111 KB at S = 5,
// 218 KB at S = 16):
//   - the millisecond is read straight from global memory during the wipe-off, with coalesced 8-byte loads issued in
//     batches of 16 per thread (N is odd at S = 5, so odd milliseconds do not start on a 16-byte boundary), while one
//     thread has the TMA unit prefetch the next millisecond into L2; every channel reads the same stream, so the
//     other CTAs find it there as well;
//   - the wiped-off samples go to the S rows in zpos() order and boxcar_column<S> turns them into the S boxcar rows in
//     place, as k_doppler_spectra does;
//   - the 2S (branch, parity) transforms run in ceil(2S / 8) rounds over the 8 warps; a warp pair exchanges through
//     its two tiles as in the kernel above, and a CTA barrier between rounds frees the tiles for the next pair;
//   - twiddles and the replica spectrum (32 KB) are read from global memory through L1: at S = 16 there is no room
//     for them in shared memory.
// The per-task prompt statistics are merged in task order, so the first index of the maximum wins as above.
constexpr int kWideWarps = kTrackThreads / 32;
constexpr int kWideCarrier = 64;  // coarse carrier entries: ceil(16368 / 256)
constexpr int kWideBatch = 16;    // loads in flight per thread during the wipe-off

template <int S>
__global__ void __launch_bounds__(kTrackThreads, 1) k_track_channels_wide(const TrackArgs a) {
    extern __shared__ __align__(16) float2 smem[];
    constexpr int n_tasks = 2 * S, n_rounds = (n_tasks + kWideWarps - 1) / kWideWarps;
    float2* ypoly = smem;                                             // [S][1024], zpos() order
    float2* tiles = ypoly + S * kFft;                                 // [8][kTileF2]
    TrackState* st = reinterpret_cast<TrackState*>(tiles + kWideWarps * kTileF2);
    TrackPartial* partial = reinterpret_cast<TrackPartial*>(st + 1);  // [2S]
    float2* el = reinterpret_cast<float2*>(partial + n_tasks);        // [2] early, late
    float2* coarse = el + 2;                                          // [64] carrier at samples 0, 256, ... (+ phase)
    double* rtab = reinterpret_cast<double*>(coarse + kWideCarrier);  // [256] 1 / n for the lock-window counts
    TrackConsts* tc = reinterpret_cast<TrackConsts*>(rtab + 256);

    const int slot = blockIdx.x;
    const int ch = a.channel_idx ? a.channel_idx[slot] : slot;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    track_prologue(a, ch, st, tc, rtab, tid);
    __syncthreads();
    const float2* crep = a.crep + static_cast<size_t>(st->prn) * 2 * kFft;
    float2* tile = tiles + warp * kTileF2;
    const float2* ptile = tiles + (warp ^ 1) * kTileF2;
    TrackMsRecord* out = a.out + static_cast<size_t>(slot) * a.n_ms;

    for (int k = 0; k < a.n_ms; ++k) {
        if (tid == 0 && k + 1 < a.n_ms) {  // 16-byte aligned part of the next millisecond
            const uintptr_t b = (reinterpret_cast<uintptr_t>(a.iq + static_cast<size_t>(k + 1) * a.N) + 15) & ~uintptr_t(15);
            const uintptr_t e = reinterpret_cast<uintptr_t>(a.iq + static_cast<size_t>(k + 2) * a.N) & ~uintptr_t(15);
            prefetch_l2_bulk(reinterpret_cast<const void*>(b), static_cast<uint32_t>(e - b));
        }
        __syncthreads();  // the previous millisecond's loop-filter update is visible; rows, tiles, el, partial are free
        if (st->lost) {
            if (tid == 0) stopped_record(st, &out[k]);
            continue;
        }
        const MsParams ms = ms_params(a, st, k, tid, coarse);
        __syncthreads();
        // ---- carrier wipe-off, polyphase de-interleave into zpos() rows ----
        const float2* src = a.iq + static_cast<size_t>(k) * a.N;
        for (int k0 = 0; k0 * kTrackThreads < a.N; k0 += kWideBatch) {
            float2 v[kWideBatch];
#pragma unroll
            for (int j = 0; j < kWideBatch; ++j) {
                const int n = tid + (k0 + j) * kTrackThreads;
                v[j] = n < a.N ? src[n] : make_float2(0.f, 0.f);
            }
#pragma unroll
            for (int j = 0; j < kWideBatch; ++j) {
                const int n = tid + (k0 + j) * kTrackThreads;
                if (n < a.N) ypoly[(n % S) * kFft + zpos(n / S)] = cmul(v[j], cmul(coarse[k0 + j], ms.fine));
            }
        }
        __syncthreads();
        if (tid < S) ypoly[tid * kFft + zpos(kFft - 1)] = ypoly[tid * kFft + zpos(0)];
        __syncthreads();
        // in place: rows of y -> rows of boxcar sums z_r (column 1023 is never read as data)
        for (int m0 = 0; m0 < kChips; m0 += kTrackThreads) {
            const int m = m0 + tid;
            float2 z[S];
            if (m < kChips) boxcar_column<S>(ypoly, m, z);
            __syncthreads();
            if (m < kChips) {
#pragma unroll
                for (int r = 0; r < S; ++r) ypoly[r * kFft + zpos(m)] = z[r];
            }
        }
        __syncthreads();
        if (tid < S) ypoly[tid * kFft + zpos(kFft - 1)] = make_float2(0.f, 0.f);  // zero padding of the 1023-point input
        __syncthreads();

        for (int round = 0; round < n_rounds; ++round) {
            const int task = round * kWideWarps + warp;
            if (task < n_tasks) {  // 2S and 8 are even: both warps of a pair are active or neither is
                const int r = task >> 1, h = task & 1;
                float2 x[32], out16[16];
                load_vec(x, lane, ypoly + r * kFft);
                track_correlate(x, lane, h, warp >> 1, a.tw1, a.tw2, crep, tile, ptile, out16);
                prompt_stats<S>(out16, lane, h, r, ms.pm, ms.kE, ms.kL, a, slot, k, el, partial + task);
            }
            if (round + 1 < n_rounds) __syncthreads();  // the partner's tile was read: the next round may overwrite it
        }
        __syncthreads();
        if (tid == 0) finish_ms(partial, n_tasks, a.N, st, el, ms.t0, tc, rtab, &out[k]);
    }
    __syncthreads();
    store_state(st, a.states + ch, tid);
}

// The kernel follows from S alone: k_track_channels while its whole-chunk layout fits (S <= 4), the wide kernel above.
constexpr bool track_wide(int s) { return s >= 5; }
template <int S>
static auto track_kernel() {
    if constexpr (track_wide(S)) return k_track_channels_wide<S>;
    else return k_track_channels<S>;
}

size_t track_smem_bytes(int N, int s) {
    if (track_wide(s))
        return (static_cast<size_t>(s) * kFft + kWideWarps * kTileF2 + 2 + kWideCarrier) * sizeof(float2) + sizeof(TrackState) +
               2 * s * sizeof(TrackPartial) + 256 * sizeof(double) + sizeof(TrackConsts);
    return (2 * static_cast<size_t>(N) + static_cast<size_t>(s) * kFft + 4 * kFft + 2 * static_cast<size_t>(s) * kTileF2) *
               sizeof(float2) +
           sizeof(TrackState) + 8 * sizeof(TrackPartial) + (2 + 16) * sizeof(float2) + 16 + 256 * sizeof(double) + sizeof(TrackConsts);
}

cudaError_t configure_track_kernel() {
    cudaError_t e;
#define GB_ATTR(S) \
    if ((e = cudaFuncSetAttribute(track_kernel<S>(), cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)) != cudaSuccess) return e;
    GB_FOR_EACH_RATE(GB_ATTR)
#undef GB_ATTR
    return cudaSuccess;
}

cudaError_t launch_track_channels(const TrackArgs& a, cudaStream_t st) {
    const size_t sm = track_smem_bytes(a.N, a.s);
    switch (a.s) {
#define GB_CASE(S) case S: track_kernel<S>()<<<a.n_channels, kTrackThreads, sm, st>>>(a); break;
        GB_FOR_EACH_RATE(GB_CASE)
#undef GB_CASE
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

}  // namespace gb
