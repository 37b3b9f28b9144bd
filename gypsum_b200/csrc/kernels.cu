// sm_90a kernels of the acquisition correlation path (reference: gypsum/utils.py:59-116 driven by
// gypsum/acquisition.py:154-190).  No cuFFT, no tensor cores, no CPU fallback.
//
//   doppler_spectra   per (Doppler, ms): carrier wipe-off (utils.py:93-97), polyphase boxcar, forward warp FFTs.
//                     This half of utils.py:65 does not depend on the PRN, so it is computed once per Doppler
//                     bin and shared by all PRNs instead of being redone per cell as the reference does.
//   correlate_cells   per (PRN, Doppler) cell: x conj(FFT(replica)) (utils.py:69, spectrum staged into shared
//                     memory with a TMA bulk copy), inverse warp FFTs (utils.py:73), |.| accumulation over ms
//                     (utils.py:102-104) in registers, peak/argmax/sum/count reduction with REDUX / warp shuffles
//                     (acquisition.py:181-189, utils.py:111-116).  Two kernels, chosen by launch_correlate:
//                     k_correlate_w2048 (one warp per pruned inverse FFT-2048; every non-coherent, record-only launch)
//                     and k_correlate_cells (a warp pair per transform pair; coherent launches, probes, full profiles).
//   refine_*          planning / selection kernels of the on-device search (acquisition.py:70-152).
#include "kernels.cuh"
#include "ptx_helpers.cuh"
#include "warp_fft.cuh"

namespace gb {

// ---------------------------------------------------------------------------------------------------------
// One-time setup
// ---------------------------------------------------------------------------------------------------------
__global__ void k_init_tables(float2* tw1, float2* tw2) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;  // 0..1023
    if (t >= 1024) return;
    {
        const int k1 = t >> 5, l = t & 31;
        double s, c;
        sincospi(-2.0 * ((l * k1) & 1023) / 1024.0, &s, &c);
        tw1[pidx(k1, l)] = make_float2(static_cast<float>(c), static_cast<float>(s));
    }
    {
        double s, c;
        sincospi(-2.0 * t / 2048.0, &s, &c);
        tw2[zpos(t)] = make_float2(static_cast<float>(c), static_cast<float>(s));
    }
}

// crep[p][g&1][g>>1] = conj(FFT2048(c'_p))[g] / 2048, direct float64 DFT with an exact-phase table (one-time;
// the reference instead recomputes np.fft.fft(prn_replica) on every call, utils.py:66).
__global__ void __launch_bounds__(128) k_replica_spectra(const uint8_t* chips, float2* crep) {
    __shared__ double2 cs[kPad];
    __shared__ uint8_t c[1024];
    const int p = blockIdx.y;
    for (int t = threadIdx.x; t < kPad; t += blockDim.x) {
        double s, co;
        sincospi(2.0 * t / kPad, &s, &co);
        cs[t] = make_double2(co, s);
    }
    for (int t = threadIdx.x; t < kChips; t += blockDim.x) c[t] = chips[p * kChips + t];
    __syncthreads();
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    double re, im;
    replica_spectrum_bin(c, g, cs, re, im);
    crep[(static_cast<size_t>(p) * 2 + (g & 1)) * kFft + zpos(g >> 1)] = make_float2(static_cast<float>(re), static_cast<float>(im));
}

// ---------------------------------------------------------------------------------------------------------
// doppler_spectra
// ---------------------------------------------------------------------------------------------------------
// One warp per (polyphase branch, bin parity) task, at most 8: a 2.046 Msps millisecond (4 tasks) gets a 128-thread
// CTA so four CTAs share an SM.
__host__ __device__ constexpr int spec_warps(int s) { return 2 * s >= 8 ? 8 : 2 * s; }
constexpr int kCarrierTable = 64;  // >= ceil(N / threads) for every supported rate

// When every (branch, parity) task has its own warp (2S <= 8) the transpose tiles take the place of the polyphase rows,
// which are dead once every warp holds its vector in registers: 35 KB instead of 52 KB per 2.046 Msps CTA and, with the
// register cap of five CTAs per SM, the 1312 units of a 32-block batch run in two waves instead of three.
__host__ __device__ constexpr bool spec_alias(int s) { return 2 * s <= 8; }
__host__ __device__ constexpr int spec_f2(int s) {  // float2 of rows + tiles
    return spec_alias(s) ? (s * kFft > spec_warps(s) * kTileF2 ? s * kFft : spec_warps(s) * kTileF2)
                         : s * kFft + spec_warps(s) * kTileF2;
}

template <int S>
__global__ void __launch_bounds__(spec_warps(S) * 32, S == 2 ? 5 : 1) k_doppler_spectra(const SpectraArgs a) {
    constexpr int kSpecWarps = spec_warps(S);
    constexpr int kSpecThreads = kSpecWarps * 32;
    extern __shared__ __align__(16) float2 smem[];
    float2* ypoly = smem;                                       // [S][1024], rows in zpos() order
    float2* tiles = spec_alias(S) ? smem : smem + S * kFft;     // [kSpecWarps][kTileF2]
    float2* coarse = smem + spec_f2(S);                         // [kCarrierTable] carrier at samples 0, 256, 512, ...

    const int unit = blockIdx.x / a.M, i = blockIdx.x % a.M;
    const int b = unit / a.n_doppler, d = unit % a.n_doppler;
    // (No early griddepcontrol.launch_dependents here: it let the FIRST dependent launch of a fresh engine read the
    // spectra before they were written; the implicit trigger at grid completion keeps the launch-latency overlap and is
    // correct.)
    const double f = a.doppler[d];
    if (isnan(f)) return;  // slot switched off by the on-device search planner
    const float2* __restrict__ src = a.iq + static_cast<size_t>(b) * a.block_stride + static_cast<size_t>(i) * a.N;
    const int tid = threadIdx.x;

    // Carrier exp(-j 2 pi f (n + i N)/fs) (utils.py:93-96) as coarse[n / 256] * fine[n % 256]: both factors get an
    // exact float64-reduced phase, so there is one sincos per thread instead of one per sample and no recurrence
    // error growth.
    constexpr int kIter = (kChips * S + kSpecThreads - 1) / kSpecThreads;  // samples per thread (16 for every S but 16: 64)
    // coalesced float2 loads of the 1-ms IQ vector, ALL issued before the carrier set-up and the first use (the loop form
    // stalls on every load)
    constexpr int kBatch = kIter < 16 ? kIter : 16;
    float2 v[kBatch];
#pragma unroll
    for (int k = 0; k < kBatch; ++k) {
        const int n = tid + k * kSpecThreads;
        v[k] = n < kChips * S ? src[n] : make_float2(0.f, 0.f);
    }
    if (tid < kIter) coarse[tid] = carrier_at(f, static_cast<double>(tid * kSpecThreads + i * a.N), a.inv_fs);
    const float2 fine = carrier_at(f, static_cast<double>(tid), a.inv_fs);
    __syncthreads();
    // wipe-off; de-interleave by polyphase branch
#pragma unroll
    for (int k = 0; k < kBatch; ++k) {
        const int n = tid + k * kSpecThreads;
        if (n < kChips * S) ypoly[(n % S) * kFft + zpos(n / S)] = cmul(v[k], cmul(coarse[k], fine));
    }
    for (int k = kBatch, n = tid + kBatch * kSpecThreads; n < a.N; ++k, n += kSpecThreads)
        ypoly[(n % S) * kFft + zpos(n / S)] = cmul(src[n], cmul(coarse[k], fine));
    __syncthreads();
    if (tid < S) ypoly[tid * kFft + zpos(kFft - 1)] = ypoly[tid * kFft + zpos(0)];
    __syncthreads();
    // in place: rows of y -> rows of boxcar sums z_r (column 1023 is never read as data)
    if (S > 1) {
        for (int m0 = 0; m0 < kChips; m0 += kSpecThreads) {
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
    }
    if (tid < S) ypoly[tid * kFft + zpos(kFft - 1)] = make_float2(0.f, 0.f);  // zero padding of the 1023-point input
    __syncthreads();

    const int warp = tid >> 5, lane = tid & 31;
    float2* tile = tiles + warp * kTileF2;
    float2* __restrict__ dst0 = a.spec + (static_cast<size_t>(unit) * a.M + i) * S * 2 * kFft;
    for (int task = warp; task < 2 * S; task += kSpecWarps) {
        const int r = task >> 1, half = task & 1;
        float2 x[32];
        load_vec(x, lane, ypoly + r * kFft);
        if (spec_alias(S)) __syncthreads();  // single pass (one task per warp): the rows are dead, the tiles may take their place
        if (half) mul_tw2(x, lane, a.tw2);
        wfft_phase1<false>(x, lane, a.tw1, tile);
        __syncwarp();
        wfft_phase2<false>(x, lane, tile);
        __syncwarp();
        store_vec(x, lane, dst0 + static_cast<size_t>(task) * kFft);
    }
}

// ---------------------------------------------------------------------------------------------------------
// correlate_cells
// ---------------------------------------------------------------------------------------------------------
// Both correlate kernels walk a contiguous range of groups per CTA; every slot (warp pair or warp) of the CTA takes one
// cell of a group, all on the group's PRN.
struct GroupCell {
    int prn, unit, out;  // PRN, spectrum unit, record slot
    bool active;         // the slot has a cell and the gate has not switched it off
};

// Decodes group g for the slot working on cell my_cell of it.  Grid mode: the group is chunk chunk0 + gch of PRN list entry
// gpl, a chunk being cells_per_group consecutive cells of the PRN's flat (block, Doppler) list; gpl / gch then step to the
// next group, with n_chunks chunks per PRN.  List mode reads the sorted group and cell tables.
__device__ __forceinline__ GroupCell decode_group(const CorrelateArgs& a, int g, int cells_per_group, int my_cell, int chunk0,
                                                  int n_chunks, int& gpl, int& gch) {
    GroupCell gc;
    int n_cells;
    gc.unit = gc.out = 0;
    if (a.grid_mode) {
        gc.prn = a.prn_idx[gpl];
        const int first = (chunk0 + gch) * cells_per_group;
        n_cells = min(cells_per_group, a.n_blocks * a.D - first);
        const int c = first + my_cell;
        const int b = c / a.D, d = c - b * a.D;
        gc.unit = c;  // = b * D + d
        gc.out = (b * a.P + gpl) * a.D + d;
        if (++gch == n_chunks) {
            gch = 0;
            ++gpl;
        }
    } else {
        gc.prn = a.grp_prn[g];
        n_cells = a.grp_count[g];
        if (my_cell < n_cells) {
            const int c = a.grp_first[g] + my_cell;
            gc.unit = a.cell_u[c];
            gc.out = a.cell_out[c];
        }
    }
    gc.active = my_cell < n_cells;
    if (gc.active && a.cell_gate) gc.active = !isnan(a.cell_gate[gc.out]);
    return gc;
}

// Stages conj(FFT(replica)) of a new PRN into crep_s with a TMA bulk copy once every warp is done with the previous one, then
// de-phases the warps by stagger_ns: warps that restart in step after the CTA-wide barrier convoy on the shared-memory pipe.
__device__ __forceinline__ void stage_replica(const CorrelateArgs& a, int prn, float2* crep_s, uint64_t* mbar, uint32_t& parity,
                                              unsigned stagger_ns) {
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(mbar, 2 * kFft * sizeof(float2));
        bulk_g2s(crep_s, a.crep + static_cast<size_t>(prn) * 2 * kFft, 2 * kFft * sizeof(float2), mbar);
    }
    mbar_wait(mbar, parity);
    parity ^= 1;
    __nanosleep(stagger_ns);
}

constexpr int kPairs = 8;  // warp pairs per k_correlate_cells CTA

template <int KIND, bool PROFILE>
__global__ void __launch_bounds__(kPairs * 64, 1) k_correlate_cells(const CorrelateArgs a) {
    extern __shared__ __align__(16) float2 smem[];
    float2* crep_s = smem;                 // [2][1024]
    float2* tw1_s = crep_s + 2 * kFft;     // [32][32]
    float2* tw2_s = tw1_s + kFft;          // [1024]
    float2* tiles = tw2_s + kFft;          // [2*kPairs][kTileF2]
    PeakPartial* partial = reinterpret_cast<PeakPartial*>(tiles + 2 * kPairs * kTileF2);  // [2*kPairs]
    uint64_t* mbar = reinterpret_cast<uint64_t*>(partial + 2 * kPairs);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int pair = warp >> 1, h = warp & 1;
    float2* tile = tiles + warp * kTileF2;
    const float2* ptile = tiles + (warp ^ 1) * kTileF2;

    uint32_t parity = 0;
    if (threadIdx.x == 0) mbar_init(mbar, 1);
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(mbar, 2 * kFft * sizeof(float2));
        bulk_g2s(tw1_s, a.tw1, kFft * sizeof(float2), mbar);
        bulk_g2s(tw2_s, a.tw2, kFft * sizeof(float2), mbar);
    }
    mbar_wait(mbar, parity);
    parity ^= 1;
    const int cells_per_group = kPairs / a.rsplit;
    const int r_per_pair = a.s / a.rsplit;
    const int my_cell = pair / a.rsplit;  // cell slot inside the group
    const int my_r0 = (pair % a.rsplit) * r_per_pair;
    const size_t unit_stride = static_cast<size_t>(a.M) * a.s * 2 * kFft;
    int cur_prn = -1;

    // Each CTA walks a contiguous range of groups: consecutive groups share the PRN, so the replica spectrum is
    // re-staged only when the PRN changes, and the (block, prn, chunk) decode is incremental.
    const int g0 = static_cast<int>(static_cast<long long>(blockIdx.x) * a.n_groups / gridDim.x);
    const int g1 = static_cast<int>(static_cast<long long>(blockIdx.x + 1) * a.n_groups / gridDim.x);
    // grid mode: groups are ordered (PRN, chunk of the PRN's n_blocks*D cells), so a CTA's contiguous range stays on
    // one PRN for many groups and only the last chunk of a PRN is partly filled
    int gpl = 0, gch = 0;
    if (a.grid_mode && g0 < g1) {
        gpl = g0 / a.chunks;
        gch = g0 - gpl * a.chunks;
    }

    for (int g = g0; g < g1; ++g) {
        const GroupCell gc = decode_group(a, g, cells_per_group, my_cell, 0, a.chunks, gpl, gch);
        const bool active = gc.active;
        const int unit = gc.unit, out = gc.out;
        if (gc.prn != cur_prn) {
            stage_replica(a, gc.prn, crep_s, mbar, parity, pair * 300);
            cur_prn = gc.prn;
        }

        if (active) {
            Peak pk;
            peak_init(pk);
            float pr_re = 0.f, pr_im = 0.f;
            int probe = -1;
            if (KIND == kKindCoherent && a.cell_probe) probe = a.cell_probe[out];
            const float2* __restrict__ spec_u = a.spec + static_cast<size_t>(unit) * unit_stride;
            const float2* crep_h = crep_s + h * kFft;
            for (int r = my_r0; r < my_r0 + r_per_pair; ++r) {
                float acc[16];
#pragma unroll
                for (int jj = 0; jj < 16; ++jj) acc[jj] = 0.f;
                const int n_iter = KIND == kKindCoherent ? 1 : a.M;
                for (int it = 0; it < n_iter; ++it) {
                    float2 x[32];
                    if (KIND == kKindCoherent) {
                        // Coherent integration (utils.py:102) commutes with the linear correlation: sum the
                        // M spectra first, transform once.
#pragma unroll
                        for (int j = 0; j < 32; ++j) x[j] = make_float2(0.f, 0.f);
                        for (int i = 0; i < a.M; ++i) {
                            const float2* __restrict__ p = spec_u + (static_cast<size_t>(i * a.s + r) * 2 + h) * kFft;
#pragma unroll
                            for (int jp = 0; jp < 16; ++jp) {
                                float2 v0, v1;
                                ld_pair(p + 2 * (jp * 32 + lane), v0, v1);
                                x[2 * jp] = c_add(x[2 * jp], v0);
                                x[2 * jp + 1] = c_add(x[2 * jp + 1], v1);
                            }
                        }
                        mul_vec(x, lane, crep_h);
                    } else {
                        const float2* __restrict__ p = spec_u + (static_cast<size_t>(it * a.s + r) * 2 + h) * kFft;
                        load_mul_vec(x, lane, p, crep_h);
                    }
                    wfft_phase1<true>(x, lane, tw1_s, tile);  // inverse warp FFT-1024
                    __syncwarp();
                    wfft_phase2<true>(x, lane, tile);
                    __syncwarp();
                    exchange_store(x, lane, h, tile);
                    pair_barrier(pair);
                    float2 out16[16];
                    if (h == 0) combine_even(x, lane, tw2_s, ptile, out16);
                    else combine_odd(x, lane, tw2_s, ptile, out16);
                    if (KIND == kKindCoherent) {
#pragma unroll
                        for (int jj = 0; jj < 16; ++jj) {
                            acc[jj] = gb_mag(out16[jj]);
                            const int q = lane + 32 * (16 * h + jj);
                            const int n = a.s * q + r;
                            if (n == probe && q < kChips) {
                                pr_re = out16[jj].x;
                                pr_im = out16[jj].y;
                            }
                            if (PROFILE) {
                                if (q < kChips) {
                                    a.profile[2 * n] = out16[jj].x;
                                    a.profile[2 * n + 1] = out16[jj].y;
                                }
                            }
                        }
                    } else {
#pragma unroll
                        for (int jj = 0; jj < 16; ++jj) acc[jj] += gb_mag(out16[jj]);
                    }
                    pair_barrier(pair);  // partner has read my tile; the next phase 1 may overwrite it
                }
                Peak t;
                float fsum;
                thread_peak16(acc, lane, h, a.s, r, t, fsum);
                t.sum = static_cast<double>(fsum);
                peak_merge(pk, t);
                if (PROFILE && KIND != kKindCoherent) {
#pragma unroll
                    for (int jj = 0; jj < 16; ++jj) {
                        const int q = lane + 32 * (16 * h + jj);
                        if (q < kChips) a.profile[a.s * q + r] = acc[jj];
                    }
                }
            }
            warp_reduce_peak(pk);
            if (KIND == kKindCoherent) warp_reduce_probe(pr_re, pr_im);
            if (lane == 0) store_partial(partial + warp, pk, pr_re, pr_im);
        }
        // ---- merge the 2*rsplit warp partials of each cell and write its record ----
        if (a.rsplit == 1) {
            if (active) pair_barrier(pair);
        } else {
            __syncthreads();
        }
        if (active && (pair % a.rsplit) == 0 && h == 0 && lane == 0) {
            float pre, pim;
            const Peak m = merge_partials(partial + warp, 2 * a.rsplit, pre, pim);
            write_record(a.records + out, m, pre, pim);
        }
        if (a.rsplit != 1) __syncthreads();  // partial[] is free again
        // rsplit == 1: the next write to partial[] comes after at least two more pair barriers
    }
}

// ---------------------------------------------------------------------------------------------------------
// correlate_cells, one warp per transform (non-coherent searches).  Same cell / group bookkeeping as above, but a
// single warp owns a whole (cell, polyphase branch): it loads both half-spectra, multiplies by the replica spectrum
// and runs the pruned inverse FFT-2048 of warp_fft.cuh (two FFT-32, 64x32 transpose, one FFT-64 per thread).  Per
// transform pair this moves 40 KB through the shared-memory pipe instead of 52 KB and needs no partner warp: no
// exchange tile, no pair barriers, no recombination twiddles, half the twiddle-table reads.
// ---------------------------------------------------------------------------------------------------------
template <int NW, bool SINGLE_MS>
__global__ void __launch_bounds__(NW * 32, 1) k_correlate_w2048(const CorrelateArgs a) {
    extern __shared__ __align__(16) float2 smem[];
    constexpr int kCrepOdd = kFft;
    float2* crep_s = smem;              // [2][1024]
    float2* tw1_s = crep_s + 2 * kFft;  // [32][32]
    float2* tiles = tw1_s + kFft;       // [NW][kTile64F2]
    PeakPartial* partial = reinterpret_cast<PeakPartial*>(tiles + NW * kTile64F2);  // [NW]
    uint64_t* mbar = reinterpret_cast<uint64_t*>(partial + NW);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float2* tile = tiles + warp * kTile64F2;

    uint32_t parity = 0;
    if (threadIdx.x == 0) mbar_init(mbar, 1);
    __syncthreads();
    if (threadIdx.x == 0) {
        mbar_expect_tx(mbar, kFft * sizeof(float2));
        bulk_g2s(tw1_s, a.tw1, kFft * sizeof(float2), mbar);
    }
    mbar_wait(mbar, parity);
    parity ^= 1;
    asm volatile("griddepcontrol.wait;" ::: "memory");  // PDL against doppler_spectra, see launch_correlate

    const int cells_per_group = NW / a.rsplit;
    const int r_per_warp = a.s / a.rsplit;
    const int my_cell = warp / a.rsplit;
    const int my_r0 = (warp % a.rsplit) * r_per_warp;
    const size_t unit_stride = static_cast<size_t>(a.M) * a.s * 2 * kFft;
    int cur_prn = -1;

    // grid mode: groups are ordered (window, PRN, chunk of the PRN's cells in the window), and every window's groups are cut into
    // one contiguous range per CTA, so a CTA stays on one PRN for many groups and only the last chunk of a PRN is partly
    // filled.  A window is a run of (block, Doppler) units whose spectra fit in L2 with room to spare: all 32 PRN passes over a
    // unit happen while the CTAs are inside the same window, so the unit is fetched from HBM once instead of ~8 times (a
    // 256-block batch carries 344 MB of spectra).  There is no barrier between windows; the split below keeps every CTA within
    // one group of the others over the whole batch.
    const int wch = (a.grid_mode && a.win_chunks > 0 && a.win_chunks < a.chunks) ? a.win_chunks : a.chunks;
    const int n_win = a.grid_mode ? (a.chunks + wch - 1) / wch : 1;
    for (int w = 0; w < n_win; ++w) {
    const int ch_w = a.grid_mode ? min(wch, a.chunks - w * wch) : 0;  // chunks per PRN in this window
    const int ng_w = a.grid_mode ? a.P * ch_w : a.n_groups;
    // even split: every CTA takes ng_w / grid groups, the first ng_w % grid slots one more; the slot numbering starts where the
    // previous window's extras ended, so the extra groups go round the CTAs
    const int n_cta = static_cast<int>(gridDim.x);
    const int per_cta = ng_w / n_cta, extra = ng_w - per_cta * n_cta;
    const int extra_full = a.grid_mode ? (a.P * wch) % n_cta : 0;  // the extras of every window before this one
    const int slot = static_cast<int>((blockIdx.x + n_cta - static_cast<int>((static_cast<long long>(w) * extra_full) % n_cta)) % n_cta);
    int g0 = slot * per_cta + min(slot, extra);
    int g1 = g0 + per_cta + (slot < extra ? 1 : 0);
    if (n_win == 1) {
        // one window (list mode, batches that fit in L2, cells too heavy to window): the proportional split.  Its range starts
        // c * n_groups / grid fall on only grid / gcd(P, grid) distinct offsets within a PRN's cell list (33 for 32 PRNs on 132
        // SMs), so four CTAs on different PRNs walk the same units at the same time.
        g0 = static_cast<int>(static_cast<long long>(blockIdx.x) * ng_w / n_cta);
        g1 = static_cast<int>(static_cast<long long>(blockIdx.x + 1) * ng_w / n_cta);
    }
    int gpl = 0, gch = 0;
    if (a.grid_mode && g0 < g1) {
        gpl = g0 / ch_w;
        gch = g0 - gpl * ch_w;
    }

    for (int g = g0; g < g1; ++g) {
        const GroupCell gc = decode_group(a, g, cells_per_group, my_cell, w * wch, ch_w, gpl, gch);
        const bool active = gc.active;
        const int unit = gc.unit, out = gc.out;
        if (gc.prn != cur_prn) {
            stage_replica(a, gc.prn, crep_s, mbar, parity, (warp >> 2) * a.stag_a + (warp & 3) * a.stag_b);
            cur_prn = gc.prn;
        }

        if (active) {
            Peak pk;
            peak_init(pk);
            const float2* __restrict__ spec_u = a.spec + static_cast<size_t>(unit) * unit_stride;
            for (int r = my_r0; r < my_r0 + r_per_warp; ++r) {
                float acc[32];
#pragma unroll
                for (int k = 0; k < 32; ++k) acc[k] = 0.f;
                const int n_iter = SINGLE_MS ? 1 : a.M;
                for (int it = 0; it < n_iter; ++it) {
                    const float2* __restrict__ p = spec_u + static_cast<size_t>(it * a.s + r) * 2 * kFft;
                    {
                        float2 hx[32];
                        load_mul_vec(hx, lane, p, crep_s);  // even bins
                        w2048_phase1<0>(hx, lane, tw1_s, tile);
                    }
                    {
                        float2 hx[32];
                        load_mul_vec(hx, lane, p + kFft, crep_s + kFft);  // odd bins
                        w2048_phase1<1>(hx, lane, tw1_s, tile);
                    }
                    __syncwarp();
                    float2 x[64];
                    w2048_phase2(x, lane, tile);
                    __syncwarp();  // the tile may be overwritten by the next transform
#pragma unroll
                    for (int k = 0; k < 32; ++k) acc[k] += gb_mag(x[k]);
                }
                // lags q = lane + 32 k: k < 16 and k >= 16 are the two halves thread_peak16 knows as h = 0 / 1
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    float v[16];
#pragma unroll
                    for (int jj = 0; jj < 16; ++jj) v[jj] = acc[16 * hh + jj];
                    Peak t;
                    float fsum;
                    thread_peak16(v, lane, hh, a.s, r, t, fsum);
                    t.sum = static_cast<double>(fsum);
                    peak_merge(pk, t);
                }
            }
            warp_reduce_peak(pk);
            if (lane == 0) {
                if (a.rsplit == 1) write_record(a.records + out, pk, 0.f, 0.f);
                else store_partial(partial + warp, pk, 0.f, 0.f);
            }
        }
        if (a.rsplit != 1) {
            __syncthreads();
            if (active && (warp % a.rsplit) == 0 && lane == 0) {
                float pre, pim;  // no probes in a non-coherent launch
                write_record(a.records + out, merge_partials(partial + warp, a.rsplit, pre, pim), 0.f, 0.f);
            }
            __syncthreads();
        }
    }
    }  // windows
}

// ---------------------------------------------------------------------------------------------------------
// Generic replica (utils.py:59-73 with ANY length-N complex prn_replica, not only chips repeated N/1023 times): the circular
// cross-correlation out[k] = sum_n y[n] conj(p[(n - k) mod N]) evaluated directly, float64 accumulation, one thread per lag.
// Not a hot path -- the receiver only ever passes its own replicas, which take the FFT kernels -- but the public helpers
// accept whatever the reference's do.  N^2 complex multiply-adds: 4.2 M at 2.046 Msps, 268 M at 16.368 Msps.
// ---------------------------------------------------------------------------------------------------------
constexpr int kGenericThreads = 128, kGenericChunk = 1024;
__global__ void __launch_bounds__(kGenericThreads) k_correlate_generic(const float2* iq, const float2* replica, int N, int n_ms,
                                                                        double doppler, double inv_fs, int kind, float* out) {
    __shared__ float2 ys[kGenericChunk];
    const int k = blockIdx.x * kGenericThreads + threadIdx.x;  // lag
    double acc_re = 0.0, acc_im = 0.0, acc_abs = 0.0;
    for (int i = 0; i < n_ms; ++i) {
        double cr = 0.0, ci = 0.0;
        for (int n0 = 0; n0 < N; n0 += kGenericChunk) {
            __syncthreads();
            for (int t = threadIdx.x; t < kGenericChunk && n0 + t < N; t += kGenericThreads) {
                const int n = n0 + t;
                // utils.py:93-97: exp(-j tau f (n + i N) / fs), phase reduced in float64 like every other kernel
                ys[t] = wipeoff(iq[static_cast<size_t>(i) * N + n], doppler * ((static_cast<double>(n) + static_cast<double>(i) * N) * inv_fs));
            }
            __syncthreads();
            if (k < N) {
                const int lim = min(kGenericChunk, N - n0);
                int idx = n0 - k;
                idx = idx < 0 ? idx + N : idx;  // (n - k) mod N for the chunk's first sample
                for (int t = 0; t < lim; ++t) {
                    const float2 y = ys[t], p = replica[idx];
                    cr += static_cast<double>(y.x) * p.x + static_cast<double>(y.y) * p.y;   // y * conj(p)
                    ci += static_cast<double>(y.y) * p.x - static_cast<double>(y.x) * p.y;
                    idx = idx + 1 == N ? 0 : idx + 1;
                }
            }
        }
        acc_re += cr;                           // utils.py:102
        acc_im += ci;
        acc_abs += sqrt(cr * cr + ci * ci);     // utils.py:104
    }
    if (k < N) {
        if (kind == kKindCoherent) {
            out[2 * k] = static_cast<float>(acc_re);
            out[2 * k + 1] = static_cast<float>(acc_im);
        } else {
            out[k] = static_cast<float>(acc_abs);
        }
    }
}
cudaError_t launch_correlate_generic(const float2* iq, const float2* replica, int N, int n_ms, double doppler, double inv_fs,
                                     int kind, float* out, cudaStream_t st) {
    k_correlate_generic<<<(N + kGenericThreads - 1) / kGenericThreads, kGenericThreads, 0, st>>>(iq, replica, N, n_ms, doppler,
                                                                                                  inv_fs, kind, out);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------
// On-device Doppler refinement: the control flow of acquisition.py:70-152 without host round trips.  The
// correlation work of every pass still runs in doppler_spectra / correlate_cells; these kernels only plan the
// next pass's bins and apply the reference's selection rules.
// ---------------------------------------------------------------------------------------------------------
__global__ void k_refine_init(int n_sv, RefineState* st) {
    const int sv = blockIdx.x * blockDim.x + threadIdx.x;
    if (sv >= n_sv) return;
    st[sv].center = 0.0;  // acquisition.py:77
    st[sv].kept_doppler = 0.0;
    st[sv].kept_strength = 0.0;
    st[sv].kept_index = 0;
    st[sv].have_kept = 0;
}

// acquisition.py:163-167: range(int(c - s), int(c + s), int(s / 10)); int() truncates toward zero.
__global__ void k_refine_plan(int n_sv, double spread, const RefineState* st, double* doppler) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_sv * kRefineMaxBins) return;
    const int sv = t / kRefineMaxBins, b = t % kRefineMaxBins;
    const double c = st[sv].center;
    const long long lo = static_cast<long long>(c - spread), hi = static_cast<long long>(c + spread);
    const long long step = static_cast<long long>(spread / 10.0);
    const long long v = lo + b * step;
    doppler[t] = v < hi ? static_cast<double>(v) : nan("");
}

// acquisition.py:179-189 (first bin with the largest profile maximum, its argmax and strength) and :89-101
// (re-centre on this pass's bin; keep the pass with the strictly greatest strength).
__global__ void k_refine_select(int n_sv, int N, const CellRecord* rec, const double* doppler, RefineState* st) {
    const int sv = blockIdx.x * blockDim.x + threadIdx.x;
    if (sv >= n_sv) return;
    int best = -1;
    float best_peak = 0.f;
    for (int b = 0; b < kRefineMaxBins; ++b) {
        const int c = sv * kRefineMaxBins + b;
        if (isnan(doppler[c])) continue;
        if (best < 0 || rec[c].peak > best_peak) {
            best = b;
            best_peak = rec[c].peak;
        }
    }
    if (best < 0) return;
    const CellRecord r = rec[sv * kRefineMaxBins + best];
    const double strength = record_strength(r.peak, r.sum, r.count, N);
    RefineState s = st[sv];
    s.center = doppler[sv * kRefineMaxBins + best];
    if (!s.have_kept || strength > s.kept_strength) {
        s.have_kept = 1;
        s.kept_strength = strength;
        s.kept_doppler = s.center;
        s.kept_index = r.argmax;
    }
    st[sv] = s;
}

// acquisition.py:120-136: one coherent integration per satellite at the kept Doppler, probed at the kept index.
__global__ void k_refine_coherent_plan(int n_sv, const RefineState* st, double* doppler, int* probe) {
    const int sv = blockIdx.x * blockDim.x + threadIdx.x;
    if (sv >= n_sv) return;
    doppler[sv] = st[sv].kept_doppler;
    probe[sv] = st[sv].kept_index;
}

__global__ void k_refine_finalize(int n_sv, const RefineState* st, const CellRecord* rec, RefineResult* out) {
    const int sv = blockIdx.x * blockDim.x + threadIdx.x;
    if (sv >= n_sv) return;
    RefineResult r;
    r.doppler = st[sv].kept_doppler;
    r.strength = st[sv].kept_strength;
    r.probe_re = rec[sv].probe_re;
    r.probe_im = rec[sv].probe_im;
    r.code_phase = st[sv].kept_index;
    r.pad_ = 0;
    out[sv] = r;
}

// acquisition.py:179-189 over every (block, prn) row of a finished grid: first Doppler bin with the largest profile
// maximum, its argmax and strength.  One thread per row (rows are D consecutive records).
__global__ void k_best_bins(int n_rows, int D, int N, const CellRecord* rec, const double* doppler, BestRecord* out) {
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n_rows) return;
    const CellRecord* r = rec + static_cast<size_t>(row) * D;
    int best = 0;
    float best_peak = r[0].peak;
    for (int d = 1; d < D; ++d) {
        const float p = r[d].peak;
        if (p > best_peak) {  // strict: the first bin wins ties (max() over dict order, acquisition.py:180-182)
            best = d;
            best_peak = p;
        }
    }
    const CellRecord w = r[best];
    BestRecord o;
    o.doppler = doppler[best];
    o.strength = record_strength(w.peak, w.sum, w.count, N);
    o.peak = w.peak;
    o.code_phase = w.argmax;
    o.bin = best;
    o.pad_ = 0;
    out[row] = o;
}
cudaError_t launch_best_bins(int n_rows, int D, int N, const CellRecord* rec, const double* doppler, BestRecord* out,
                             cudaStream_t s) {
    k_best_bins<<<(n_rows + 127) / 128, 128, 0, s>>>(n_rows, D, N, rec, doppler, out);
    return cudaGetLastError();
}

cudaError_t launch_refine_init(int n_sv, RefineState* st, cudaStream_t s) {
    k_refine_init<<<(n_sv + 63) / 64, 64, 0, s>>>(n_sv, st);
    return cudaGetLastError();
}
cudaError_t launch_refine_plan(int n_sv, double spread, const RefineState* st, double* doppler, cudaStream_t s) {
    const int n = n_sv * kRefineMaxBins;
    k_refine_plan<<<(n + 127) / 128, 128, 0, s>>>(n_sv, spread, st, doppler);
    return cudaGetLastError();
}
cudaError_t launch_refine_select(int n_sv, int N, const CellRecord* rec, const double* doppler, RefineState* st, cudaStream_t s) {
    k_refine_select<<<(n_sv + 63) / 64, 64, 0, s>>>(n_sv, N, rec, doppler, st);
    return cudaGetLastError();
}
cudaError_t launch_refine_coherent_plan(int n_sv, const RefineState* st, double* doppler, int* probe, cudaStream_t s) {
    k_refine_coherent_plan<<<(n_sv + 63) / 64, 64, 0, s>>>(n_sv, st, doppler, probe);
    return cudaGetLastError();
}
cudaError_t launch_refine_finalize(int n_sv, const RefineState* st, const CellRecord* rec, RefineResult* out, cudaStream_t s) {
    k_refine_finalize<<<(n_sv + 63) / 64, 64, 0, s>>>(n_sv, st, rec, out);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------------
// launch wrappers
// ---------------------------------------------------------------------------------------------------------
size_t spectra_smem_bytes(int s) {
    return (static_cast<size_t>(spec_f2(s)) + kCarrierTable) * sizeof(float2);
}
size_t correlate_smem_bytes() {
    return (4 * static_cast<size_t>(kFft) + 2 * kPairs * kTileF2) * sizeof(float2) + 2 * kPairs * sizeof(PeakPartial) + 16;
}

size_t correlate_w2048_smem_bytes(int nw) {
    return (3 * static_cast<size_t>(kFft) + static_cast<size_t>(nw) * kTile64F2) * sizeof(float2) +
           nw * sizeof(PeakPartial) + 16;
}

bool spectra_supports(int s) {
    switch (s) {
#define GB_CASE(S) case S:
        GB_FOR_EACH_RATE(GB_CASE) return true;
#undef GB_CASE
        default: return false;
    }
}

template <int S>
static cudaError_t spectra_attr() {
    return cudaFuncSetAttribute(k_doppler_spectra<S>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(spectra_smem_bytes(S)));
}
cudaError_t configure_kernels() {
    cudaError_t e;
#define GB_ATTR(S) if ((e = spectra_attr<S>()) != cudaSuccess) return e;
    GB_FOR_EACH_RATE(GB_ATTR)
#undef GB_ATTR
    const int sm = static_cast<int>(correlate_smem_bytes());
    if ((e = cudaFuncSetAttribute(k_correlate_cells<kKindCoherent, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm))) return e;
    if ((e = cudaFuncSetAttribute(k_correlate_cells<kKindCoherent, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm))) return e;
    if ((e = cudaFuncSetAttribute(k_correlate_cells<kKindNonCoherent, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm))) return e;
    if ((e = cudaFuncSetAttribute(k_correlate_w2048<12, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(correlate_w2048_smem_bytes(12)))) != cudaSuccess)
        return e;
    return cudaFuncSetAttribute(k_correlate_w2048<8, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(correlate_w2048_smem_bytes(8)));
}

cudaError_t launch_init_tables(float2* tw1, float2* tw2, cudaStream_t st) {
    k_init_tables<<<4, 256, 0, st>>>(tw1, tw2);
    return cudaGetLastError();
}
cudaError_t launch_replica_spectra(const uint8_t* chips_dev, int n_prn, float2* crep, cudaStream_t st) {
    k_replica_spectra<<<dim3(kPad / 128, n_prn), 128, 0, st>>>(chips_dev, crep);
    return cudaGetLastError();
}
cudaError_t launch_doppler_spectra(const SpectraArgs& a, cudaStream_t st) {
    const int grid = a.n_units * a.M;
    const size_t sm = spectra_smem_bytes(a.s);
    switch (a.s) {
#define GB_CASE(S) case S: k_doppler_spectra<S><<<grid, spec_warps(S) * 32, sm, st>>>(a); break;
        GB_FOR_EACH_RATE(GB_CASE)
#undef GB_CASE
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

// Start stagger of the one-warp kernel's warps after each replica re-stage, in ns: (warp / 4) * row + (warp % 4) * column.
constexpr int kW2048StaggerRowNs = 600, kW2048StaggerColNs = 150;

// Coherent launches, coherent probes and full profiles need the pair kernel; every other launch takes the one-warp kernel,
// which is faster on every record-only shape measured on the H100 (DESIGN.md §4).
static bool pair_kernel(int kind, bool profile) { return kind == kKindCoherent || profile; }

int correlate_slots(int kind, int M, bool profile) {
    if (pair_kernel(kind, profile)) return kPairs;
    return M == 1 ? 12 : 8;  // 8 warps when the 32 accumulators live across the milliseconds
}

// Launch as a programmatic dependent of the previous kernel in the stream (doppler_spectra): the grid may start its
// prologue while the producer drains; it blocks at griddepcontrol.wait until the producer's writes are visible.  Only
// k_correlate_w2048 executes that wait, so only it may be launched this way.
template <class K>
static void launch_dependent(K kernel, const CorrelateArgs& a, int grid, int block, size_t sm, cudaStream_t st) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = sm;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaLaunchKernelEx(&cfg, kernel, a);
}

cudaError_t launch_correlate(const CorrelateArgs& a0, int grid, cudaStream_t st) {
    if (pair_kernel(a0.kind, a0.profile != nullptr)) {
        const size_t sm = correlate_smem_bytes();
        if (a0.kind != kKindCoherent) k_correlate_cells<kKindNonCoherent, true><<<grid, kPairs * 64, sm, st>>>(a0);
        else if (a0.profile) k_correlate_cells<kKindCoherent, true><<<grid, kPairs * 64, sm, st>>>(a0);
        else k_correlate_cells<kKindCoherent, false><<<grid, kPairs * 64, sm, st>>>(a0);
        return cudaGetLastError();
    }
    CorrelateArgs a = a0;
    a.stag_a = kW2048StaggerRowNs;
    a.stag_b = kW2048StaggerColNs;
    if (a.M == 1) launch_dependent(k_correlate_w2048<12, true>, a, grid, 12 * 32, correlate_w2048_smem_bytes(12), st);
    else launch_dependent(k_correlate_w2048<8, false>, a, grid, 8 * 32, correlate_w2048_smem_bytes(8), st);
    return cudaGetLastError();
}

}  // namespace gb
