// The literal north-star kernel: ONE block per (PRN, Doppler) cell doing the whole reference pipeline of
// gypsum/utils.py:77-108 -- the 1-ms IQ vector and the PRN's replica spectrum staged into shared memory by TMA
// bulk copies, carrier wipe-off, forward warp FFTs, product with conj(FFT(replica)), inverse warp FFTs, |.|
// (or complex) accumulation over the milliseconds in registers, warp-reduced peak.
//
// Against the de-duplicated pair doppler_spectra + correlate_cells (DESIGN.md section 2.5): the forward half of the
// pipeline does not depend on the PRN, so on a 32-PRN x shared-Doppler grid this kernel redoes every wipe-off and forward
// transform 32 times and loses ~3x; when every cell has its own Doppler (the refinement passes of
// acquisition.py:81-101) nothing can be shared and it wins ~2x because nothing round-trips through HBM.  The engine
// therefore uses it in gb200_detect and, by automatic choice, for cell lists with mostly distinct Dopplers
// (gb200_set_fused overrides); grids always run the split pair.  Parity tests run both.
#include "kernels.cuh"
#include "ptx_helpers.cuh"
#include "warp_fft.cuh"

namespace gb {

// Shared memory per CTA (2.046 Msps): IQ chunk 16 KB + replica spectrum 16 KB + 4 transpose tiles 34 KB = 67 KB, so
// three CTAs (12 transform warps) share an SM.  The polyphase rows live inside the tile area (they are dead once the
// transforms start) and the twiddle tables are read through L1 from global memory (every CTA reads the same 16 KB).
template <int S, int KIND>
__global__ void __launch_bounds__(2 * S * 32, (S == 2 ? 3 : 1)) k_acquire_fused(const FusedArgs a) {
    constexpr int kWarps = 2 * S;
    constexpr int kThreads = kWarps * 32;
    extern __shared__ __align__(16) float2 smem[];
    float2* iqbuf = smem;                  // [N]      one millisecond of IQ (TMA destination)
    float2* crep_s = iqbuf + a.N;          // [2][1024]
    float2* tiles = crep_s + 2 * kFft;     // [2S][kTileF2]
    float2* ypoly = tiles;                 // [S][1024] aliases the tiles: written by the wipe-off, read by build_z only
    const float2* __restrict__ tw1_s = a.tw1;
    const float2* __restrict__ tw2_s = a.tw2;
    PeakPartial* partial = reinterpret_cast<PeakPartial*>(tiles + kWarps * kTileF2);    // [2S]
    float2* coarse = reinterpret_cast<float2*>(partial + kWarps);                      // [32]
    uint64_t* mbar = reinterpret_cast<uint64_t*>(coarse + 32);                          // [2]: tables, IQ chunk

    const int cell = blockIdx.x;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int r = warp >> 1, h = warp & 1;
    const double f = a.doppler[cell];
    if (isnan(f)) return;  // slot switched off by the on-device search planner (uniform for the whole CTA)
    const int prn = a.prn[cell];
    const int probe = (KIND == kKindCoherent && a.probe) ? a.probe[cell] : -1;
    const uint32_t chunk_bytes = static_cast<uint32_t>(a.N) * sizeof(float2);

    if (tid == 0) {
        mbar_init(mbar, 1);
        mbar_init(mbar + 1, 1);
    }
    __syncthreads();
    if (tid == 0) {
        mbar_expect_tx(mbar, 2 * kFft * sizeof(float2));
        bulk_g2s(crep_s, a.crep + static_cast<size_t>(prn) * 2 * kFft, 2 * kFft * sizeof(float2), mbar);
        mbar_expect_tx(mbar + 1, chunk_bytes);
        bulk_g2s(iqbuf, a.iq, chunk_bytes, mbar + 1);  // millisecond 0
    }
    const float2 fine = carrier_at(f, static_cast<double>(tid), a.inv_fs);
    mbar_wait(mbar, 0);

    float2* tile = tiles + warp * kTileF2;
    const float2* ptile = tiles + (warp ^ 1) * kTileF2;
    float acc_re[16], acc_im[16];  // non-coherent: acc_re = sum over ms of |corr|; coherent: complex sum
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) acc_re[jj] = acc_im[jj] = 0.f;

    for (int i = 0; i < a.M; ++i) {
        // carrier exp(-j 2 pi f (n + i N)/fs) = coarse[n / T] * fine[n % T]
        if (tid < (a.N + kThreads - 1) / kThreads)
            coarse[tid] = carrier_at(f, static_cast<double>(tid * kThreads) + static_cast<double>(i) * a.N, a.inv_fs);
        mbar_wait(mbar + 1, i & 1);  // millisecond i has landed in shared memory
        __syncthreads();
        for (int kk = 0, n = tid; n < a.N; ++kk, n += kThreads)
            ypoly[(n % S) * kFft + n / S] = cmul(iqbuf[n], cmul(coarse[kk], fine));
        __syncthreads();  // iqbuf is free: fetch the next millisecond while this one is transformed
        if (tid == 0 && i + 1 < a.M) {
            mbar_expect_tx(mbar + 1, chunk_bytes);
            bulk_g2s(iqbuf, a.iq + static_cast<size_t>(i + 1) * a.N, chunk_bytes, mbar + 1);
        }
        if (tid < S) ypoly[tid * kFft + (kFft - 1)] = ypoly[tid * kFft];
        __syncthreads();

        float2 x[32];
        build_z(x, lane, r, S, ypoly);
        __syncthreads();  // every warp is done with ypoly; the next millisecond may overwrite it
        // forward transform, spectrum product, inverse transform as conj(forward(conj(.))): one copy of the warp-FFT code
#pragma unroll 1
        for (int pass = 0; pass < 2; ++pass) {
            if (pass == 0) {
                if (h) mul_tw2(x, lane, tw2_s);
            } else {
                mul_vec(x, lane, crep_s + h * kFft);
#pragma unroll
                for (int j = 0; j < 32; ++j) x[j].y = -x[j].y;
            }
            wfft_phase1<false>(x, lane, tw1_s, tile);
            __syncwarp();
            wfft_phase2<false>(x, lane, tile);
            __syncwarp();
        }
#pragma unroll
        for (int j = 0; j < 32; ++j) x[j].y = -x[j].y;
        exchange_store(x, lane, h, tile);
        pair_barrier(r);
        float2 out16[16];
        if (h == 0) combine_even(x, lane, tw2_s, ptile, out16);
        else combine_odd(x, lane, tw2_s, ptile, out16);
        if (KIND == kKindCoherent) {
#pragma unroll
            for (int jj = 0; jj < 16; ++jj) {
                acc_re[jj] += out16[jj].x;  // utils.py:102: the complex correlation is summed over the milliseconds
                acc_im[jj] += out16[jj].y;
            }
        } else {
#pragma unroll
            for (int jj = 0; jj < 16; ++jj) acc_re[jj] += gb_mag(out16[jj]);  // utils.py:104
        }
        // the next millisecond's CTA-wide barriers order the tile reuse
    }

    float pr_re = 0.f, pr_im = 0.f;
    float v[16];
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
        if (KIND == kKindCoherent) {
            v[jj] = gb_mag(make_float2(acc_re[jj], acc_im[jj]));
            const int q = lane + 32 * (16 * h + jj);
            if (q < kChips && S * q + r == probe) {
                pr_re = acc_re[jj];
                pr_im = acc_im[jj];
            }
        } else {
            v[jj] = acc_re[jj];
        }
    }
    Peak pk;
    float fsum;
    thread_peak16(v, lane, h, S, r, pk, fsum);
    pk.sum = static_cast<double>(fsum);
    warp_reduce_peak(pk);
    warp_reduce_probe(pr_re, pr_im);
    if (lane == 0) store_partial(partial + warp, pk, pr_re, pr_im);
    __syncthreads();
    if (tid == 0) {
        float pre, pim;
        const Peak m = merge_partials(partial, kWarps, pre, pim);
        write_record(a.records + cell, m, pre, pim);
    }
}

size_t fused_smem_bytes(int N, int s) {
    return (static_cast<size_t>(N) + 2 * kFft + 2 * static_cast<size_t>(s) * kTileF2 + 32) * sizeof(float2) +
           2 * s * sizeof(PeakPartial) + 32;
}

bool fused_supports(int s) { return s == 2 || s == 4; }

cudaError_t configure_fused_kernel() {
    cudaError_t e;
    if ((e = cudaFuncSetAttribute(k_acquire_fused<2, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024))) return e;
    if ((e = cudaFuncSetAttribute(k_acquire_fused<2, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024))) return e;
    if ((e = cudaFuncSetAttribute(k_acquire_fused<4, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024))) return e;
    return cudaFuncSetAttribute(k_acquire_fused<4, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
}

cudaError_t launch_acquire_fused(const FusedArgs& a, int s, int kind, cudaStream_t st) {
    const size_t sm = fused_smem_bytes(a.N, s);
    if (s == 2) {
        if (kind == kKindCoherent) k_acquire_fused<2, 1><<<a.n_cells, 128, sm, st>>>(a);
        else k_acquire_fused<2, 2><<<a.n_cells, 128, sm, st>>>(a);
    } else if (s == 4) {
        if (kind == kKindCoherent) k_acquire_fused<4, 1><<<a.n_cells, 256, sm, st>>>(a);
        else k_acquire_fused<4, 2><<<a.n_cells, 256, sm, st>>>(a);
    } else {
        return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

}  // namespace gb
