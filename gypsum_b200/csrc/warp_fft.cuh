// Lane-level building blocks of the warp FFT-1024 and of the polyphase correlation.
//
// Every function here is a pure function of (lane, registers, shared tile) with no warp intrinsics, so the
// same code is compiled for the device kernels (kernels.cu) and for the host lane emulator (tests/emu), which
// runs the 32 lanes of a warp as a loop.  Synchronisation is the caller's job.
//
// Math (DESIGN.md section 3).  A 1-ms replica at N = s*1023 samples is chips repeated s times
// (reference satellite.py:20-31), so the length-N circular correlation of utils.py:59-73 splits exactly into
// s circular correlations of length 1023 against the +-1 chip sequence:
//     corr[s*q + r] = sum_m z_r[m] * c[(m - q) mod 1023],   z_r[m] = sum_{t<s} y[(s*m + r + t) mod N].
// Each length-1023 circular correlation is carried, exactly, by a zero-padded length-2048 linear one, and the
// 2048-point transforms are split radix-2 into two 1024-point warp transforms:
//     forward (input half zero):  Z[2f] = FFT1024(z)[f],  Z[2f+1] = FFT1024(z * W2048^n)[f]
//     inverse (only k < 1024):    out[k] = IFFT1024(Y_even)[k] + W2048^-k * IFFT1024(Y_odd)[k]
// A warp transform holds x[lane + 32 j] in registers: FFT-32 over j, twiddle W1024^(lane*k1), 32x32 transpose
// through a padded shared tile, FFT-32 over lane.  Output X[lane + 32 k2] lands in the same layout.
#pragma once
#include "cplx2.cuh"
#include "fft32_gen.cuh"
#include "gb_common.cuh"

namespace gb {

// Complex values are float2 = (re, im) and all complex arithmetic goes through cplx2.cuh (packed FADD2 / FMUL2 / FFMA2 on the
// device, the same IEEE operations lane by lane on the host): the rounding of a product-sum never depends on a contraction
// the compiler happens to pick in a given inlining context -- all kernels (and the host lane emulator) that run the same
// sequence of operations agree bit for bit, which the parity tests rely on.

// Pair-interleaved layout used by every per-thread table and vector (spectra, replica spectra, twiddles, exchange
// tiles, polyphase rows): element j of lane `lane` (i.e. logical index lane + 32 j) sits at pidx(j, lane), so a thread's
// elements (2jp, 2jp+1) are one aligned 16-byte word and a warp access is 512 contiguous bytes: half the load/store
// instructions of a float2 layout, still fully coalesced / conflict-free.
GB_HD GB_INLINE int pidx(int j, int lane) { return (((j >> 1) * 32 + lane) << 1) | (j & 1); }
GB_HD GB_INLINE int zpos(int m) { return pidx(m >> 5, m & 31); }  // logical index m = lane + 32 j

GB_HD GB_INLINE void ld_pair(const float2* p, float2& a, float2& b) {
#if defined(__CUDA_ARCH__)
    const float4 v = *reinterpret_cast<const float4*>(p);
    a = make_float2(v.x, v.y);
    b = make_float2(v.z, v.w);
#else
    a = p[0];
    b = p[1];
#endif
}
GB_HD GB_INLINE void st_pair(float2* p, float2 a, float2 b) {
#if defined(__CUDA_ARCH__)
    *reinterpret_cast<float4*>(p) = make_float4(a.x, a.y, b.x, b.y);
#else
    p[0] = a;
    p[1] = b;
#endif
}

// Phase 1 of the warp FFT-1024.  x[j] = x[lane + 32 j].  Writes u[lane][k1] * W1024^(+-lane k1) to the tile, row k1, column
// lane.  tw1[pidx(k1, lane)] = exp(-2 pi i lane k1 / 1024); the inverse multiplies by its conjugate.
template <bool INV>
GB_HD GB_INLINE void wfft_phase1(float2 (&x)[32], int lane, const float2* tw1, float2* tile) {
    if (INV) fft32_inv(x);
    else fft32_fwd(x);
#pragma unroll
    for (int kp = 0; kp < 16; ++kp) {
        float2 w0, w1;
        ld_pair(tw1 + 2 * (kp * 32 + lane), w0, w1);
        const int k1 = 2 * kp;
        if (kp == 0) tile[lane] = x[0];
        else tile[k1 * kTStride + lane] = INV ? cmulc(x[k1], w0) : cmul(x[k1], w0);
        tile[(k1 + 1) * kTStride + lane] = INV ? cmulc(x[k1 + 1], w1) : cmul(x[k1 + 1], w1);
    }
}
// Phase 2: thread `lane` owns column k1 = lane: reads u[l][lane], l = 0..31, FFT-32 over l.  Afterwards
// x[k2] = X[lane + 32 k2].
template <bool INV>
GB_HD GB_INLINE void wfft_phase2(float2 (&x)[32], int lane, const float2* tile) {
#pragma unroll
    for (int lp = 0; lp < 16; ++lp) ld_pair(tile + lane * kTStride + 2 * lp, x[2 * lp], x[2 * lp + 1]);
    if (INV) fft32_inv(x);
    else fft32_fwd(x);
}

// registers <-> a pair-interleaved vector (global or shared)
GB_HD GB_INLINE void load_vec(float2 (&x)[32], int lane, const float2* v) {
#pragma unroll
    for (int jp = 0; jp < 16; ++jp) ld_pair(v + 2 * (jp * 32 + lane), x[2 * jp], x[2 * jp + 1]);
}
GB_HD GB_INLINE void store_vec(const float2 (&x)[32], int lane, float2* v) {
#pragma unroll
    for (int jp = 0; jp < 16; ++jp) st_pair(v + 2 * (jp * 32 + lane), x[2 * jp], x[2 * jp + 1]);
}
// x[j] *= w[j] for a pair-interleaved vector w (spectrum product, twiddles)
GB_HD GB_INLINE void mul_vec(float2 (&x)[32], int lane, const float2* w) {
#pragma unroll
    for (int jp = 0; jp < 16; ++jp) {
        float2 a, b;
        ld_pair(w + 2 * (jp * 32 + lane), a, b);
        x[2 * jp] = cmul(x[2 * jp], a);
        x[2 * jp + 1] = cmul(x[2 * jp + 1], b);
    }
}
// x = a[j] * w[j]: load a pair-interleaved vector and multiply in one pass (half-spectrum x replica spectrum)
GB_HD GB_INLINE void load_mul_vec(float2 (&x)[32], int lane, const float2* a, const float2* w) {
#pragma unroll
    for (int jp = 0; jp < 16; ++jp) {
        float2 a0, a1, w0, w1;
        ld_pair(a + 2 * (jp * 32 + lane), a0, a1);
        ld_pair(w + 2 * (jp * 32 + lane), w0, w1);
        x[2 * jp] = cmul(a0, w0);
        x[2 * jp + 1] = cmul(a1, w1);
    }
}

// Carrier wipe-off of one sample (utils.py:93-97 / tracker.py:278-281): x * exp(-j 2 pi cycles), with the
// phase reduced to [-0.5, 0.5] cycles in float64 BEFORE going to float32 (SURVEY.md H3).
GB_HD GB_INLINE float2 wipeoff(float2 x, double cycles) {
#if defined(__CUDA_ARCH__)
    const double fr = cycles - rint(cycles);
    float s, c;
    sincospif(2.0f * static_cast<float>(fr), &s, &c);
#else
    const double fr = cycles - __builtin_rint(cycles);
    const double a = 6.283185307179586476925 * static_cast<double>(static_cast<float>(fr));
    const float s = static_cast<float>(__builtin_sin(a)), c = static_cast<float>(__builtin_cos(a));
#endif
    return cmulc(x, make_float2(c, s));  // x * (c - j s)
}

// exp(-j 2 pi frac(f * idx / fs)): the carrier at sample index idx, phase reduced in float64 first.
GB_HD GB_INLINE float2 carrier_at(double f, double idx, double inv_fs) { return wipeoff(make_float2(1.f, 0.f), f * (idx * inv_fs)); }

// All s polyphase boxcar sums of column m at once, from rows stored as ypoly[t][zpos(m')] = y[s*m' + t] (row
// length 1024, column 1023 = copy of column 0 for the circular wrap):
//     z_r[m] = sum_{t>=r} y[s m + t] + sum_{t<r} y[s (m+1) + t].
// The caller reads every column of a round, synchronises, then writes z_r[m] back over ypoly[r][zpos(m)].
template <int S>
GB_HD GB_INLINE void boxcar_column(const float2* ypoly, int m, float2 (&z)[S]) {
    float2 v[S], w[S];
#pragma unroll
    for (int t = 0; t < S; ++t) {
        v[t] = ypoly[t * kFft + zpos(m)];
        w[t] = ypoly[t * kFft + zpos(m + 1)];
    }
    float2 suf[S + 1];
    suf[S] = make_float2(0.f, 0.f);
#pragma unroll
    for (int t = S - 1; t >= 0; --t) suf[t] = c_add(suf[t + 1], v[t]);
    float2 pre = make_float2(0.f, 0.f);
#pragma unroll
    for (int r = 0; r < S; ++r) {
        z[r] = c_add(suf[r], pre);
        pre = c_add(pre, w[r]);
    }
}

// Polyphase boxcar computed directly (tracking kernel, s = 2 or 4): z_r[m] for m = lane + 32 j, from the wiped-off
// millisecond stored linearly as ypoly[t][m'] = y[s*m' + t], row length 1024, ypoly[t][1023] = ypoly[t][0].
GB_HD GB_INLINE void build_z(float2 (&x)[32], int lane, int r, int s, const float2* ypoly) {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        const int m = lane + 32 * j;
        float2 a = make_float2(0.f, 0.f);
        if (m < kChips) {
            for (int t = 0; t < s; ++t) {
                const int rt = r + t;
                const int row = rt >= s ? rt - s : rt;
                a = c_add(a, ypoly[row * kFft + m + (rt >= s ? 1 : 0)]);
            }
        }
        x[j] = a;
    }
}

// x[n] *= W2048^n (forward odd half) for n = lane + 32 j;  tw2[pidx(j, lane)] = exp(-2 pi i n / 2048), n < 1024.
GB_HD GB_INLINE void mul_tw2(float2 (&x)[32], int lane, const float2* tw2) { mul_vec(x, lane, tw2); }

// Fast magnitude: MUFU.SQRT (sqrt.approx, ~1 ulp) on the device instead of the IEEE sequence with its slow path.
GB_HD GB_INLINE float gb_sqrt(float x) {
#if defined(__CUDA_ARCH__)
    float y;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
#else
    return __builtin_sqrtf(x);
#endif
}

GB_HD GB_INLINE float gb_mag(float2 z) { return gb_sqrt(fmaf(z.x, z.x, z.y * z.y)); }  // |re + j im|

// Radix-2 recombination of the two inverse half transforms, out[k] = E[k] + conj(W2048^k) O[k], split so both
// warps of a pair do the same amount of work: the even-bin warp finishes lags k = lane + 32 jj (jj < 16) from
// its own E and the partner's raw O; the odd-bin warp finishes k = lane + 32 (16 + jj) from its own O and the
// partner's E.  `theirs` is the partner's exchange tile ([jj*32 + lane]).
GB_HD GB_INLINE void combine_even(const float2 (&x)[32], int lane, const float2* tw2, const float2* theirs, float2 (&out)[16]) {
#pragma unroll
    for (int p = 0; p < 8; ++p) {
        float2 o0, o1, w0, w1;
        ld_pair(theirs + 2 * (p * 32 + lane), o0, o1);
        ld_pair(tw2 + 2 * (p * 32 + lane), w0, w1);
        out[2 * p] = cfmac(x[2 * p], o0, w0);
        out[2 * p + 1] = cfmac(x[2 * p + 1], o1, w1);
    }
}
GB_HD GB_INLINE void combine_odd(const float2 (&x)[32], int lane, const float2* tw2, const float2* theirs, float2 (&out)[16]) {
#pragma unroll
    for (int p = 0; p < 8; ++p) {
        float2 e0, e1, w0, w1;
        ld_pair(theirs + 2 * (p * 32 + lane), e0, e1);
        ld_pair(tw2 + 2 * ((8 + p) * 32 + lane), w0, w1);
        const int j = 16 + 2 * p;
        out[2 * p] = cfmac(e0, x[j], w0);
        out[2 * p + 1] = cfmac(e1, x[j + 1], w1);
    }
}
// What each warp hands to its partner (pair-interleaved, [pidx(jj, lane)]): the even-bin warp its E[k] for the upper
// lags, the odd-bin warp its raw O[k] for the lower lags.
GB_HD GB_INLINE void exchange_store(const float2 (&x)[32], int lane, int h, float2* mine) {
    if (h == 0) {
#pragma unroll
        for (int p = 0; p < 8; ++p) st_pair(mine + 2 * (p * 32 + lane), x[16 + 2 * p], x[17 + 2 * p]);
    } else {
#pragma unroll
        for (int p = 0; p < 8; ++p) st_pair(mine + 2 * (p * 32 + lane), x[2 * p], x[2 * p + 1]);
    }
}

// Branch-free reduction of one thread's 16 finished lags (q = lane + 32 (16 h + jj), profile index s q + r) into
// (max, first index of max, count of max, sum).  Lag 1023 does not exist (only lane 31, h = 1, jj = 15).
GB_HD GB_INLINE void thread_peak16(const float (&v)[16], int lane, int h, int s, int r, Peak& out, float& fsum) {
    const bool last_invalid = (h == 1) && (lane == 31);
    float m = v[0];
    float sm = v[0];
#pragma unroll
    for (int jj = 1; jj < 15; ++jj) {
        m = fmaxf(m, v[jj]);  // magnitudes: no NaN ordering to preserve; one FMNMX(3) instead of FSETP + FSEL
        sm += v[jj];
    }
    const float v15 = last_invalid ? -1.0f : v[15];
    m = fmaxf(m, v15);
    sm += last_invalid ? 0.0f : v[15];
    int first = 15, c = 0;
    {
        const bool eq = v15 == m;
        c += eq ? 1 : 0;
    }
#pragma unroll
    for (int jj = 14; jj >= 0; --jj) {
        const bool eq = v[jj] == m;
        first = eq ? jj : first;
        c += eq ? 1 : 0;
    }
    out.mx = m;
    out.idx = s * (lane + 32 * (16 * h + first)) + r;
    out.cnt = c;
    out.sum = 0.0;
    fsum = sm;
}

// One thread's 32 finished lags q = lane + 32 k of a whole transform at once (one-warp kernel): the (max, first index of max,
// count of max) of both thread_peak16 halves merged, from a bit mask of the lags equal to the max instead of a running first
// index and count.  fsum[h] is thread_peak16's sum of half h, added in the same order, so the record's float64 sum is unchanged.
GB_HD GB_INLINE void thread_peak32(const float (&v)[32], int lane, int s, int r, Peak& out, float (&fsum)[2]) {
    const bool last_invalid = lane == 31;  // lag 1023
    const float v31 = last_invalid ? -1.0f : v[31];
    float m = v[0], s0 = v[0], s1 = v[16];
#pragma unroll
    for (int k = 1; k < 31; ++k) m = fmaxf(m, v[k]);
    m = fmaxf(m, v31);
#pragma unroll
    for (int k = 1; k < 16; ++k) s0 += v[k];
#pragma unroll
    for (int k = 17; k < 31; ++k) s1 += v[k];
    s1 += last_invalid ? 0.0f : v[31];
    unsigned eq = v31 == m ? 1u << 31 : 0u;
#pragma unroll
    for (int k = 0; k < 31; ++k) eq |= v[k] == m ? 1u << k : 0u;
#if defined(__CUDA_ARCH__)
    const int first = __ffs(eq) - 1, c = __popc(eq);
#else
    const int first = eq ? __builtin_ctz(eq) : -1, c = __builtin_popcount(eq);
#endif
    out.mx = m;
    out.idx = s * (lane + 32 * first) + r;
    out.cnt = c;
    out.sum = 0.0;
    fsum[0] = s0;
    fsum[1] = s1;
}

}  // namespace gb

namespace gb {

// Padded +-1 chip sequence c'[m], m in [0, 2048): c'[m] = c[m] for m < 1023, c'[2048 - t] = c[1023 - t] for
// t = 1..1022, zero at 1023..1025.  A circular length-2048 correlation against c' of a signal supported on
// [0, 1023) equals the circular length-1023 correlation against c (lags 0..1022).
GB_HD GB_INLINE int padded_chip(const uint8_t* chips, int m) {
    if (m < kChips) return chips[m] ? 1 : -1;
    if (m >= kPad - (kChips - 1)) return chips[m - (kPad - kChips)] ? 1 : -1;
    return 0;
}

// conj(FFT2048(c'))[g] / 2048 in float64 from an exact-phase table cs[t] = (cos, sin)(2 pi t / 2048).
// The 1/2048 is the ifft scaling of utils.py:73 folded in.
GB_HD GB_INLINE void replica_spectrum_bin(const uint8_t* chips, int g, const double2* cs, double& re, double& im) {
    double ar = 0.0, ai = 0.0;
    for (int m = 0; m < kPad; ++m) {
        const int c = padded_chip(chips, m);
        if (c == 0) continue;
        const double2 w = cs[(g * m) & (kPad - 1)];  // exp(-2 pi i g m/2048) = cos - j sin; conj -> cos + j sin
        ar += c * w.x;
        ai += c * w.y;
    }
    re = ar / kPad;
    im = ai / kPad;
}

}  // namespace gb

namespace gb {

// ---------------------------------------------------------------------------------------------------------------------
// One-warp inverse FFT-2048 (pruned to the 1024 outputs a padded correlation needs).  n = l' + 64 j'' with
// l' = 2*lane + h: a thread holds, for both bin parities h, the 32 elements Y_h[lane + 32 j''] -- exactly the
// two half-spectra of the pair design, in the same memory layout -- so
//     X[k1 + 32 k2] = sum_{l'} W64^(l' k2) * [ W2048^(l' k1) * sum_{j''} Y[l' + 64 j''] W32^(j'' k1) ]
// is: two in-register FFT-32 (one per parity), twiddle W2048^((2 lane + h) k1) = tw1[k1][lane] * W2048^(h k1) (the
// second factor is a compile-time constant), a 64x32 transpose through the warp's tile, one in-register FFT-64
// over l' per thread (column k1 = lane) of which only outputs k2 < 32 are used.  Output: X[lane + 32 k2] -- the same lag
// layout as before.  No partner warp, no exchange, no recombination twiddles.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kT64Stride = 33;                 // float2 per tile row: consecutive rows hit different banks
constexpr int kTile64F2 = 64 * kT64Stride;     // 64 rows (l') x 32 columns (k1)

// W2048^m, m = 0..31 (forward sign), for the odd-parity twiddle
#define GB_W2048_TABLE                                                                                                  \
    {1.000000000e+00f, 0.000000000e+00f}, {9.999952938e-01f, -3.067956763e-03f}, {9.999811753e-01f, -6.135884649e-03f},  \
    {9.999576446e-01f, -9.203754782e-03f}, {9.999247018e-01f, -1.227153829e-02f}, {9.998823475e-01f, -1.533920628e-02f}, \
    {9.998305818e-01f, -1.840672991e-02f}, {9.997694054e-01f, -2.147408028e-02f}, {9.996988187e-01f, -2.454122852e-02f}, \
    {9.996188225e-01f, -2.760814578e-02f}, {9.995294175e-01f, -3.067480318e-02f}, {9.994306046e-01f, -3.374117185e-02f}, \
    {9.993223846e-01f, -3.680722294e-02f}, {9.992047586e-01f, -3.987292759e-02f}, {9.990777278e-01f, -4.293825693e-02f}, \
    {9.989412932e-01f, -4.600318213e-02f}, {9.987954562e-01f, -4.906767433e-02f}, {9.986402182e-01f, -5.213170468e-02f}, \
    {9.984755806e-01f, -5.519524435e-02f}, {9.983015449e-01f, -5.825826450e-02f}, {9.981181129e-01f, -6.132073630e-02f}, \
    {9.979252862e-01f, -6.438263093e-02f}, {9.977230666e-01f, -6.744391956e-02f}, {9.975114561e-01f, -7.050457339e-02f}, \
    {9.972904567e-01f, -7.356456360e-02f}, {9.970600703e-01f, -7.662386139e-02f}, {9.968202993e-01f, -7.968243797e-02f}, \
    {9.965711458e-01f, -8.274026455e-02f}, {9.963126122e-01f, -8.579731234e-02f}, {9.960447009e-01f, -8.885355258e-02f}, \
    {9.957674145e-01f, -9.190895650e-02f}, {9.954807555e-01f, -9.496349533e-02f}

// Phase 1 for one parity h of the INVERSE transform: x[j] = Y_h[lane + 32 j].  tw1 is the W1024^(lane k1) table
// (pair-interleaved); the inverse multiplies by conjugates.
template <int H>
GB_HD GB_INLINE void w2048_phase1(float2 (&x)[32], int lane, const float2* tw1, float2* tile) {
    constexpr float kW[32][2] = {GB_W2048_TABLE};
    fft32_inv(x);
    float2* row = tile + (H * 32 + lane) * kT64Stride;  // physical row of l' = 2*lane + H
#pragma unroll
    for (int kp = 0; kp < 16; ++kp) {
        float2 w0, w1;
        ld_pair(tw1 + 2 * (kp * 32 + lane), w0, w1);
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            const int k1 = 2 * kp + q;
            float2 w = q ? w1 : w0;
            if (H == 1) w = cmul(w, make_float2(kW[k1][0], kW[k1][1]));
            if (k1 == 0 && H == 0) row[0] = x[0];
            else row[k1] = cmulc(x[k1], w);
        }
    }
}

// The odd-parity twiddle product tw1[k1][lane] * W2048^k1 of w2048_phase1<1> depends on (k1, lane) only.  For k1 = 16..31
// a CTA forms it once into tw1o[pidx(k1 - 16, lane)] (4 KB: what shared memory has left beside 12 tiles), with the same
// complex product, so w2048_phase1_odd reads the same values w2048_phase1<1> computes on every transform.
GB_HD GB_INLINE void w2048_odd_twiddles(int lane, const float2* tw1, float2* tw1o) {
    constexpr float kW[32][2] = {GB_W2048_TABLE};
#pragma unroll
    for (int k1 = 16; k1 < 32; ++k1) tw1o[pidx(k1 - 16, lane)] = cmul(tw1[pidx(k1, lane)], make_float2(kW[k1][0], kW[k1][1]));
}

// w2048_phase1<1> with the products for k1 >= 16 read from w2048_odd_twiddles' table: bit-identical results, 64 fewer FP32
// instructions per transform.
GB_HD GB_INLINE void w2048_phase1_odd(float2 (&x)[32], int lane, const float2* tw1, const float2* tw1o, float2* tile) {
    constexpr float kW[32][2] = {GB_W2048_TABLE};
    fft32_inv(x);
    float2* row = tile + (32 + lane) * kT64Stride;  // physical row of l' = 2*lane + 1
#pragma unroll
    for (int kp = 0; kp < 16; ++kp) {
        float2 w0, w1;
        if (kp < 8) {
            ld_pair(tw1 + 2 * (kp * 32 + lane), w0, w1);
            w0 = cmul(w0, make_float2(kW[2 * kp][0], kW[2 * kp][1]));
            w1 = cmul(w1, make_float2(kW[2 * kp + 1][0], kW[2 * kp + 1][1]));
        } else {
            ld_pair(tw1o + 2 * ((kp - 8) * 32 + lane), w0, w1);
        }
        row[2 * kp] = cmulc(x[2 * kp], w0);
        row[2 * kp + 1] = cmulc(x[2 * kp + 1], w1);
    }
}

// Phase 2: thread `lane` owns column k1 = lane: gathers the 64 rows (l' natural order), inverse FFT-64 over l'.
// Afterwards x[k2] = X[lane + 32 k2]; only k2 < 32 are meaningful for the pruned transform.
GB_HD GB_INLINE void w2048_phase2(float2 (&x)[64], int lane, const float2* tile) {
#pragma unroll
    for (int p = 0; p < 32; ++p) {
        x[2 * p] = tile[p * kT64Stride + lane];             // l' = 2p
        x[2 * p + 1] = tile[(32 + p) * kT64Stride + lane];  // l' = 2p + 1
    }
    fft64_inv(x);
}

}  // namespace gb
