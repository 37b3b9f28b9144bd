// Lane-level building blocks of the one-warp exact 1023-point correlation (DESIGN.md section 2, step 2b).
//
// Like warp_fft.cuh, every function is a pure function of (lane, registers, shared tile) with no warp intrinsics, so the host
// lane emulator runs the same code; synchronisation is the caller's job.
//
// Good-Thomas DFT-1023, 1023 = 31 x 33 (coprime, no twiddles).  Time index n = (33 n1 + 31 n2) mod 1023 (n1 < 31, n2 < 33),
// bin k = (528 k1 + 496 k2) mod 1023 (the CRT map: k = k1 mod 31, k = k2 mod 33), and
//     X[k1, k2] = sum_n2 W33^(n2 k2) sum_n1 W31^(n1 k1) x[n1, n2].
// Spectra live in this permuted bin order, pair-interleaved as X[k1, k2] at pidx(k2, k1) (k1 = lane, lane 31 zero).
// The 33-point stage runs one column per lane (lanes 0..30).  The 31-point stage has 33 rows: lane L runs row L, and the
// 33rd row is spread over the warp in the symmetric form (row31_*).
#pragma once
#include "cplx2.cuh"
#include "dft1023_gen.cuh"
#include "warp_fft.cuh"

namespace gb {

constexpr int kPfaStride = 33;   // float2 per tile row: 64-bit row and column accesses are conflict-free
// A warp's tile: 33 x 33 transpose, then the spread row's scratch (its input, a_k, j b_k, the per-lane halves).
constexpr int kPfaSrc = 33 * kPfaStride, kPfaA = kPfaSrc + 32, kPfaB = kPfaA + 16, kPfaX = kPfaB + 16;
constexpr int kPfaTileF2 = kPfaX + 33;  // even, so every warp's tile starts 16-byte aligned
static_assert(kPfaTileF2 % 2 == 0, "tiles hold 16-byte pair loads");

GB_HD GB_INLINE int pfa_lag(int n1, int n2) {  // (33 n1 + 31 n2) mod 1023
    const int q = 33 * n1 + 31 * n2;
    return q >= kChips ? q - kChips : q;
}
GB_HD GB_INLINE int pfa_bin(int k1, int k2) { return (528 * k1 + 496 * k2) % kChips; }

// The spread 31-point row (forward or inverse DFT-31 of src[0..30]).  Lane j = 1..15 forms a_j = x_j + x_{31-j} and
// j b_j = j (x_j - x_{31-j}); then lane 0 sums X_0 = x_0 + sum a_k, lane j the half A_j = x_0 + sum cos a_k and lane 15 + j the
// half j B_j = sum sin (j b_k), each with 15 multiply-adds (coefficients GB_ROW31_COEF, staged per CTA); row31_combine pairs the
// halves into bins j and 31 - j.  Lane L ends up with bin row31_index(L) (lanes 0..30).
GB_HD GB_INLINE int row31_index(int lane) { return lane < 16 ? lane : 46 - lane; }
GB_HD GB_INLINE void row31_prep(int lane, const float2* src, float2* scr) {
    if (lane >= 1 && lane <= 15) {
        const float2 x = src[lane], y = src[31 - lane];
        scr[kPfaA + lane - 1] = c_add(x, y);
        const float2 b = c_sub(x, y);
        scr[kPfaB + lane - 1] = make_float2(-b.y, b.x);
    }
}
GB_HD GB_INLINE void row31_dot(int lane, const float2* src, float2* scr, const float* coef) {
    const float2* v = scr + (lane < 16 ? kPfaA : kPfaB);
    float2 acc = lane < 16 ? src[0] : make_float2(0.f, 0.f);
    const float* c = coef + 16 * lane;
#pragma unroll
    for (int k = 0; k < 15; ++k) acc = c_fma(c[k], v[k], acc);
    scr[kPfaX + lane] = acc;
}
template <bool INV>
GB_HD GB_INLINE float2 row31_combine(int lane, const float2* scr) {
    const float2 mine = scr[kPfaX + lane];
    if (lane == 0) return mine;
    const float2 v = scr[kPfaX + (lane < 16 ? lane + 15 : lane - 15)];
    // forward X_j = A_j - j B_j, X_{31-j} = A_j + j B_j; the inverse swaps the signs
    if (lane < 16) return INV ? c_add(mine, v) : c_sub(mine, v);
    return INV ? c_sub(v, mine) : c_add(v, mine);
}

// Replica product of the inverse: x[k2] = X[lane, k2] * R[lane, k2] for pair-interleaved spec and replica vectors.
GB_HD GB_INLINE void pfa_load_mul(float2 (&x)[33], int lane, const float2* spec, const float2* rep) {
#pragma unroll
    for (int jp = 0; jp < 16; ++jp) {
        float2 a0, a1, w0, w1;
        ld_pair(spec + 2 * (jp * 32 + lane), a0, a1);
        ld_pair(rep + 2 * (jp * 32 + lane), w0, w1);
        x[2 * jp] = cmul(a0, w0);
        x[2 * jp + 1] = cmul(a1, w1);
    }
    x[32] = cmul(spec[pidx(32, lane)], rep[pidx(32, lane)]);
}

// Inverse, phase 1: the 33-point column of bin k1 = lane, written to the tile as row n2, column k1.
GB_HD GB_INLINE void pfa_inv_phase1(float2 (&x)[33], int lane, float2* tile) {
    dft33_inv(x);
#pragma unroll
    for (int k = 0; k < 33; ++k) tile[k * kPfaStride + lane] = x[k];
}
// Inverse, phase 2 (after a warp sync): lane L gathers row n2 = L; the spread row n2 = 32 is prepared.
GB_HD GB_INLINE void pfa_inv_phase2(float2 (&y)[31], int lane, float2* tile) {
#pragma unroll
    for (int k = 0; k < 31; ++k) y[k] = tile[lane * kPfaStride + k];
    row31_prep(lane, tile + 32 * kPfaStride, tile);
}
// Inverse, phase 3 (after a warp sync): y[n1] = out[pfa_lag(n1, lane)], and the spread row's halves.
GB_HD GB_INLINE void pfa_inv_phase3(float2 (&y)[31], int lane, float2* tile, const float* coef) {
    dft31_inv(y);
    row31_dot(lane, tile + 32 * kPfaStride, tile, coef);
}
// Inverse, phase 4 (after a warp sync): out[pfa_lag(row31_index(lane), 32)] for lanes 0..30.
GB_HD GB_INLINE float2 pfa_inv_phase4(int lane, const float2* tile) { return row31_combine<true>(lane, tile); }

// Forward, phase 1: lane L gathers row n2 = L of the time-domain vector z (m < 1023, at zv[zpos(m)]) into y, and stages row
// n2 = 32 into the tile's scratch.
GB_HD GB_INLINE void pfa_fwd_gather(float2 (&y)[31], float2& e, int lane, const float2* zv) {
#pragma unroll
    for (int k = 0; k < 31; ++k) y[k] = zv[zpos(pfa_lag(k, lane))];
    e = lane < 31 ? zv[zpos(pfa_lag(lane, 32))] : make_float2(0.f, 0.f);
}
GB_HD GB_INLINE void pfa_fwd_phase1(float2 e, int lane, float2* tile) {
    if (lane < 31) tile[kPfaSrc + lane] = e;
}
// Forward, phase 2 (after a warp sync)
GB_HD GB_INLINE void pfa_fwd_phase2(float2 (&y)[31], int lane, float2* tile) {
    row31_prep(lane, tile + kPfaSrc, tile);
    dft31_fwd(y);
}
// Forward, phase 3 (after a warp sync)
GB_HD GB_INLINE void pfa_fwd_phase3(int lane, float2* tile, const float* coef) { row31_dot(lane, tile + kPfaSrc, tile, coef); }
// Forward, phase 4 (after a warp sync): the 31-point results go to the tile as row k1, column n2.
GB_HD GB_INLINE void pfa_fwd_phase4(const float2 (&y)[31], int lane, float2* tile) {
    const float2 e = row31_combine<false>(lane, tile);
#pragma unroll
    for (int k = 0; k < 31; ++k) tile[k * kPfaStride + lane] = y[k];
    if (lane < 31) tile[row31_index(lane) * kPfaStride + 32] = e;
}
// Forward, phase 5 (after a warp sync): the 33-point row of bin k1 = lane, stored as X[lane, k2] at dst[pidx(k2, lane)]
// (zero for lane 31).
GB_HD GB_INLINE void pfa_fwd_phase5(int lane, const float2* tile, float2* dst) {
    float2 x[33];
#pragma unroll
    for (int k = 0; k < 33; ++k) x[k] = lane < 31 ? tile[lane * kPfaStride + k] : make_float2(0.f, 0.f);
    dft33_fwd(x);
#pragma unroll
    for (int jp = 0; jp < 16; ++jp) st_pair(dst + 2 * (jp * 32 + lane), x[2 * jp], x[2 * jp + 1]);
    dst[pidx(32, lane)] = x[32];
}

// Branch-free reduction of one thread's 32 finished lags: v[n1] at lag pfa_lag(n1, lane) (n1 < 31) and v[31] at lag
// pfa_lag(row31_index(lane), 32) (none for lane 31).  First index = the smallest profile index s q + r among equal maxima: along
// n1 the lags rise by 33 and wrap once, at n1 = w, so the smallest equal lag is the first mask bit from w on, else the first bit.
GB_HD GB_INLINE void thread_peak_pfa(const float (&v)[32], int lane, int s, int r, Peak& out, float& fsum) {
    const bool has_e = lane < 31;
    const float ve = has_e ? v[31] : -1.0f;
    float m = v[0], sm = v[0];
#pragma unroll
    for (int k = 1; k < 31; ++k) {
        m = fmaxf(m, v[k]);
        sm += v[k];
    }
    m = fmaxf(m, ve);
    sm += has_e ? v[31] : 0.0f;
    unsigned eq = 0u;
#pragma unroll
    for (int k = 0; k < 31; ++k) eq |= v[k] == m ? 1u << k : 0u;
    const int w = (kChips - 31 * lane + 32) / 33;  // first n1 whose lag wraps (31 = none)
    const unsigned hi = eq >> w;
#if defined(__CUDA_ARCH__)
    const int first = hi ? __ffs(hi) - 1 + w : __ffs(eq) - 1;
    int c = __popc(eq);
#else
    const int first = hi ? __builtin_ctz(hi) + w : (eq ? __builtin_ctz(eq) : -1);
    int c = __builtin_popcount(eq);
#endif
    int q = eq ? pfa_lag(first, lane) : kChips;
    if (ve == m) {
        ++c;
        const int qe = pfa_lag(row31_index(lane), 32);
        q = qe < q ? qe : q;
    }
    out.mx = m;
    out.idx = s * q + r;
    out.cnt = c;
    out.sum = 0.0;
    fsum = sm;
}

// conj(DFT1023(c))[k] / 1023 in float64 from an exact-phase table cs[t] = (cos, sin)(2 pi t / 1023); the 1/1023 is the
// inverse transform's scaling.
GB_HD GB_INLINE void replica_spectrum_bin1023(const uint8_t* chips, int k, const double2* cs, double& re, double& im) {
    double ar = 0.0, ai = 0.0;
    for (int m = 0; m < kChips; ++m) {
        const int c = chips[m] ? 1 : -1;
        const double2 w = cs[(k * m) % kChips];
        ar += c * w.x;
        ai += c * w.y;
    }
    re = ar / kChips;
    im = ai / kChips;
}

}  // namespace gb
