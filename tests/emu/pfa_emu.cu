// Host lane emulator for the one-warp kernel's exact 1023-point transforms (warp_pfa.cuh): forward as k_doppler_spectra runs
// it, inverse and the peak reduction as k_correlate_pfa runs them.  Test infrastructure; never loaded by the product.
#include <vector>

#include "../../gypsum_b200/csrc/warp_pfa.cuh"

using namespace gb;

static const float kCoef[32][16] = GB_ROW31_COEF;

extern "C" {

// spec[pidx(k2, k1)] = DFT1023(z)[pfa_bin(k1, k2)] (zero for k1 = 31), from z[m], m < 1023.
void emu_dft1023_fwd(const float2* z, float2* spec) {
    std::vector<float2> zv(kFft), tile(kPfaTileF2);
    for (int m = 0; m < kChips; ++m) zv[zpos(m)] = z[m];
    float2 y[32][31], e[32];
    for (int l = 0; l < 32; ++l) pfa_fwd_gather(y[l], e[l], l, zv.data());
    for (int l = 0; l < 32; ++l) pfa_fwd_phase1(e[l], l, tile.data());
    for (int l = 0; l < 32; ++l) pfa_fwd_phase2(y[l], l, tile.data());
    for (int l = 0; l < 32; ++l) pfa_fwd_phase3(l, tile.data(), &kCoef[0][0]);
    for (int l = 0; l < 32; ++l) pfa_fwd_phase4(y[l], l, tile.data());
    for (int l = 0; l < 32; ++l) pfa_fwd_phase5(l, tile.data(), spec);
}

// out[q] = sum_k spec(k) rep(k) exp(+2 pi i k q / 1023), spec and rep in the permuted order above.
void emu_dft1023_inv(const float2* spec, const float2* rep, float2* out) {
    std::vector<float2> tile(kPfaTileF2);
    float2 y[32][31], e[32];
    for (int l = 0; l < 32; ++l) {
        float2 x[33];
        pfa_load_mul(x, l, spec, rep);
        pfa_inv_phase1(x, l, tile.data());
    }
    for (int l = 0; l < 32; ++l) pfa_inv_phase2(y[l], l, tile.data());
    for (int l = 0; l < 32; ++l) pfa_inv_phase3(y[l], l, tile.data(), &kCoef[0][0]);
    for (int l = 0; l < 32; ++l) e[l] = pfa_inv_phase4(l, tile.data());
    for (int l = 0; l < 32; ++l) {
        for (int n1 = 0; n1 < 31; ++n1) out[pfa_lag(n1, l)] = y[l][n1];
        if (l < 31) out[pfa_lag(row31_index(l), 32)] = e[l];
    }
}

// Record of n_r profiles v[r][1023] as k_correlate_pfa forms it: thread_peak_pfa per lane and branch, merged over r, then over
// the lanes in lane order.
void emu_peak(const float* v, int n_r, float* mx, int* idx, int* cnt, double* sum) {
    Peak warp;
    peak_init(warp);
    for (int l = 0; l < 32; ++l) {
        Peak pk;
        peak_init(pk);
        for (int r = 0; r < n_r; ++r) {
            float acc[32];
            for (int n1 = 0; n1 < 31; ++n1) acc[n1] = v[r * kChips + pfa_lag(n1, l)];
            acc[31] = l < 31 ? v[r * kChips + pfa_lag(row31_index(l), 32)] : 0.f;
            Peak t;
            float fsum;
            thread_peak_pfa(acc, l, n_r, r, t, fsum);
            t.sum = static_cast<double>(fsum);
            peak_merge(pk, t);
        }
        peak_merge(warp, pk);
    }
    *mx = warp.mx;
    *idx = warp.idx;
    *cnt = warp.cnt;
    *sum = warp.sum;
}
}
