// Host lane emulator for the one-warp kernel's per-CTA odd-parity twiddle table (w2048_odd_twiddles, w2048_phase1_odd) and
// its whole-transform peak reduction (thread_peak32), next to the functions they stand in for (w2048_phase1<1>,
// thread_peak16).  Test infrastructure; never loaded by the product.
#include <cmath>
#include <vector>

#include "../../gypsum_b200/csrc/warp_fft.cuh"

using namespace gb;

static std::vector<float2> tw1_table() {
    std::vector<float2> tw1(1024);
    for (int k1 = 0; k1 < 32; ++k1)
        for (int l = 0; l < 32; ++l) {
            const double a = -2.0 * M_PI * ((l * k1) % 1024) / 1024.0;
            tw1[pidx(k1, l)] = make_float2((float)cos(a), (float)sin(a));
        }
    return tw1;
}

extern "C" {

// Pruned inverse FFT-2048 (out[k], k < 1024) with the odd parity through w2048_phase1_odd (table != 0) or w2048_phase1<1>.
void emu_ifft2048_odd(const float2* y_even, const float2* y_odd, int table, float2* out) {
    const std::vector<float2> tw1 = tw1_table();
    std::vector<float2> tw1o(512), tile(kTile64F2);
    for (int lane = 0; lane < 32; ++lane) w2048_odd_twiddles(lane, tw1.data(), tw1o.data());
    for (int lane = 0; lane < 32; ++lane) {
        float2 a[32], b[32];
        for (int j = 0; j < 32; ++j) {
            a[j] = y_even[lane + 32 * j];
            b[j] = y_odd[lane + 32 * j];
        }
        w2048_phase1<0>(a, lane, tw1.data(), tile.data());
        if (table) w2048_phase1_odd(b, lane, tw1.data(), tw1o.data(), tile.data());
        else w2048_phase1<1>(b, lane, tw1.data(), tile.data());
    }
    for (int lane = 0; lane < 32; ++lane) {
        float2 x[64];
        w2048_phase2(x, lane, tile.data());
        for (int k2 = 0; k2 < 32; ++k2) out[lane + 32 * k2] = x[k2];
    }
}

// Record of n_r profiles v[r][1024] (lags q = lane + 32 k, s = n_r branches, lag 1023 unused) as the one-warp kernel forms it
// from each lane's 32 lags: thread_peak32 (fast != 0) or the two thread_peak16 halves, merged over r, then over the lanes in
// lane order.  out: mx, idx, cnt as float / int / int and the float64 sum.
void emu_peak(const float* v, int n_r, int fast, float* mx, int* idx, int* cnt, double* sum) {
    Peak warp;
    peak_init(warp);
    for (int lane = 0; lane < 32; ++lane) {
        Peak pk;
        peak_init(pk);
        for (int r = 0; r < n_r; ++r) {
            float acc[32];
            for (int k = 0; k < 32; ++k) acc[k] = v[r * 1024 + lane + 32 * k];
            if (fast) {
                Peak t;
                float fsum[2];
                thread_peak32(acc, lane, n_r, r, t, fsum);
                t.sum = static_cast<double>(fsum[0]);
                peak_merge(pk, t);
                pk.sum += static_cast<double>(fsum[1]);
            } else {
                for (int hh = 0; hh < 2; ++hh) {
                    float h16[16];
                    for (int jj = 0; jj < 16; ++jj) h16[jj] = acc[16 * hh + jj];
                    Peak t;
                    float fsum;
                    thread_peak16(h16, lane, hh, n_r, r, t, fsum);
                    t.sum = static_cast<double>(fsum);
                    peak_merge(pk, t);
                }
            }
        }
        peak_merge(warp, pk);
    }
    *mx = warp.mx;
    *idx = warp.idx;
    *cnt = warp.cnt;
    *sum = warp.sum;
}
}
