// Shared between device code and the host-side lane emulator (tests/emu).  No reference code here.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define GB_HD __host__ __device__
#define GB_INLINE __forceinline__
#else
#define GB_HD
#define GB_INLINE inline
#endif

// The sample rates the engine supports, as samples per millisecond / 1023: X(S) once per rate.  Every rate switch, kernel
// configuration and the error message for an unsupported rate expand this one list.
#define GB_FOR_EACH_RATE(X) X(1) X(2) X(3) X(4) X(5) X(6) X(8) X(10) X(12) X(16)

namespace gb {

constexpr int kChips = 1023;   // constants.py:7  PRN_CHIP_COUNT
constexpr int kFft = 1024;     // one warp-level transform
constexpr int kPad = 2048;     // zero-padded length carrying a length-1023 circular correlation (>= 2*1023-1)
constexpr int kTStride = 34;   // padded row of the 32x32 transpose tile (float2 units): 16-byte aligned rows, conflict-free
                               // for the 64-bit column writes and the 128-bit row reads
constexpr int kTileF2 = 32 * kTStride;

// Result of reducing one correlation profile; mirrors include/gypsum_b200.h gb200_cell_record (32 bytes).
struct CellRecord {
    float peak;      // max of the (non-coherent) profile, or of |coherent profile|
    int32_t argmax;  // first index attaining it (np.argmax rule, acquisition.py:184)
    double sum;      // sum over all N profile values
    int32_t count;   // how many values equal the max (utils.py:113 excludes all of them)
    float probe_re;  // coherent profile value at the requested index (acquisition.py:136)
    float probe_im;
    int32_t pad_;
};
static_assert(sizeof(CellRecord) == 32, "record must stay 32 bytes");

struct Peak {
    float mx;
    int idx;
    int cnt;
    double sum;
};

GB_HD GB_INLINE void peak_init(Peak& p) {
    p.mx = -1.0f;
    p.idx = 0x7fffffff;
    p.cnt = 0;
    p.sum = 0.0;
}
// Profile values are >= 0.  First index wins ties; cnt counts elements equal to the running max.
GB_HD GB_INLINE void peak_push(Peak& p, float v, int n) {
    if (v > p.mx) {
        p.mx = v;
        p.idx = n;
        p.cnt = 1;
    } else if (v == p.mx) {
        p.cnt += 1;
        p.idx = n < p.idx ? n : p.idx;
    }
}
GB_HD GB_INLINE void peak_merge(Peak& a, const Peak& b) {
    if (b.mx > a.mx) {
        a.mx = b.mx;
        a.idx = b.idx;
        a.cnt = b.cnt;
    } else if (b.mx == a.mx) {
        a.cnt += b.cnt;
        a.idx = b.idx < a.idx ? b.idx : a.idx;
    }
    a.sum += b.sum;
}

// One warp's (or warp pair's) peak and probe share, exchanged through shared memory when several work on one cell.
struct PeakPartial {
    float mx;
    int idx;
    int cnt;
    float pr_re;
    double sum;
    float pr_im;
    int pad;
};

GB_HD GB_INLINE void store_partial(PeakPartial* dst, const Peak& p, float pr_re, float pr_im) {
    PeakPartial pp;
    pp.mx = p.mx;
    pp.idx = p.idx;
    pp.cnt = p.cnt;
    pp.sum = p.sum;
    pp.pr_re = pr_re;
    pp.pr_im = pr_im;
    pp.pad = 0;
    *dst = pp;
}

// Merges n partials in order (first index wins ties, counts and sums add) and sums their probe shares.
GB_HD GB_INLINE Peak merge_partials(const PeakPartial* part, int n, float& pr_re, float& pr_im) {
    Peak m;
    peak_init(m);
    pr_re = pr_im = 0.f;
    for (int w = 0; w < n; ++w) {
        const PeakPartial pp = part[w];
        Peak o;
        o.mx = pp.mx;
        o.idx = pp.idx;
        o.cnt = pp.cnt;
        o.sum = pp.sum;
        peak_merge(m, o);
        pr_re += pp.pr_re;
        pr_im += pp.pr_im;
    }
    return m;
}

GB_HD GB_INLINE void write_record(CellRecord* dst, const Peak& p, float probe_re, float probe_im) {
    CellRecord rec;
    rec.peak = p.mx;
    rec.argmax = p.idx;
    rec.sum = p.sum;
    rec.count = p.cnt;
    rec.probe_re = probe_re;
    rec.probe_im = probe_im;
    rec.pad_ = 0;
    *dst = rec;
}

// Correlation strength of a profile (utils.py:111-116): its peak over the mean of the values not equal to the peak.
GB_HD GB_INLINE double record_strength(double peak, double sum, int count, int N) {
    return peak / ((sum - count * peak) / (N - count));
}

}  // namespace gb
