// The world model's position fix for every millisecond of a parse call (fix_core.cuh), from the observations
// k_sv_observations computes.  One tracker is one receiver, so it has one clock slide and one world-model order.
//
// The slide enters a fix only through slide + receiver_timestamp, which every row shares, so round 0 absorbs any error
// in it into the clock bias and the slide a fix leaves does not depend on the slide it entered with, up to rounding
// (DESIGN.md §8c measures this).  So the chain of fixes, each starting from the slide the one before left, runs in two
// parallel passes instead of one serial walk:
//
// k_fix_plan: one warp per receiver.  Lane 0 reads the change tables: the millisecond the receiver stops at (a decoder
// raise), the slide every subframe resets (the last one of a millisecond wins, channel by channel) and the order in
// which satellites enter the world model.  Then the lanes walk the milliseconds 32 at a time: each finds its ready
// channels (flags 2 and 4) in that order, and warp ballots carry the slide of the current segment (the milliseconds
// since the last reset), the previous fixing millisecond of the segment and the first millisecond with five or more
// ready, where the reference raises.
// k_fix_pass<1>: one float64 thread per fixing millisecond runs the fix from its segment's slide.
// k_fix_pass<2>: again, from the slide pass 1 left at the previous fixing millisecond of the segment (at a reset
// millisecond: the reset value exactly; at the segment's first fix: the segment's slide).  These are the records.
// Each pass-2 fix checks that it left the slide pass 1 left (fix_same_slide), which the next fix of its segment started
// from.  k_fix_repair: where that check fails anywhere, one thread runs the chain serially from the first miss, each
// fix from the slide the fix before it left -- the reference's serial chain, at its serial cost.
// k_fix_finish: one warp.  Everything after the first raise stops, and the receiver's slide is carried to the next call.
//
// The least-squares mode (FixArgs::solver) runs k_fix_plan_lsq, k_fix_pass_lsq<1/2> and k_fix_repair_lsq, the same
// templates instantiated for it: five or more ready is a fix like any other, over all ready rows (fix_compute_lsq).
// Such rows can change inside a segment, and a fix that has not converged can depend on its entering slide; the chain
// check and the repair cover that as they cover a clock jump (DESIGN.md §8c).  The reference-mode kernels keep their
// names and code.
#include "fix_core.cuh"
#include "kernels.cuh"

namespace gb {

constexpr int kFixThreads = 128;
constexpr unsigned kFixFull = 0xffffffffu;

template <int kSolver>
__device__ __forceinline__ void fix_plan(const FixArgs& a) {
    const int lane = threadIdx.x;
    const int nc = a.n_channels, n_ms = a.n_ms;
    FixBank& bk = *a.bank;
    for (int m = lane; m < n_ms; m += 32) a.reset[m] = NAN;
    __syncwarp();
    int stop = n_ms;
    if (lane == 0) {
        if (bk.stopped) stop = 0;
        for (int c = 0; c < nc; ++c) {  // the first decoder raise stops the receiver before its millisecond
            const OrbitSnap* chg = a.changes + static_cast<size_t>(c) * a.change_stride;
            if (chg[0].frozen) stop = 0;
            for (int k = 1; k < a.change_counts[c]; ++k)
                if (chg[k].frozen) {
                    stop = min(stop, chg[k].ms);
                    break;
                }
        }
        for (int c = 0; c < nc; ++c) {  // channel by channel, each in event order: the last reset of a millisecond wins
            const OrbitSnap* chg = a.changes + static_cast<size_t>(c) * a.change_stride;
            for (int k = 1; k < a.change_counts[c]; ++k)
                if (fix_change_is_subframe(chg[k]) && chg[k].ms < stop) a.reset[chg[k].ms] = fix_reset_slide(chg[k]);
        }
        // First touches: a satellite enters satellite_ids_to_orbital_parameters at its first subframe or lost lock.
        // Within a millisecond the drops go first, then the subframes, each in channel order.  A satellite that holds
        // parameters from parse calls before the first fix call ranks before this call's, in channel order.
        bk.n_touched_before = bk.n_touched;
        for (int c = 0; c < nc; ++c) {
            a.touch_ms[c] = 0x7fffffff;
            if (a.rank[c] >= 0) continue;
            const OrbitSnap* chg = a.changes + static_cast<size_t>(c) * a.change_stride;
            if (chg[0].set) {
                a.touch_ms[c] = -1;
                continue;
            }
            for (int k = 1; k < a.change_counts[c]; ++k) {
                const OrbitSnap& s = chg[k];
                if (s.ms >= stop) break;
                if (fix_change_is_subframe(s) || fix_change_is_drop(s)) {
                    a.touch_ms[c] = 2 * s.ms + (fix_change_is_subframe(s) ? 1 : 0);
                    break;
                }
            }
        }
        for (;;) {
            int best = -1;
            for (int c = 0; c < nc; ++c)
                if (a.rank[c] < 0 && a.touch_ms[c] != 0x7fffffff && (best < 0 || a.touch_ms[c] < a.touch_ms[best])) best = c;
            if (best < 0) break;
            a.rank[best] = bk.n_touched++;
        }
        for (int c = 0; c < nc; ++c)
            if (a.rank[c] >= 0) a.order[a.rank[c]] = c;
    }
    stop = __shfl_sync(kFixFull, stop, 0);
    __syncwarp();
    const int n_touched = bk.n_touched;
    double seg = bk.slide;  // the slide entering the current segment
    int have = bk.has_slide;
    int last_reset = -1, chain = -1, raise5 = n_ms;
    for (int m0 = 0; m0 < n_ms; m0 += 32) {
        const int m = m0 + lane;
        const bool live = m < n_ms && m < stop && raise5 == n_ms;
        int n_ready = 0, rows[kFixRows] = {-1, -1, -1, -1};
        double r = NAN;
        if (live) {
            r = a.reset[m];
            for (int k = 0; k < n_touched; ++k) {
                const int c = a.order[k];
                if ((a.obs[static_cast<size_t>(c) * n_ms + m].flags & (kObsComplete | kObsFixGate)) == (kObsComplete | kObsFixGate)) {
                    if (n_ready < kFixRows) rows[n_ready] = c;
                    ++n_ready;
                }
            }
        }
        const unsigned live_resets = __ballot_sync(kFixFull, live && !isnan(r));
        const unsigned mine = live_resets & (kFixFull >> (31 - lane));  // resets at or before this millisecond
        const int reset_lane = mine ? 31 - __clz(mine) : -1;
        const double rv = __shfl_sync(kFixFull, r, reset_lane < 0 ? 0 : reset_lane);
        const double slide = reset_lane >= 0 ? rv : seg;
        const int has = reset_lane >= 0 ? 1 : have;
        // five or more ready with a slide: the first such millisecond raises, and everything after it has stopped (in
        // the least-squares mode they are fixes like any other)
        const unsigned many = kSolver == kFixSolverReference ? __ballot_sync(kFixFull, live && n_ready > kFixRows && has) : 0u;
        const int first5 = many ? m0 + __ffs(many) - 1 : n_ms;
        const bool stopped = !live || m > first5;
        const bool raised = !stopped && m == first5;
        const unsigned resets = many ? live_resets & (kFixFull >> (31 - (__ffs(many) - 1))) : live_resets;
        const bool cand = !stopped && (kSolver == kFixSolverReference ? n_ready == kFixRows : n_ready >= kFixRows) && has;
        const unsigned links = __ballot_sync(kFixFull, cand || raised);
        // the previous link of the segment: before this millisecond, at or after the segment's reset
        unsigned earlier = links & ((1u << lane) - 1u);
        if (reset_lane >= 0) earlier &= ~((1u << reset_lane) - 1u);
        const int prev = earlier ? m0 + 31 - __clz(earlier) : (reset_lane >= 0 ? -1 : chain);
        if (m < n_ms) {
            FixRecord f;
            fix_record_clear(f, a.rx[m]);
            f.status = stopped ? kFixStopped : raised ? kFixRaised : cand ? kFixSolved : kFixNone;
            if (!stopped) {
                f.n_ready = n_ready;
                for (int i = 0; i < kFixRows; ++i) f.channel[i] = rows[i];
            }
            if (cand || raised) f.slide_in = has ? slide : NAN;
            a.out[m] = f;
            a.prev[m] = prev;
        }
        if (resets) {
            const int l = 31 - __clz(resets);
            seg = __shfl_sync(kFixFull, r, l);
            have = 1;
            last_reset = m0 + l;
            const unsigned tail = links & ~((1u << l) - 1u);
            chain = tail ? m0 + 31 - __clz(tail) : -1;
        } else if (links) {
            chain = m0 + 31 - __clz(links);
        }
        raise5 = min(raise5, first5);
    }
    if (lane == 0) {
        bk.first_raise = n_ms;
        bk.last_fix = -1;
        bk.last_reset = last_reset;
        bk.reset_slide = seg;
        bk.reset_has = have;
        bk.stop_frozen = stop < n_ms;
        bk.first_miss = n_ms;
    }
}

__global__ void __launch_bounds__(32) k_fix_plan(const FixArgs a) { fix_plan<kFixSolverReference>(a); }
__global__ void __launch_bounds__(32) k_fix_plan_lsq(const FixArgs a) { fix_plan<kFixSolverLeastSquares>(a); }

// The fix of millisecond m from slide s, over the rows the plan chose.
__device__ int fix_at(const FixArgs& a, int m, double s, FixRecord& f) {
    FixRow r[kFixRows];
    for (int i = 0; i < kFixRows; ++i) {
        const SvObservation& o = a.obs[static_cast<size_t>(f.channel[i]) * a.n_ms + m];
        r[i] = FixRow{o.tow, o.x, o.y, o.z};
    }
    return fix_compute(r, f.receiver_timestamp, s, f);
}

// The ready rows of millisecond m in the world model's order, for fix_compute_lsq: read from the observations again
// on every iteration, so any number of rows needs no storage.
struct FixReadyRows {
    const FixArgs& a;
    int m, n_touched;
    template <class F>
    __device__ __forceinline__ void operator()(F&& fn) const {
        int i = 0;
        for (int k = 0; k < n_touched; ++k) {
            const SvObservation& o = a.obs[static_cast<size_t>(a.order[k]) * a.n_ms + m];
            if ((o.flags & (kObsComplete | kObsFixGate)) == (kObsComplete | kObsFixGate)) fn(i++, FixRow{o.tow, o.x, o.y, o.z});
        }
    }
};

// fix_at in the least-squares mode: five or more rows take the least-squares fix.
__device__ __forceinline__ int fix_at_lsq(const FixArgs& a, int m, double s, FixRecord& f) {
    if (f.n_ready == kFixRows) return fix_at(a, m, s, f);
    return fix_compute_lsq(FixReadyRows{a, m, a.bank->n_touched}, f.n_ready, f.receiver_timestamp, s, f);
}

template <int kSolver, int kPass>
__device__ __forceinline__ void fix_pass(const FixArgs& a) {
    const int m = blockIdx.x * kFixThreads + threadIdx.x;
    if (m >= a.n_ms) return;
    FixRecord f = a.out[m];
    if (f.status != kFixSolved && f.status != kFixRaised) return;
    double s = f.slide_in;
    if (kPass == 2 && a.prev[m] >= 0) s = a.slide1[a.prev[m]];
    int status = kFixRaised;
    if (kSolver == kFixSolverLeastSquares) {  // the plan marks no raise in this mode
        status = fix_at_lsq(a, m, s, f);
    } else if (f.status == kFixRaised) {  // five or more ready: np.linalg.solve raises before anything changes
        f.slide_in = f.slide_out = s;
    } else {
        status = fix_at(a, m, s, f);
    }
    if (kPass == 1) {
        a.slide1[m] = f.slide_out;
        return;
    }
    f.status = status;
    a.out[m] = f;
    if (status == kFixRaised) atomicMin(&a.bank->first_raise, m);
    atomicMax(&a.bank->last_fix, m);
    // The next fix of the segment started from pass 1's slide: the chain holds only if this fix left the same one.
    if (!fix_same_slide(f.slide_out, a.slide1[m])) atomicMin(&a.bank->first_miss, m);
}

template <int kPass>
__global__ void __launch_bounds__(kFixThreads) k_fix_pass(const FixArgs a) {
    fix_pass<kFixSolverReference, kPass>(a);
}
template <int kPass>
__global__ void __launch_bounds__(kFixThreads) k_fix_pass_lsq(const FixArgs a) {
    fix_pass<kFixSolverLeastSquares, kPass>(a);
}

// Where the chain check failed, the serial chain: from the first miss on, every fix that does not start from a reset
// runs again from the slide the fix before it left, in order, in one thread.  The comparison is exact, not the check's
// 4 ulp: after a miss every fix of the call, in later segments too, is the serial chain's bit for bit, and n_repaired
// counts each fix whose entering slide changed.
template <int kSolver>
__device__ __forceinline__ void fix_repair(const FixArgs& a) {
    FixBank& bk = *a.bank;
    if (threadIdx.x != 0 || bk.first_miss >= a.n_ms) return;
    int last = bk.first_miss;
    for (int m = last + 1; m < a.n_ms && m <= bk.first_raise; ++m) {
        FixRecord f = a.out[m];
        if (f.status != kFixSolved && f.status != kFixRaised) continue;
        const double s = a.out[last].slide_out;
        if (a.prev[m] >= 0 && !(f.slide_in == s)) {
            if (kSolver == kFixSolverReference && f.n_ready > kFixRows) {
                f.slide_in = f.slide_out = s;
            } else {
                f.status = kSolver == kFixSolverReference ? fix_at(a, m, s, f) : fix_at_lsq(a, m, s, f);
                if (f.status == kFixRaised && m < bk.first_raise) bk.first_raise = m;
            }
            a.out[m] = f;
            ++bk.n_repaired;
        }
        last = m;
    }
}

__global__ void __launch_bounds__(32) k_fix_repair(const FixArgs a) { fix_repair<kFixSolverReference>(a); }
__global__ void __launch_bounds__(32) k_fix_repair_lsq(const FixArgs a) { fix_repair<kFixSolverLeastSquares>(a); }

__global__ void __launch_bounds__(32) k_fix_finish(const FixArgs a) {
    const int lane = threadIdx.x;
    FixBank& bk = *a.bank;
    const int first = bk.first_raise;
    for (int m = first + 1 + lane; m < a.n_ms; m += 32) {  // the receiver's step never returns after a raise
        FixRecord& f = a.out[m];
        if (f.status == kFixStopped) continue;
        fix_record_clear(f, f.receiver_timestamp);
        f.status = kFixStopped;
    }
    if (lane != 0) return;
    if (first < a.n_ms) {
        bk.slide = a.out[first].slide_out;
        bk.has_slide = !isnan(bk.slide);
        bk.stopped = 1;
        for (int c = 0; c < a.n_channels; ++c)  // satellites this call touched after the raise never got there
            if (a.rank[c] >= bk.n_touched_before && a.touch_ms[c] >= 0 && a.touch_ms[c] / 2 > first) {
                a.rank[c] = -1;
                --bk.n_touched;
            }
    } else {
        if (bk.last_fix >= 0 && bk.last_fix >= bk.last_reset) {
            bk.slide = a.out[bk.last_fix].slide_out;
            bk.has_slide = 1;
        } else {
            bk.slide = bk.reset_slide;
            bk.has_slide = bk.reset_has;
        }
        if (bk.stop_frozen) bk.stopped = 1;
    }
}

cudaError_t launch_position_fixes(const FixArgs& a, cudaStream_t st) {
    const int blocks = (a.n_ms + kFixThreads - 1) / kFixThreads;
    if (a.solver == kFixSolverLeastSquares) {
        k_fix_plan_lsq<<<1, 32, 0, st>>>(a);
        k_fix_pass_lsq<1><<<blocks, kFixThreads, 0, st>>>(a);
        k_fix_pass_lsq<2><<<blocks, kFixThreads, 0, st>>>(a);
        k_fix_repair_lsq<<<1, 32, 0, st>>>(a);
    } else {
        k_fix_plan<<<1, 32, 0, st>>>(a);
        k_fix_pass<1><<<blocks, kFixThreads, 0, st>>>(a);
        k_fix_pass<2><<<blocks, kFixThreads, 0, st>>>(a);
        k_fix_repair<<<1, 32, 0, st>>>(a);
    }
    k_fix_finish<<<1, 32, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace gb
