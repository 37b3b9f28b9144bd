// The receiver's velocity, clock drift, geodetic position and dilution of precision for every millisecond of the last
// parse call with a solved position fix (velocity_core.cuh), from the fix records, the observations and change tables
// the fix call used and each channel's tracker Doppler.
//
// Unlike the fix, velocity needs no serial chain: the fix carries the receiver's clock slide from one millisecond to the
// next, but the velocity solve is linear in its unknowns and starts from nothing but the millisecond's own fix position,
// rows and Dopplers.  So k_velocity_fixes is one float64 thread per millisecond, and nothing is checked or repaired.
//
// Rows: a fix with exactly four ready satellites (every fix of the reference mode) used its record's channel[0..3], and
// so does the velocity.  A least-squares fix over more than four used every ready channel (flags 2 and 4) in the world
// model's order, which the record does not hold; they are found again as k_fix_plan found them, from the order and
// n_touched the fix call left in its scratch and bank.  Their number must be the record's n_ready (status 2 otherwise).
// Each row's satellite velocity and clock drift is orbit_velocity at the observation's time of week, on the orbit
// snapshot (orbit_change_at) that gave the observation.
#include "kernels.cuh"
#include "velocity_core.cuh"

namespace gb {

constexpr int kVelocityThreads = 128;

// The row of channel c at millisecond m.
__device__ __forceinline__ VelocityRow velocity_row_at(const VelocityArgs& a, int c, int m) {
    const SvObservation& o = a.obs[static_cast<size_t>(c) * a.n_ms + m];
    const OrbitSnap& s = orbit_change_at(a.changes + static_cast<size_t>(c) * a.change_stride, a.change_counts[c], m);
    VelocityRow w;
    w.x = o.x;
    w.y = o.y;
    w.z = o.z;
    orbit_velocity(s.p, o.tow, w.vx, w.vy, w.vz, w.drift);
    w.doppler = a.doppler[static_cast<size_t>(c) * a.doppler_channel_stride + static_cast<size_t>(m) * a.doppler_ms_stride];
    return w;
}

// The four rows of the record.
struct VelocityFixRows {
    const VelocityArgs& a;
    const FixRecord& f;
    int m;
    template <class F>
    __device__ __forceinline__ void operator()(F&& fn) const {
        for (int i = 0; i < kFixRows; ++i) fn(i, velocity_row_at(a, f.channel[i], m));
    }
};

// The ready rows in the world model's order.
struct VelocityReadyRows {
    const VelocityArgs& a;
    int m, n_touched;
    template <class F>
    __device__ __forceinline__ void operator()(F&& fn) const {
        int i = 0;
        for (int k = 0; k < n_touched; ++k) {
            const int c = a.order[k];
            if (velocity_row_ready(a.obs[static_cast<size_t>(c) * a.n_ms + m].flags)) fn(i++, velocity_row_at(a, c, m));
        }
    }
};

__global__ void __launch_bounds__(kVelocityThreads) k_velocity_fixes(const VelocityArgs a) {
    const int m = blockIdx.x * kVelocityThreads + threadIdx.x;
    if (m >= a.n_ms) return;
    const FixRecord f = a.fixes[m];
    VelocityRecord v;
    velocity_record_clear(v, f.receiver_timestamp);
    if (f.status == kFixSolved) {
        if (f.n_ready == kFixRows) {
            velocity_compute(VelocityFixRows{a, f, m}, kFixRows, f.x, f.y, f.z, v);
        } else {
            const int n_touched = a.bank->n_touched;
            int n = 0;
            for (int k = 0; k < n_touched; ++k)
                n += velocity_row_ready(a.obs[static_cast<size_t>(a.order[k]) * a.n_ms + m].flags) ? 1 : 0;
            if (n == f.n_ready) {
                velocity_compute(VelocityReadyRows{a, m, n_touched}, n, f.x, f.y, f.z, v);
            } else {  // the order no longer gives the fix's rows: the geodetic position only
                velocity_compute(VelocityReadyRows{a, m, 0}, 0, f.x, f.y, f.z, v);
                v.n_rows = n;
            }
        }
    }
    a.out[m] = v;
}

cudaError_t launch_velocity_fixes(const VelocityArgs& a, cudaStream_t st) {
    k_velocity_fixes<<<(a.n_ms + kVelocityThreads - 1) / kVelocityThreads, kVelocityThreads, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace gb
