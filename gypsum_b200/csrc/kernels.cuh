// Kernel argument blocks and launch wrappers (implemented in kernels.cu, used by engine.cu and receiver.cu).
#pragma once
#include "gb_common.cuh"
#include "tracker_core.cuh"

namespace gb {

constexpr int kKindCoherent = 1;     // utils.py:23-25: IntegrationType.Coherent = auto() -> 1
constexpr int kKindNonCoherent = 2;  // IntegrationType.NonCoherent -> 2

// doppler_spectra: one CTA per (unique Doppler u, millisecond i); with T > 1 (segment_spectra) or align (aligned_segment_spectra)
// one per (u, segment i of T milliseconds), M being the segments per block.
struct SpectraArgs {
    const float2* iq;        // complex64 samples, block b starts at b * block_stride
    const double* doppler;   // [n_doppler] Hz
    float2* spec;            // [n_blocks*n_doppler][M][s][2][1024]
    const float2* tw1;       // [32][32]  exp(-2 pi i lane k1 / 1024)
    const float2* tw2;       // [1024]    exp(-2 pi i n / 2048)
    long long block_stride;  // samples between consecutive blocks (= M*N, or M*T*N with segments)
    int pfa;                 // spectra for k_correlate_pfa: DFT1023(z_r) per branch r (warp_pfa.cuh order) in [r][0]; else both halves
    double inv_fs;
    int N, s, M, n_doppler, n_units;  // n_units = n_blocks * n_doppler
    int T;                   // milliseconds per coherent segment; T > 1 selects segment_spectra
    // Weak grids (align = 1 selects aligned_segment_spectra, at any T): the Doppler axis is folded as n_doppler =
    // B * phase_dopplers slots, slot d being bit phase j = d / phase_dopplers, whose segment i starts at block millisecond
    // j * phase_step + i * T.  Each millisecond m is realigned by its code Doppler (code_shift).
    int align, phase_step, phase_dopplers;
};

// The whole-sample code-Doppler shift of block millisecond m at Doppler f (N samples per millisecond): the code of a
// satellite closing at f runs fast by f / f_L1, so its lag at millisecond m is tau0 - m * N * f / f_L1 samples, and a
// sample added at row position (n + shift) mod N lines its millisecond up with millisecond 0.  The float64 expression is
// evaluated in this order on the host, in the kernel and in the tests' oracle.
__host__ __device__ inline double code_shift(int m, int N, double f) {
    return rint(static_cast<double>(m) * N * f / 1575.42e6);
}

// correlate_cells: one warp (k_correlate_pfa) or warp pair (k_correlate_cells) per (cell, r-range); every slot of a CTA
// works on the same PRN.
struct CorrelateArgs {
    const float2* spec;
    const float2* crep;  // [n_prn][2][1024]  conj(FFT2048(c'))/2048, even / odd bins
    const float2* crep1023;  // [n_prn][kPfaVecF2]  conj(DFT1023(c))/1023 in warp_pfa.cuh's bin order (k_correlate_pfa)
    const float2* tw1;   // [32][32]
    const float2* tw2;   // [1024]
    CellRecord* records;
    float* profile;      // optional: full profile of the single cell (N floats, or 2N when coherent)
    int N, s, M, kind;
    int rsplit;          // slots cooperating on one cell (divides s and correlate_slots)
    int n_groups;
    // grid mode (cells = blocks x prn list x doppler list)
    int grid_mode, P, D, n_blocks, chunks;  // chunks = ceil(n_blocks * D / cells_per_group): groups per PRN
    int win_chunks;  // k_correlate_pfa, grid mode: chunks per L2 window (0 = the whole batch is one window), see the kernel
    const int* prn_idx;           // [P]
    // list mode (cells sorted by PRN)
    const int* grp_first;
    const int* grp_count;
    const int* grp_prn;
    const int* cell_u;      // spectrum unit of each sorted cell
    const int* cell_out;    // where its record goes
    const int* cell_probe;  // coherent probe index or -1 (both modes, indexed by output slot; may be null)
    int stag_a, stag_b;       // k_correlate_pfa start stagger in ns: (warp / 4) * stag_a + (warp % 4) * stag_b (set by launch_correlate)
    const double* cell_gate;  // optional, indexed by output slot: NaN = this cell is switched off (device-planned lists)
};

// On-device Doppler refinement (reference acquisition.py:70-152): per-satellite search state and result.
constexpr int kRefineMaxBins = 32;  // acquisition.py:163-167 yields 20..28 bins per pass
struct RefineState {
    double center;         // center_doppler_shift_estimation
    double kept_doppler;   // best_..._across_all_search_space.doppler_shift
    double kept_strength;  // .correlation_strength
    int kept_index;        // .sample_offset_of_correlation_peak
    int have_kept;
};
struct RefineResult {  // 32 bytes, mirrored by gb200_acquisition_result
    double doppler;
    double strength;
    float probe_re, probe_im;  // coherent profile value at the kept peak index
    int code_phase;
    int pad_;
};
struct BestRecord {  // 32 bytes, mirrored by gb200_best_record
    double doppler;
    double strength;
    float peak;
    int code_phase;
    int bin;
    int pad_;
};
cudaError_t launch_best_bins(int n_rows, int D, int N, const CellRecord* rec, const double* doppler, BestRecord* out,
                             cudaStream_t s);
cudaError_t launch_refine_plan(int n_sv, double spread, const RefineState* st, double* doppler, cudaStream_t s);
cudaError_t launch_refine_select(int n_sv, int N, const CellRecord* rec, const double* doppler, RefineState* st, cudaStream_t s);
cudaError_t launch_refine_coherent_plan(int n_sv, const RefineState* st, double* doppler, int* probe, cudaStream_t s);
cudaError_t launch_refine_finalize(int n_sv, const RefineState* st, const CellRecord* rec, RefineResult* out, cudaStream_t s);
cudaError_t launch_refine_init(int n_sv, RefineState* st, cudaStream_t s);

// track_channels: one persistent CTA per channel.
struct TrackArgs {
    const float2* iq;           // [n_ms * N] the stream every channel consumes
    const double* start_times;  // [n_ms] chunk start timestamps (antenna_sample_provider.py:88-89)
    TrackState* states;         // [n_channels]
    TrackMsRecord* out;         // [n_channels][n_ms]
    float* profiles;            // optional [n_channels][n_ms][N]: |prompt profile| (tracker.py:308-309)
    const float2* crep;
    const float2* tw1;
    const float2* tw2;
    double fs, inv_fs;
    int N, s, n_ms, n_channels;
    double t0_single;           // start time used when start_times is null (single-millisecond launches: no upload)
    const int* channel_idx;     // optional [n_channels]: CTA b runs channel channel_idx[b] (records still go to out[b]); null = b
    TrackState* shadow;         // optional [capacity]: every launched channel's state as it was BEFORE this launch (rollback)
    double code_wrap;           // the DLL accumulator's modulus: kReferenceCodeWrap or N (tracker_core.cuh)
};

// integrate_bits: one warp per tracking channel (bits.cu, bits_core.cuh).
struct BitState;
struct BitEvent;
struct BitArgs {
    const TrackMsRecord* records;  // [n_channels][n_ms] as written by k_track_channels
    const double* start_times;     // [n_ms] chunk start / end timestamps
    const double* end_times;
    BitState* states;              // [n_channels]
    BitEvent* events;              // [n_channels][max_events]
    int* counts;                   // [n_channels] events produced (may exceed max_events: truncated)
    int n_ms, n_channels, max_events;
    double code_wrap;              // the tracker's code-phase modulus: each symbol's delay is code_phase / code_wrap ms
};

// decode_subframes: one warp per channel over its bit events (nav.cu, nav_core.cuh).
struct NavState;
struct SubframeEvent;
struct NavArgs {
    const BitEvent* bits;        // [n_channels][stride]
    const int* counts;           // [n_channels] bit events per channel
    const BitState* bit_states;  // optional: a channel whose integrator stopped stops after these bits
    NavState* states;            // [n_channels]
    SubframeEvent* events;       // [n_channels][max_events]
    int* event_counts;           // [n_channels] events produced (may exceed max_events: truncated)
    int stride, n_channels, max_events;
};

// parse_subframes / sv_observations: subframe fields, the world model's per-satellite state and its per-millisecond
// satellite time and position (orbit.cu, orbit_core.cuh).
struct OrbitSnap;
struct SubframeFields;
struct SvObservation;
struct OrbitArgs {
    const SubframeEvent* events;   // [n_channels][stride]
    const int* counts;             // [n_channels] events per channel
    const int* event_ms;           // explicit: [n_channels][stride] millisecond of each event; null = from `bits`
    const BitEvent* bits;          // chain: the bit events the events' bit_index refers to, [n_channels][bit_stride]
    const TrackMsRecord* records;  // chain: the tracking records, [n_channels][n_ms]; a `lost` one drops the channel
    const int* drop_ms;            // explicit: [n_channels] millisecond the channel is dropped at, -1 = none
    OrbitSnap* states;             // [n_channels] carried from call to call
    SubframeFields* fields;        // [n_channels][stride] parsed kind-0 events
    int* field_counts;             // [n_channels]
    OrbitSnap* changes;            // [n_channels][stride + 2] the state after each change, by millisecond
    int* change_counts;            // [n_channels]
    int stride, bit_stride, n_ms, n_channels;
};
cudaError_t launch_parse_subframes(const OrbitArgs& a, cudaStream_t st);
cudaError_t launch_sv_observations(const OrbitSnap* changes, const int* change_counts, int change_stride, int n_channels,
                                   int n_ms, SvObservation* out, cudaStream_t st);

// position_fixes: the world model's fix for every millisecond of the last parse call (fix.cu, fix_core.cuh).
struct FixBank;
struct FixRecord;
struct FixArgs {
    const OrbitSnap* changes;    // the last parse call's change tables, [n_channels][change_stride]
    const int* change_counts;    // [n_channels]
    int change_stride;
    const SvObservation* obs;    // [n_channels][n_ms]
    const double* rx;            // [n_ms] receiver timestamps (chunk start times)
    FixBank* bank;               // the receiver's state, carried from call to call
    int* rank;                   // [n_channels] world-model order, -1 = not in it; carried
    int* order;                  // [n_channels] scratch: the channels by rank
    int* touch_ms;               // [n_channels] scratch: 2 * first-touch ms + (1 subframe, 0 drop); -1 before the call
    double* reset;               // [n_ms] scratch: the slide the millisecond's subframes set, NaN = none
    int* prev;                   // [n_ms] scratch: the previous fixing millisecond of the segment, -1 = none
    double* slide1;              // [n_ms] scratch: pass 1's slide after each fix
    FixRecord* out;              // [n_ms]
    int n_channels, n_ms;
    int solver;                  // FixSolver: which kernels launch_position_fixes runs
};
cudaError_t launch_position_fixes(const FixArgs& a, cudaStream_t st);

// velocity_fixes: velocity, clock drift, geodetic position and DOP of every solved fix (velocity.cu, velocity_core.cuh).
struct VelocityRecord;
struct VelocityArgs {
    const FixRecord* fixes;             // [n_ms] the position fixes of the last parse call
    const SvObservation* obs;           // [n_channels][n_ms] the observations the fix call computed
    const OrbitSnap* changes;           // the last parse call's change tables, [n_channels][change_stride]
    const int* change_counts;           // [n_channels]
    int change_stride;
    const double* doppler;              // channel c, millisecond m at c * doppler_channel_stride + m * doppler_ms_stride
    long long doppler_channel_stride;   // (in doubles: a caller's [n_channels][n_ms] array or the tracking records)
    int doppler_ms_stride;
    const int* order;                   // [n_channels] the fix call's world-model order
    const FixBank* bank;                // its n_touched
    VelocityRecord* out;                // [n_ms]
    int n_ms;
};
cudaError_t launch_velocity_fixes(const VelocityArgs& a, cudaStream_t st);

// signal_windows: C/N0 and phase-lock windows of every channel's tracking records (signal.cu, signal_core.cuh).
struct SignalState;
struct SignalWindow;
struct SignalArgs {
    const TrackMsRecord* records;  // [n_channels][n_ms] as written by k_track_channels
    const double* start_times;     // [n_ms] chunk start timestamps
    SignalState* states;           // [n_channels] carried from call to call
    SignalState* carried;          // [n_channels] scratch: the states as the call found them
    int* stop;                     // [n_channels] scratch: the channel's first lost record in the call (>= n_ms: none)
    SignalWindow* out;             // [n_channels][max_windows]
    int* counts;                   // [n_channels] windows produced (may exceed max_windows: truncated)
    double floor_dbhz;             // signal_noise_floor_dbhz(N)
    int n_ms, n_channels, window_ms, max_windows;
};
cudaError_t launch_signal_windows(const SignalArgs& a, cudaStream_t st);

// acquire_fused: one CTA per (PRN, Doppler) cell, the whole pipeline in one kernel (fused.cu).
struct FusedArgs {
    const float2* iq;       // [M*N] one block
    const double* doppler;  // [n_cells]
    const int* prn;         // [n_cells] replica row
    const int* probe;       // [n_cells] coherent probe index or -1 (may be null)
    CellRecord* records;    // [n_cells]
    const float2* crep;
    const float2* tw1;
    const float2* tw2;
    double inv_fs;
    int N, M, n_cells;
};
bool fused_supports(int s);
cudaError_t configure_fused_kernel();
cudaError_t launch_acquire_fused(const FusedArgs& a, int s, int kind, cudaStream_t st);

size_t track_smem_bytes(int N, int s);
cudaError_t configure_track_kernel();
cudaError_t launch_track_channels(const TrackArgs& a, cudaStream_t st);
cudaError_t launch_integrate_bits(const BitArgs& a, cudaStream_t st);
cudaError_t launch_decode_subframes(const NavArgs& a, cudaStream_t st);
size_t spectra_smem_bytes(int s);
bool spectra_supports(int s);
cudaError_t launch_init_tables(float2* tw1, float2* tw2, cudaStream_t st);
cudaError_t launch_replica_spectra(const uint8_t* chips_dev, int n_prn, float2* crep, float2* crep1023, cudaStream_t st);
cudaError_t launch_doppler_spectra(const SpectraArgs& a, cudaStream_t st);
// Slots per CTA of the correlate kernel that runs a launch of this kind, M milliseconds and profile output: warps of the
// one-warp-per-transform kernel, or warp pairs of the pair kernel.  rsplit must divide it.
int correlate_slots(int kind, int M, bool profile);
// Whether the correlate launch of (kind, profile) reads spectra made with SpectraArgs::pfa.
bool spectra_pfa(int kind, bool profile);
// Runs the kernel correlate_slots(a.kind, a.M, a.profile != nullptr) describes.
cudaError_t launch_correlate(const CorrelateArgs& a, int grid, cudaStream_t st);
cudaError_t launch_correlate_generic(const float2* iq, const float2* replica, int N, int n_ms, double doppler, double inv_fs,
                                     int kind, float* out, cudaStream_t st);
cudaError_t configure_kernels();

}  // namespace gb
