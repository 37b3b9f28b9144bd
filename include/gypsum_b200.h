/* gypsum_b200 -- C ABI of the H100 acquisition / tracking correlation engine.
 *
 * The reference (codyd51/gypsum) has no FFI: its boundary for this path is two Python classes and one pure
 * function.  Each entry point below names the reference interface it stands behind (paths relative to the
 * reference checkout).  Plain pointers and sizes only; the library owns every device allocation behind the
 * handle; host arrays belong to the caller and are only read/written during the call.  All functions return 0
 * on success or a GB200_E* code; gb200_last_error() gives the message.  There is no CPU fallback: without a
 * CUDA device gb200_create fails.
 *
 * Threading: one caller thread per engine (the reference is single-threaded, receiver.py:85-146).  Host-pointer
 * entry points return after the results are on the host; *_device entry points only enqueue work on the
 * engine's stream (gb200_set_stream).
 */
#ifndef GYPSUM_B200_H
#define GYPSUM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GB200_ABI_VERSION 2

#define GB200_OK 0
#define GB200_EINVAL 1  /* bad argument            -> ValueError  (utils.py:106) */
#define GB200_ECUDA 2   /* CUDA runtime failure     -> RuntimeError */
#define GB200_ESTATE 3  /* replicas / IQ not loaded -> RuntimeError (acquisition.py:112) */

/* utils.py:23-25  IntegrationType(Enum): Coherent = auto() (1), NonCoherent = auto() (2) */
#define GB200_COHERENT 1
#define GB200_NON_COHERENT 2

typedef struct gb200_engine gb200_engine;

/* One reduced correlation profile (32 bytes).  Replaces the f64[N] profile that utils.py:77-108 returns and
 * that acquisition.py:180-189 immediately reduces with np.max / np.argmax /
 * get_normalized_correlation_peak_strength (utils.py:111-116):
 *     strength = peak / ((sum - count*peak) / (N - count)).                                             */
typedef struct gb200_cell_record {
    float peak;      /* np.max(profile); for coherent integration, max |profile|                */
    int32_t argmax;  /* np.argmax(profile): first index attaining the max, 0..N-1               */
    double sum;      /* sum of all N profile values                                             */
    int32_t count;   /* number of values equal to peak (utils.py:113 drops every one of them)   */
    float probe_re;  /* coherent only: profile[probe_idx] (acquisition.py:136 np.angle input)    */
    float probe_im;
    int32_t reserved;
} gb200_cell_record;

int gb200_abi_version(void);

/* receiver.py:46-66: one engine per stream format.  samples_per_ms must be a multiple of 1023
 * (antenna_sample_provider.py:131-136, SampleProviderAttributes).                                  */
int gb200_create(int device_ordinal, int samples_per_second, int samples_per_ms, gb200_engine** out);
int gb200_destroy(gb200_engine* e);
/* e may be NULL: message of the last failed gb200_create on this thread. */
const char* gb200_last_error(const gb200_engine* e);

/* Work is enqueued on this cudaStream_t (0 / NULL = the engine's own stream). */
int gb200_set_stream(gb200_engine* e, void* cuda_stream);

/* satellite.py:20-31 GpsSatellite.prn_as_complex + gps_ca_prn_codes.py:120-131: chips[n_prn][1023] in {0,1};
 * replica index p in later calls refers to row p.  Builds conj(FFT(replica)) on the device once
 * (the reference redoes np.fft.fft(prn_replica) on every call, utils.py:66).                        */
int gb200_set_replicas(gb200_engine* e, const uint8_t* chips, int n_prn);

/* receiver.py:219 antenna_data: complex64[n_samples] (interleaved float32 I,Q -- the on-disk format of
 * antenna_sample_provider.py:112-119).  upload copies from the host; bind uses a device buffer in place.
 * A pageable iq_host is copied into a staging buffer before upload returns, so the caller may reuse it at once.  From a
 * pinned iq_host the copy is only enqueued: the caller must not rewrite the buffer until a call that synchronises
 * the engine's stream has returned (any call that hands results back to the host, e.g. gb200_acquire_grid).  The same
 * holds for gb200_ring_append and gb200_grid_stream_submit; gb200_acquire_grid_host synchronises before it returns.  */
int gb200_upload_iq(gb200_engine* e, const float* iq_host, int64_t n_samples);
/* iq_device must be 16-byte aligned (the fused and tracking kernels stage it with bulk / cp.async copies). */
int gb200_bind_iq_device(gb200_engine* e, const void* iq_device, int64_t n_samples);

/* receiver.py:68,100,219 rolling_samples_buffer (deque(maxlen=ACQUISITION_INTEGRATION_PERIOD_MS)) on the device: every
 * new millisecond of antenna_sample_provider.py:94-124 is uploaded ONCE (one 8*N-byte copy) and both the detector's
 * 10-ms window and every tracking channel read it in place.  The newest n_ms <= capacity_ms milliseconds are always
 * contiguous in device memory (each millisecond is stored twice, capacity_ms apart).                                  */
typedef struct gb200_ring gb200_ring;
int gb200_ring_create(gb200_engine* e, int capacity_ms, gb200_ring** out);
int gb200_ring_destroy(gb200_ring* r);
/* Append n_ms whole milliseconds (complex64[n_ms * N]) from host memory.  A pinned iq_host is read after the call
 * returns: do not rewrite it before a synchronising call (see gb200_upload_iq).                                  */
int gb200_ring_append(gb200_ring* r, const float* iq_host, int n_ms);
/* The engine's IQ binding := the newest n_ms milliseconds (zero copy); what gb200_detect / gb200_acquire_* /
 * gb200_tracker_process* then read.  n_ms <= min(capacity_ms, milliseconds appended so far).                          */
int gb200_ring_bind_newest(gb200_ring* r, int n_ms);
int gb200_ring_appended(const gb200_ring* r, int64_t* total_ms);

/* Benchmark-shaped search grid (SURVEY.md 8d): the loaded IQ holds n_blocks independent blocks of
 * ms_per_block milliseconds; every (block, prn_idx[a], doppler_hz[b]) cell is one
 * utils.py:77 integrate_correlation_with_doppler_shifted_prn evaluation reduced to a record.
 * out[(block*n_prn + a)*n_doppler + b].
 * Every Doppler a caller passes -- to the grid calls below, gb200_grid_stream_create, gb200_acquire_cells and both
 * gb200_correlation_profile calls -- must be finite: NaN or +-inf is GB200_EINVAL naming the first such index, and
 * nothing is launched (the reference's profile of such a cell is all NaN, which no record can stand for).
 * Every gb200_acquire_grid* call but gb200_acquire_grid_host checks its rules in one order and reports the first one
 * broken: a null output, then an empty grid and the Dopplers, then the segment rules of the semi-coherent and weak
 * grids, then the integration type, the replicas, the bound IQ, the milliseconds and samples asked of it, and the PRN
 * range; nothing is launched on an error.                                                                           */
int gb200_acquire_grid(gb200_engine* e, int n_blocks, int ms_per_block, const int32_t* prn_idx, int n_prn,
                       const double* doppler_hz, int n_doppler, int integration_type, gb200_cell_record* out_host);
int gb200_acquire_grid_device(gb200_engine* e, int n_blocks, int ms_per_block, const int32_t* prn_idx, int n_prn,
                              const double* doppler_hz, int n_doppler, int integration_type, void* out_device);
/* The same grid host to host in ONE call for latency-bound callers (receiver.py:219-224 hands over one window per
 * scan): copy-in, both kernels and copy-out are replayed as one CUDA graph per grid shape, one host synchronisation.
 * iq_host: complex64[n_blocks * ms_per_block * N].  Pageable and pinned buffers are both accepted; with pinned ones
 * (cudaHostAlloc / cudaHostRegister) inputs above 64 KB are read by the copy engine in place and small record sets
 * (<= 256 KB) are stored by the kernel straight into out_host, which saves the two staging copies.  The call
 * synchronises before it returns, so both buffers may be reused, a pinned iq_host rewritten, as soon as it has.      */
int gb200_acquire_grid_host(gb200_engine* e, const float* iq_host, int n_blocks, int ms_per_block, const int32_t* prn_idx,
                            int n_prn, const double* doppler_hz, int n_doppler, int integration_type,
                            gb200_cell_record* out_host);

/* acquisition.py:179-189 applied to every (block, prn) row of a grid on the device: the first Doppler bin with the
 * largest profile maximum, its code phase and strength -- 32 bytes per (block, prn) instead of 32 bytes per cell
 * (SURVEY.md 8e: what a multi-GPU gather has to move).  out[(block * n_prn + a)].                                    */
typedef struct gb200_best_record {
    double doppler_hz;  /* BestNonCoherentCorrelationProfile.doppler_shift                  (acquisition.py:186) */
    double strength;    /* .correlation_strength                                            (acquisition.py:189) */
    float peak;         /* np.max of the winning bin's profile                                                    */
    int32_t code_phase; /* .sample_offset_of_correlation_peak                               (acquisition.py:184) */
    int32_t bin;        /* index of the winning bin in doppler_hz                                                */
    int32_t reserved;
} gb200_best_record;
int gb200_acquire_grid_best(gb200_engine* e, int n_blocks, int ms_per_block, const int32_t* prn_idx, int n_prn,
                            const double* doppler_hz, int n_doppler, int integration_type, gb200_best_record* out_host);
int gb200_acquire_grid_best_device(gb200_engine* e, int n_blocks, int ms_per_block, const int32_t* prn_idx, int n_prn,
                                   const double* doppler_hz, int n_doppler, int integration_type, void* out_device);

/* Semi-coherent grid for weak signals (no counterpart in the reference, which offers only its two IntegrationTypes):
 * each block's ms_per_block milliseconds are cut into K = ms_per_block / coherent_ms segments, each segment's 1-ms
 * correlations are summed coherently, and the K magnitudes are added:  profile = sum_k |sum_{t<T} corr(k*T + t)|.
 * A segment gains 10*log10(T) dB of SNR before its magnitude is taken, and needs Doppler bins of about 1/(2T) s
 * (50 Hz at T = 10 ms).  Records, best records and the layouts of out are those of the gb200_acquire_grid* quartet
 * above over that profile, with the same strength formula.  Rules: coherent_ms >= 1, ms_per_block a multiple of it
 * (a partial segment is GB200_EINVAL, never dropped), and every rule of gb200_acquire_grid, in the order given above.
 * coherent_ms == 1 is gb200_acquire_grid(..., GB200_NON_COHERENT), byte for byte.
 * Not handled here (the weak grid below handles both): a navigation data bit edge inside a segment (every 20 ms)
 * cancels part of that segment, up to all of it; code Doppler smears the peak by |f| / 1540 chips per second, as in
 * the non-coherent grid.  There is no detection threshold: the reference's strength threshold was set for its own
 * statistic.                                                                                                        */
int gb200_acquire_grid_semicoherent(gb200_engine* e, int n_blocks, int ms_per_block, int coherent_ms, const int32_t* prn_idx,
                                    int n_prn, const double* doppler_hz, int n_doppler, gb200_cell_record* out_host);
int gb200_acquire_grid_semicoherent_device(gb200_engine* e, int n_blocks, int ms_per_block, int coherent_ms,
                                           const int32_t* prn_idx, int n_prn, const double* doppler_hz, int n_doppler,
                                           void* out_device);
int gb200_acquire_grid_semicoherent_best(gb200_engine* e, int n_blocks, int ms_per_block, int coherent_ms,
                                         const int32_t* prn_idx, int n_prn, const double* doppler_hz, int n_doppler,
                                         gb200_best_record* out_host);
int gb200_acquire_grid_semicoherent_best_device(gb200_engine* e, int n_blocks, int ms_per_block, int coherent_ms,
                                                const int32_t* prn_idx, int n_prn, const double* doppler_hz, int n_doppler,
                                                void* out_device);

/* Weak grid: the semi-coherent grid searched over the navigation data bit phase, with each millisecond realigned by its
 * code Doppler.  With T = coherent_ms, B = bit_phases, M = ms_per_block and the phase step d = T / B, bit phase j
 * (0 <= j < B) sums the K = (M - (B-1)*d) / T segments of milliseconds j*d + k*T .. j*d + k*T + T - 1 of the block:
 *     profile_j[n] = sum_{k<K} | sum_{t<T} corr_aligned(j*d + k*T + t)[n] |
 * One of the B phases keeps every segment inside one 20-ms data bit (within d ms) when B divides T and T divides 20.
 * corr_aligned(m) is millisecond m (counted from the block's first millisecond), wiped off at its own time as in every
 * grid, with its samples moved to row position (n + s_m) mod N before the correlation, where
 *     s_m = rint((double)m * N * f / 1575.42e6)        (evaluated in exactly this order)
 * takes back the code Doppler of a satellite at Doppler f (its lag drifts by -m*N*f/f_L1 samples), so code phases are
 * those of the block's first sample.
 * out holds out[((block * n_prn + a) * B + j) * n_doppler + d]: the Doppler axis folded as B * n_doppler bins, each with
 * the record and strength formula of gb200_acquire_grid.  The best records are the best of each (block, PRN) row's
 * B * n_doppler folded bins: bin = j * n_doppler + d, doppler_hz = doppler_hz[d].
 * Rules: coherent_ms >= 1, bit_phases >= 1 dividing coherent_ms, ms_per_block >= coherent_ms + (B-1)*d and
 * ms_per_block - (B-1)*d a multiple of coherent_ms (a partial segment is GB200_EINVAL, never dropped), and every rule of
 * gb200_acquire_grid, in the order given above.  With B = 1 on a grid where every s_m is 0, the records equal
 * gb200_acquire_grid_semicoherent's byte for byte.  coherent_ms = 1 (B = 1) is a non-coherent grid with realignment.
 * Not handled: a bit edge falls at the satellite's code epoch, inside a millisecond, so even the right phase has up to
 * 1 ms of one segment with the other sign; s_m is a whole sample, which leaves up to 1/2 sample (1/2 chip at 1.023 Msps)
 * of misalignment between milliseconds; there are no weak variants of gb200_acquire_grid_host, the grid streams, cell
 * lists, gb200_detect or the sharded searches.  There is no detection threshold.                                     */
int gb200_acquire_grid_weak(gb200_engine* e, int n_blocks, int ms_per_block, int coherent_ms, int bit_phases,
                            const int32_t* prn_idx, int n_prn, const double* doppler_hz, int n_doppler,
                            gb200_cell_record* out_host);
int gb200_acquire_grid_weak_device(gb200_engine* e, int n_blocks, int ms_per_block, int coherent_ms, int bit_phases,
                                   const int32_t* prn_idx, int n_prn, const double* doppler_hz, int n_doppler, void* out_device);
int gb200_acquire_grid_weak_best(gb200_engine* e, int n_blocks, int ms_per_block, int coherent_ms, int bit_phases,
                                 const int32_t* prn_idx, int n_prn, const double* doppler_hz, int n_doppler,
                                 gb200_best_record* out_host);
int gb200_acquire_grid_weak_best_device(gb200_engine* e, int n_blocks, int ms_per_block, int coherent_ms, int bit_phases,
                                        const int32_t* prn_idx, int n_prn, const double* doppler_hz, int n_doppler,
                                        void* out_device);

/* acquisition.py:154-190 get_best_doppler_shift_estimation / :122-136: an arbitrary list of (prn, Doppler)
 * cells over the first n_ms milliseconds of the loaded IQ.  probe_idx (may be NULL) gives, per cell, the
 * profile index whose complex value is wanted for coherent integration, or -1.                      */
int gb200_acquire_cells(gb200_engine* e, int n_cells, const int32_t* prn_idx, const double* doppler_hz,
                        const int32_t* probe_idx, int n_ms, int integration_type, gb200_cell_record* out_host);

/* acquisition.py:70-152 for a batch of satellites, entirely on the device: the ten refinement passes
 * (spread 7000 Hz halved while >= 10, bins range(int(c-s), int(c+s), int(s/10)), first bin with the largest
 * profile maximum, kept result = strictly greatest strength), then one coherent integration at the kept Doppler.
 * No host round trip between passes.  out[i] belongs to prn_idx[i].                                    */
typedef struct gb200_acquisition_result {
    double doppler_hz;  /* SatelliteAcquisitionAttemptResult.doppler_shift        (acquisition.py:120)       */
    double strength;    /* .correlation_strength                                   (acquisition.py:138)       */
    float probe_re;     /* coherent profile at the kept peak index; np.angle of it */
    float probe_im;     /*   is .carrier_wave_phase_shift                          (acquisition.py:136)       */
    int32_t code_phase; /* .prn_phase_shift                                        (acquisition.py:137)       */
    int32_t reserved;
} gb200_acquisition_result;
int gb200_detect(gb200_engine* e, int n_sv, const int32_t* prn_idx, int n_ms, gb200_acquisition_result* out_host);

/* utils.py:77-108 in full: the N-value profile of one cell.  out_host holds N floats (non-coherent) or
 * 2N floats (coherent, interleaved re,im).                                                          */
int gb200_correlation_profile(gb200_engine* e, int prn_idx, double doppler_hz, int n_ms, int integration_type,
                              float* out_host);
/* The same for ANY replica (utils.py:59-73 / :77-108 accept an arbitrary complex prn_replica of N samples, not only the
 * chips-repeated form GpsSatellite.prn_as_complex produces): replica_host is complex64[N]; the circular correlation is
 * evaluated directly (N^2 multiply-adds, float64 accumulation).  Slow path for the public helpers, never used by the
 * receiver's own calls.                                                                                              */
int gb200_correlation_profile_replica(gb200_engine* e, const float* replica_host, double doppler_hz, int n_ms,
                                      int integration_type, float* out_host);

/* ---------------------------------------------------------------------------------------------------------
 * Tracking (gypsum/tracker.py).  A tracker is a bank of channels sharing the engine's loaded IQ stream; every
 * channel is one GpsSatelliteTracker (tracker.py:206-389): state {Doppler, carrier phase, code phase} seeded
 * from an acquisition result (satellite_signal_processing_pipeline.py:56-62).
 * --------------------------------------------------------------------------------------------------------- */
typedef struct gb200_tracker gb200_tracker;

/* One millisecond of one channel (112 bytes): what GpsSatelliteTracker.process_samples (tracker.py:331-389)
 * leaves in tracking_params' histories plus the emitted pseudosymbol.                                        */
typedef struct gb200_track_record {
    double doppler;        /* current_doppler_shift when process_samples returns (tracker.py:260, :385)      */
    double carrier_phase;  /* current_carrier_wave_phase_shift when it returns   (tracker.py:258-259, :386)   */
    double error;          /* Costas discriminator I*Q                       (tracker.py:249, :261)           */
    double disc;           /* (|E|^2 - |L|^2) / 2                            (tracker.py:297, :300)           */
    double phase_acc;      /* self.phase after the update                    (tracker.py:298-303)             */
    double doppler_hist;       /* what :352 appends to doppler_shifts: the value BEFORE the 6-s adjustment of :380-387 */
    double carrier_phase_hist; /* what :353 appends to carrier_wave_phases, likewise                          */
    float peak_re, peak_im; /* coherent prompt correlation peak              (tracker.py:313, :346)           */
    float strength;        /* get_normalized_correlation_peak_strength       (tracker.py:311, :347)           */
    float early_re, early_im, late_re, late_im; /* np.correlate taps         (tracker.py:293-295)             */
    int32_t code_phase;    /* current_prn_code_phase_shift after this ms     (tracker.py:299)                 */
    int32_t symbol;        /* sign(Re peak): +1 / -1 (0 only if Re peak == 0) (tracker.py:316)                */
    int32_t locked;        /* is_locked() used for this ms's loop bandwidth  (tracker.py:251)                 */
    int32_t lost;          /* 1: LostSatelliteLockError raised at this ms (tracker.py:378); 2: channel already stopped */
    int32_t peak_offset;   /* np.argmax of the prompt profile                (tracker.py:310)                 */
    int32_t reserved[2];
} gb200_track_record;

/* satellite_signal_processing_pipeline.py:56-63: one channel per (replica row, Doppler, carrier phase, code
 * phase).  Works at every rate gb200_create accepts (samples_per_ms / 1023 in {1, 2, 3, 4, 5, 6, 8, 10, 12,
 * 16}).  By default, like the reference, the code-phase accumulator wraps at 2046 and the pseudosymbol delay is code
 * phase / 2046 ms at every rate (tracker.py:301-303,319): above 2.046 Msps only code phases below 2046 can be kept.
 * gb200_tracker_set_code_phase_mode(GB200_CODE_PHASE_SAMPLES) keeps every code phase in [0, N) at every rate.     */
int gb200_tracker_create(gb200_engine* e, int n_channels, const int32_t* prn_idx, const double* doppler_hz,
                         const double* carrier_phase, const int32_t* code_phase, gb200_tracker** out);
int gb200_tracker_destroy(gb200_tracker* t);
/* tracker.py:331 process_samples for n_ms consecutive 1-ms chunks of the engine's loaded IQ, every channel.
 * start_times[n_ms]: AntennaSampleChunk.start_time of each chunk.  out_host[channel*n_ms + ms].
 * profiles_host (may be NULL): [channel][ms][N] |prompt correlation profile| (tracker.py:309), float32.      */
int gb200_tracker_process(gb200_tracker* t, int n_ms, const double* start_times, gb200_track_record* out_host,
                          float* profiles_host);
/* Enqueue only; records stay on the device (out_device: n_channels*n_ms records). */
int gb200_tracker_process_device(gb200_tracker* t, int n_ms, const double* start_times, void* out_device);
/* Read / overwrite the loop state of one channel (tracking_params.current_* and tracker.phase). */
int gb200_tracker_get_state(gb200_tracker* t, int channel, double* doppler_hz, double* carrier_phase, double* phase_acc,
                            int32_t* code_phase, int32_t* lost);
/* set_state also clears the channel's `lost` flag (the reference tracker object keeps working after it raised). */
int gb200_tracker_set_state(gb200_tracker* t, int channel, double doppler_hz, double carrier_phase, double phase_acc,
                            int32_t code_phase);

/* A pool of channel slots for callers that create and drop trackers one at a time (receiver.py:226-267: one
 * GpsSatelliteTracker per acquired satellite, dropped on LostSatelliteLockError).  gb200_tracker_create_pool makes
 * `capacity` idle slots; gb200_tracker_reset_channel seeds one like satellite_signal_processing_pipeline.py:56-63 does
 * (fresh histories, lost = 0).  gb200_tracker_process_channels is gb200_tracker_process for a chosen subset in ONE
 * launch: out_host[i * n_ms + ms] belongs to channels[i].  With keep_undo != 0 every launched channel's state before
 * the call is kept, and gb200_tracker_undo_channel puts it back -- used by the drop-in GpsSatelliteTracker objects,
 * which advance all channels that share a chunk with one launch when the first of them is asked
 * (receiver.py:103-106 loops the same chunk over every pipeline) and take the step back for a channel that turns
 * out not to be asked.                                                                                                */
int gb200_tracker_create_pool(gb200_engine* e, int capacity, gb200_tracker** out);
int gb200_tracker_reset_channel(gb200_tracker* t, int channel, int32_t prn_idx, double doppler_hz, double carrier_phase,
                                int32_t code_phase);
int gb200_tracker_process_channels(gb200_tracker* t, int n_sel, const int32_t* channels, int n_ms, const double* start_times,
                                   int keep_undo, gb200_track_record* out_host, float* profiles_host);
int gb200_tracker_undo_channel(gb200_tracker* t, int channel);

/* A pipelined stream of equally shaped grid batches -- the receiver's steady state (receiver.py:85-146 hands over one
 * block after another): `submit` copies a batch of n_blocks*M*N complex64 samples from host memory, runs the grid of
 * gb200_acquire_grid on it and sends the n_blocks*P*D records to out_host; `collect` waits for the OLDEST batch in
 * flight.  Up to `depth` batches are in flight: the host->device copy of batch k+1 and the device->host copy of batch
 * k-1 run on their own streams under the kernels of batch k.  iq_host / out_host are DMA'd directly when they are
 * pinned, staged otherwise; both must stay valid, and a pinned iq_host unchanged, until the batch is collected.  While
 * a stream exists it owns the engine's IQ binding (gb200_upload_iq / gb200_bind_iq_device must be called again before
 * other acquire calls).  A stream needs no IQ bound to be created: each submit binds its own.  destroy waits for the
 * batches in flight; their records are in a pinned out_host by then, and a staged batch's are dropped uncollected.  */
typedef struct gb200_grid_stream gb200_grid_stream;
int gb200_grid_stream_create(gb200_engine* e, int n_blocks, int n_ms, const int32_t* prn_idx, int n_prn,
                             const double* doppler_hz, int n_doppler, int kind, int depth, gb200_grid_stream** out);
int gb200_grid_stream_submit(gb200_grid_stream* g, const float* iq_host, gb200_cell_record* out_host);
int gb200_grid_stream_collect(gb200_grid_stream* g);
int gb200_grid_stream_destroy(gb200_grid_stream* g);

/* Pseudosymbol -> navigation bit integration (gypsum/navigation_bit_intergrator.py), the consumer of the tracker's
 * +-1 stream (satellite_signal_processing_pipeline.py:77-79).  One EmitNavigationBitEvent (:29-39), 32 bytes. */
typedef struct gb200_bit_event {
    double receiver_timestamp;               /* start_of_pseudosymbol of the bit's first symbol      (:188) */
    double trailing_edge_receiver_timestamp; /* end_of_pseudosymbol of its last symbol               (:189) */
    int32_t ms_index;   /* millisecond (within this call) whose symbol completed the bit                    */
    int32_t bit_value;  /* 1 = BitValue.ONE, 0 = BitValue.ZERO, -1 = BitValue.UNKNOWN                (:149-161) */
    int32_t slide;      /* NavigationBitIntegrator.slide when the bit was emitted                           */
    int32_t pad_;
} gb200_bit_event;

/* NavigationBitIntegrator.process_pseudosymbol (:278-288) for every channel over n_ms millisecond records that are
 * in device memory: records_device ([channel][n_ms] gb200_track_record), or NULL for the records the last
 * gb200_tracker_process call of this tracker left on the device (same n_ms).  start_times / end_times: the chunk
 * timestamps (antenna_sample_provider.py:88-91); receiver_timestamp of :278 is the chunk start.  Each channel keeps
 * one integrator (bit phase, queue, health history) across calls; a channel whose record says `lost` stops there.
 * events_host: [channel][max_events]; counts_host: [channel] events produced (> max_events means truncated). */
int gb200_tracker_integrate_bits(gb200_tracker* t, int n_ms, const double* start_times, const double* end_times,
                                 const void* records_device, gb200_bit_event* events_host, int32_t max_events,
                                 int32_t* counts_host);
/* history of one channel's integrator: out[0..7] = emitted_bit_count, failed_bit_count, processed_pseudosymbol_count,
 * slide, determined_bit_phase (-1 = None), previous_bit_phase_decision (-1 = None), pseudosymbol_cursor_within_queue,
 * stopped. */
int gb200_tracker_bit_state(gb200_tracker* t, int channel, int64_t out[8]);

/* Navigation-message subframe decoding (gypsum/navigation_message_decoder.py), the consumer of the bit events
 * (satellite_signal_processing_pipeline.py:121-136).  One event, 96 bytes; `kind`:
 *   0  EmitSubframeEvent: a subframe with a valid TLM prelude and HOW subframe id (:263-269);
 *   1  DeterminedSubframePhaseEvent (:141): `phase`, `polarity`;
 *   2  CannotDetermineSubframePhaseEvent (:170): no preamble pair among >= 3600 queued bits, on every such bit;
 *   3  the reference raises ValueError here (subframe 5 whose data id is not 01, navigation_message_parser.py:626):
 *      the channel's decoder stops, and events the same bit produced before are dropped, as the exception drops them.
 * `words` holds the 300 bits the reference's NavigationMessageSubframeParser is given;
 * gb200_tracker_parse_subframes below parses them into NavigationMessageSubframe1..5 fields.  A channel whose decoder
 * raised (kind 3) freezes its orbit state there, as the reference receiver's step never returns from the exception. */
typedef struct gb200_subframe_event {
    double receiver_timestamp;               /* receiver_timestamp of the subframe's first bit             (:203) */
    double trailing_edge_receiver_timestamp; /* trailing edge of its last bit                              (:204) */
    uint32_t words[10];   /* the 300 bits after the polarity flip, 30 per word, IS-GPS-200 bit 1 in bit 29       */
    int32_t kind;         /* 0..3, see above                                                                    */
    int32_t bit_index;    /* bit event (within this call) whose arrival produced the event                      */
    int32_t subframe_id;  /* HOW subframe id 1..5 (kinds 0, 3)                                                   */
    int32_t tow;          /* HOW time-of-week count, 17 bits (kinds 0, 3)                                        */
    int32_t phase;        /* determined_subframe_phase, -1 = None                                                */
    int32_t polarity;     /* +1 POSITIVE, -1 NEGATIVE, 0 None                                                   */
    int32_t parity_ok;    /* bit k: word k+1 meets the IS-GPS-200 parity equations (reported only, as the
                             reference only logs parity failures)                                             */
    int32_t pad_[3];
} gb200_subframe_event;
typedef char gb200_subframe_event_is_96_bytes[sizeof(gb200_subframe_event) == 96 ? 1 : -1]; /* C99 static assert */

/* NavigationMessageDecoder.process_bit_from_satellite (:173-196) for every channel.  bits_device: a device array
 * [channel][bits_stride] of gb200_bit_event with bit_counts_host[channel] events per channel, or NULL for the events
 * the last gb200_tracker_integrate_bits call left on the device (its counts and stride; GB200_ESTATE if there is no
 * such call not yet decoded, GB200_EINVAL if that call truncated a channel's events).  Each channel keeps one decoder
 * across calls; with NULL, a channel whose integrator stopped decodes these bits and then stops.  The queue holds at
 * most 4096 bits: a bit that arrives while 4096 are queued (the reference's queue is unbounded) stops the channel's
 * decoder.  events_host: [channel][max_events]; counts_host: [channel] events produced (> max_events: truncated). */
int gb200_tracker_decode_subframes(gb200_tracker* t, const void* bits_device, const int32_t* bit_counts_host,
                                   int32_t bits_stride, gb200_subframe_event* events_host, int32_t max_events,
                                   int32_t* counts_host);
/* one channel's decoder: out[0..5] = determined_subframe_phase (-1 = None), emitted_subframe_count, polarity
 * (+1 / -1 / 0 = None), queued bits, stopped (0 running, 1 raised, 2 queue overflow, 3 the integrator stopped),
 * bit events processed. */
int gb200_tracker_subframe_state(gb200_tracker* t, int channel, int64_t out[6]);

/* Subframe fields (gypsum/navigation_message_parser.py:426-673), one per kind-0 subframe event, 144 bytes.  Bit-list
 * fields are packed with their first bit most significant.  By subframe id (dataclass order):
 *   1  ints: week_num_mod_1024_bits, l2_p_data_flag; bits: ca_or_p_on_l2 (2), ura_index (4), sv_health (6),
 *      issue_of_data_clock (10); values: estimated_group_delay_differential, t_oc, a_f2, a_f1, a_f0
 *   2  ints: fit_interval_flag; bits: issue_of_data_ephemeris (8), age_of_data_offset (5); values:
 *      correction_to_orbital_radius_sin, mean_motion_difference_from_computed_value, mean_anomaly_at_reference_time,
 *      correction_to_latitude_cos, eccentricity, correction_to_latitude_sin, sqrt_semi_major_axis,
 *      reference_time_ephemeris
 *   3  bits: issue_of_data_ephemeris (8); values: correction_to_inclination_angle_cos, longitude_of_ascending_node,
 *      correction_to_inclination_angle_sin, inclination_angle, correction_to_orbital_radius_cos, argument_of_perigee,
 *      rate_of_right_ascension, rate_of_inclination_angle
 *   4  ints: data_id, page_id
 *   5  bits: data_id (2), satellite_id (6), sv_health (8); values: eccentricity, time_of_ephemeris,
 *      delta_inclination_angle, right_ascension_rate, semi_major_axis_sqrt, longitude_of_ascension_mode,
 *      argument_of_perigree, mean_anomaly_at_reference_time, a_f0, a_f1
 * Every value is exact (powers of two on integers of at most 32 bits).                                            */
typedef struct gb200_subframe_fields {
    int32_t event_index;  /* index of the event among the channel's events of the decode call                      */
    int32_t ms;           /* millisecond (within the call chain) whose bit completed the subframe                  */
    int32_t subframe_id;  /* 1..5                                                                                 */
    int32_t reserved;
    double tow_seconds;   /* HandoverWord.time_of_week_in_seconds (:85-93)                                         */
    int32_t ints[2];
    uint32_t bits[4];
    int32_t bit_widths[4];
    double values[10];
} gb200_subframe_fields;
typedef char gb200_subframe_fields_is_144_bytes[sizeof(gb200_subframe_fields) == 144 ? 1 : -1]; /* C99 static assert */

/* The world model's per-satellite state (gypsum/world_model.py GpsWorldModel), one per channel and kept across calls:
 * handle_subframe_emitted (:707-861) for every subframe, handle_prn_observed once per millisecond while the channel is
 * tracked, and handle_lost_satellite_lock when it is dropped, in the receiver's order (receiver.py:106-137): within a
 * millisecond the dropped channels go first (none of their events of that millisecond count), then every tracked
 * channel counts one PRN, then the subframes of that millisecond reset the count to 0.  Like the reference, parameters
 * of different IODE / IODC issues mix.  A channel's drop is per call: it counts again from the next call on.
 *
 * events_device: a device array [channel][stride] of gb200_subframe_event with counts_host[channel] events, their
 * milliseconds event_ms_host[channel * stride + j] (non-decreasing per channel, in [0, n_ms)), drop_ms_host[channel]
 * (-1 = none) and n_ms; or NULL for the chain: the events the last gb200_tracker_decode_subframes(NULL) call left on the
 * device, of bits from gb200_tracker_integrate_bits(NULL records) over the records of the last gb200_tracker_process
 * call.  On the chain an event's millisecond is its bit's ms_index and a channel drops at its first tracking record
 * with `lost` set or at its first CannotDetermine event (kind 2), and the explicit arguments are ignored; GB200_ESTATE
 * if the chain is broken or already parsed.  GB200_EINVAL if two seeded channels track the same replica row (the world
 * model is keyed by satellite).  fields_host: [channel][max_fields]; field_counts_host: [channel] (> max: truncated). */
int gb200_tracker_parse_subframes(gb200_tracker* t, const void* events_device, const int32_t* counts_host, int32_t stride,
                                  const int32_t* event_ms_host, const int32_t* drop_ms_host, int32_t n_ms,
                                  gb200_subframe_fields* fields_host, int32_t max_fields, int32_t* field_counts_host);
/* One channel's state after the last parse call: params[26] in OrbitalParameterType order (SQRT_SEMI_MAJOR_AXIS ..
 * ESTIMATED_GROUP_DELAY_DIFFERENTIAL), set_mask bit k = params[k] is not None, the PRN count and whether it counts. */
int gb200_tracker_orbit_state(gb200_tracker* t, int channel, double params[26], uint32_t* set_mask, int64_t* prn_count,
                              int32_t* counting);

/* What the world model knows of one satellite at the end of one millisecond (56 bytes).  flags:
 *   1  _can_interrogate_precise_timings_for_satellite (:330-360): tow and dsv are set
 *   2  is_complete(): with flag 1, x, y, z are set
 *   4  counting and prn_count <= 6000 (attempt_position_fix, :582-585)
 *   8  counting (the channel is tracked)
 *  16  frozen (the decoder raised)
 * Values that are not set are NaN.                                                                                  */
typedef struct gb200_sv_observation {
    double tow;        /* _gps_observed_system_time_of_week_for_satellite (:635-705)                               */
    double dsv;        /* its delta_sv_time after the 10th iteration                                               */
    double x, y, z;    /* _get_satellite_position_at_time_of_week(tow) (:410-487), ECEF metres                     */
    int64_t prn_count; /* PRNs since the last HOW, -1 when not counting                                            */
    int32_t flags;
    int32_t reserved;
} gb200_sv_observation;
typedef char gb200_sv_observation_is_56_bytes[sizeof(gb200_sv_observation) == 56 ? 1 : -1]; /* C99 static assert */

/* Every (channel, millisecond) of the last gb200_tracker_parse_subframes call: out[channel * n_ms + ms].  The _device
 * variant only enqueues (out_device: n_channels * n_ms records), for a solver on the device. */
int gb200_tracker_observations(gb200_tracker* t, gb200_sv_observation* out_host);
int gb200_tracker_observations_device(gb200_tracker* t, void* out_device);

/* The world model's position fix for one millisecond (112 bytes): GpsWorldModel.attempt_position_fix (:567-633), which
 * the reference receiver calls every millisecond with the chunk's start time.  A tracker is one receiver: it has one
 * clock slide, which every subframe of any channel resets to tow - trailing_edge_receiver_timestamp (:749-752, the last
 * one of a millisecond wins, channels in order), and one world-model order, in which satellites enter at their first
 * subframe or lost lock.  A millisecond's ready channels have flags 2 and 4; with exactly 4, _compute_position runs 5
 * rounds of 20 Newton iterations from zero, and after each round the slide drops by the clock bias.  With 5 or more,
 * the reference raises; in the least-squares mode (gb200_tracker_set_fix_solver) the same rounds run over all of them,
 * each step the least-squares solution (n_ready holds their number, channel and pseudorange the first four).  status:
 *   0  no fix: fewer than 4 ready, or no slide yet
 *   1  fixed: everything set
 *   2  the reference raises here (5 or more ready: numpy's non-square solve; or an exactly singular system); in the
 *      least-squares mode only an exactly singular 4-row system or a rank-deficient one of 5 or more rows; slide_in
 *      and slide_out hold the slide at the raise
 *   3  stopped: the receiver raised earlier, or a channel's decoder raised (event kind 3) at or before this ms
 * Values that are not set are NaN.  Parity with the reference is a bound (DESIGN.md §6): numpy's LAPACK cannot be
 * matched bit for bit. */
typedef struct gb200_position_fix {
    double receiver_timestamp;
    double slide_in;        /* receiver_clock_slide entering _compute_position                                   */
    double slide_out;       /* and after it                                                                      */
    double clock_bias;      /* ReceiverSolution.clock_bias, seconds                                              */
    double x, y, z;         /* ReceiverSolution.receiver_pos, ECEF metres                                        */
    double pseudorange[4];  /* round 0's get_pseudorange_for_satellite of each row, seconds                      */
    int32_t status;
    int32_t n_ready;        /* channels with flags 2 and 4                                                       */
    int32_t channel[4];     /* the rows in world-model order, -1 where unused                                    */
} gb200_position_fix;
typedef char gb200_position_fix_is_112_bytes[sizeof(gb200_position_fix) == 112 ? 1 : -1]; /* C99 static assert */

/* One record per millisecond of the last gb200_tracker_parse_subframes call, receiver_timestamps_host[n_ms] being the
 * chunk start times; the receiver's slide, order and stop carry to the next call.  GB200_ESTATE if there has been no
 * parse call, if that call's fixes were already computed, or if an earlier parse call's fixes were skipped after the
 * first fix call (the slide chain would have a gap).  The _device variant only enqueues (out_device: n_ms records). */
int gb200_tracker_position_fixes(gb200_tracker* t, const double* receiver_timestamps_host, gb200_position_fix* out_host);
int gb200_tracker_position_fixes_device(gb200_tracker* t, const double* receiver_timestamps_host, void* out_device);
/* Which fix a millisecond with 5 or more ready satellites gets: GB200_FIX_SOLVER_REFERENCE (the default) raises as
 * the reference does, and the receiver stops; GB200_FIX_SOLVER_LEAST_SQUARES solves the reference's equations over
 * every ready satellite by least squares (Gauss-Newton; DESIGN.md §8c) and goes on.  Milliseconds with 4 ready fix
 * alike in both.  GB200_EINVAL for another value; GB200_ESTATE after the tracker's first fix call, since the
 * receiver's slide and stop depend on the mode. */
#define GB200_FIX_SOLVER_REFERENCE 0
#define GB200_FIX_SOLVER_LEAST_SQUARES 1
int gb200_tracker_set_fix_solver(gb200_tracker* t, int solver);
/* How a tracker (bank or pool) counts code phase: GB200_CODE_PHASE_REFERENCE (the default) wraps the DLL accumulator at
 * 2046 and delays each pseudosymbol by code phase / 2046 ms at every rate, as the reference does; GB200_CODE_PHASE_SAMPLES
 * wraps it at N, the engine's samples per millisecond, and delays each pseudosymbol by code phase / N ms, so that a
 * satellite acquired at any code phase in [0, N) stays tracked and its bits, subframes and fixes carry its true delay.
 * The two are the same computation at 2.046 Msps.  Nothing else about the loop changes (DESIGN.md §7).  GB200_EINVAL
 * for another value; GB200_ESTATE after the tracker's first gb200_tracker_process, _process_device, _process_channels
 * or _integrate_bits call, whose accumulators and stamps used the mode in force. */
#define GB200_CODE_PHASE_REFERENCE 0
#define GB200_CODE_PHASE_SAMPLES 1
int gb200_tracker_set_code_phase_mode(gb200_tracker* t, int mode);
/* The receiver's state after the last fix call: the clock slide (NaN = None), whether it has stopped, and
 * order[n_channels]: the channels in world-model order, -1 after the last. */
int gb200_tracker_receiver_state(gb200_tracker* t, double* slide, int32_t* stopped, int32_t* order);
/* Fixes the serial chain recomputed so far.  The fixes of a call run in two parallel passes (DESIGN.md §8c): each fix
 * from the slide its segment's last reset set, then again from the slide the first pass left at the previous fix.
 * Every fix checks that it left, to 4 ulp, the slide the next one started from; from the first one that did not, the
 * call's chain runs again serially, each fix from the slide the fix before it left.  This counts the fixes so
 * recomputed: those after the first miss, up to the first raise, that do not start a segment and whose entering slide
 * differed in any bit from the slide the fix before them left.  A receiver-clock jump inside a segment (a gap in the
 * sample stream) is an input that makes the check fail. */
int gb200_tracker_fix_repairs(gb200_tracker* t, int64_t* n);

/* The receiver's velocity and clock drift, geodetic position and dilution of precision at one millisecond with a
 * solved position fix (128 bytes; DESIGN.md §8d).  The rows are the fix's: channel[0..3] of a four-row fix, every
 * ready channel in world-model order for a least-squares fix of more.  Row i is -u_i . v + c drift = rho'_i - u_i . v_sv,i
 * + c drift_sv,i, u_i the line of sight from the fix position to the satellite, rho'_i = -(c / 1575.42 MHz) * Doppler_i
 * the measured range rate and v_sv, drift_sv the satellite's velocity and clock drift from its ephemeris; solved by least
 * squares in the fix's frame (ECEF, no Sagnac term).  DOP is (G^T G)^-1 of the rows G_i = [-u_i, 1] in east/north/up
 * at the geodetic position.  status:
 *   0  no solved position fix at this millisecond: every number is NaN
 *   1  solved: residual_rms is set with more than four rows (NaN with four)
 *   2  not solvable (rank < 4, or a non-finite input in a row): velocity, drift and DOP are NaN; latitude, longitude
 *      and height are set
 * Values that are not set are NaN. */
typedef struct gb200_velocity_fix {
    double receiver_timestamp; /* the fix's                                                                           */
    double vx, vy, vz;         /* receiver ECEF velocity, m/s                                                         */
    double clock_drift;        /* receiver clock drift, s/s                                                           */
    double latitude_deg, longitude_deg, height; /* WGS-84 geodetic position of the fix, degrees and metres            */
    double gdop, pdop, hdop, vdop, tdop;
    double residual_rms;       /* RMS of the range-rate residuals, m/s                                                */
    int32_t status;
    int32_t n_rows;            /* the rows solved over (the fix's n_ready)                                            */
    int32_t reserved[2];
} gb200_velocity_fix;
typedef char gb200_velocity_fix_is_128_bytes[sizeof(gb200_velocity_fix) == 128 ? 1 : -1]; /* C99 static assert */

/* One record per millisecond of the last gb200_tracker_parse_subframes call, from its position fixes.
 * doppler_device: [n_channels][n_ms] float64 Doppler in Hz on the device, or NULL for the `doppler` field of the
 * tracking records of the gb200_tracker_process call that fed that parse call through the chain.  fixes_device: the
 * n_ms gb200_position_fix records of that parse call on the device, or NULL for those the last
 * gb200_tracker_position_fixes call kept.  The rows of a least-squares fix come from the world-model order the last fix
 * call left.  A pure function of its inputs: the tracker's state does not change.  GB200_ESTATE if there has been no
 * parse call, if its fixes are not computed yet, if doppler_device is NULL and that parse call was not fed by the
 * chain or a later process call replaced its records, or if fixes_device is NULL and the last fix call wrote to caller
 * memory (gb200_tracker_position_fixes_device: pass that buffer).  The _device variant only enqueues (out_device: n_ms
 * records). */
int gb200_tracker_velocity_fixes(gb200_tracker* t, const double* doppler_device, const void* fixes_device,
                                 gb200_velocity_fix* out_host);
int gb200_tracker_velocity_fixes_device(gb200_tracker* t, const double* doppler_device, const void* fixes_device,
                                        void* out_device);
/* The carrier-to-noise density and phase-lock indicator of one tracking channel over one window of W consecutive
 * milliseconds of its tracking records (64 bytes; DESIGN.md §8e).  With P_k the record's prompt (peak_re, peak_im) and
 * s_k its strength, over the window's n records
 *     M2 = sum |P_k|^2 / n,  Pn = (4/pi) sum (|P_k| / s_k)^2 / n,  C/N0 = 10 log10((M2 - Pn) / (Pn * 1 ms)),
 *     PLI = (sum I^2 - sum Q^2) / (sum I^2 + sum Q^2).
 * For noise alone the estimate sits at the floor 10 log10((H_N - 1) / 1 ms), H_N = sum_{k=1..N} 1/k, N the samples per
 * millisecond (38.57 dB-Hz at N = 2046).  status:
 *   0  not estimated: a stop cut the window below 20 records, or a sum is not finite; cn0_dbhz is NaN
 *   1  a signal: cn0_dbhz >= floor + 1 dB
 *   2  nothing distinguishable from noise: cn0_dbhz < floor + 1 dB, or NaN when M2 <= Pn */
typedef struct gb200_signal_window {
    double receiver_timestamp; /* chunk start time of the window's first millisecond                                */
    double cn0_dbhz;           /* C/N0, dB-Hz                                                                        */
    double prompt_power;       /* M2                                                                                 */
    double noise_power;        /* Pn                                                                                 */
    double pll_lock;           /* PLI, -1..1                                                                         */
    int64_t first_ms;          /* the window's first record, counted from the first one this channel's estimator consumed */
    int32_t ms_index;          /* millisecond of this call holding the window's last counted record, -1 = an earlier call */
    int32_t n_ms;              /* records in the window: W, or fewer when a stop cut it                              */
    int32_t locked_ms;         /* of them with `locked` set                                                          */
    int32_t status;
} gb200_signal_window;
typedef char gb200_signal_window_is_64_bytes[sizeof(gb200_signal_window) == 64 ? 1 : -1]; /* C99 static assert */

/* The windows every channel closes over n_ms millisecond records in device memory: records_device ([channel][n_ms]
 * gb200_track_record), or NULL for the records of the last whole-bank gb200_tracker_process call (GB200_ESTATE unless
 * that call held n_ms).  start_times[n_ms]: the chunk start times.  Each channel keeps one estimator across calls:
 * windows are W = window_ms consecutive milliseconds of its records (20 <= W <= 60000), and the window a call leaves
 * open carries into the next call.  Each window's sums run in millisecond order, so the same stream split into calls of
 * any sizes gives byte-identical windows apart from ms_index.  W is fixed by the tracker's first call: another W later
 * is GB200_ESTATE.  A channel stops at its first record with `lost` set, which is not counted: its open window is
 * emitted at once if it holds a record, and the channel emits nothing afterwards, even after gb200_tracker_set_state.
 * Reads the chain and changes none of it.  out_host: [channel][max_windows]; counts_host: [channel] windows produced
 * (> max_windows: truncated). */
int gb200_tracker_signal_windows(gb200_tracker* t, int n_ms, const double* start_times, int32_t window_ms,
                                 const void* records_device, gb200_signal_window* out_host, int32_t max_windows,
                                 int32_t* counts_host);

/* The sizes of what the chain holds, for sizing the outputs of the calls that read it: out[0] = bit events per
 * channel the last gb200_tracker_integrate_bits call kept (its max_events), out[1] = subframe events per channel the
 * last gb200_tracker_decode_subframes call kept (its max_events), out[2] = n_ms of the last
 * gb200_tracker_parse_subframes call, which gb200_tracker_observations and gb200_tracker_position_fixes cover.  Each is
 * 0 before the first such call. */
int gb200_tracker_chain_sizes(const gb200_tracker* t, int32_t out[3]);

/* Kernel selection for gb200_acquire_cells.  Two implementations of the same arithmetic exist:
 *   0  doppler_spectra + correlate_cells: the PRN-independent half of the pipeline (wipe-off, forward transform) is
 *      computed once per distinct Doppler bin and shared by every PRN -- the grid shape (gb200_acquire_grid always
 *      uses it);
 *   1  the single fused block-per-(PRN, Doppler) kernel: IQ chunk and replica spectrum staged by TMA, whole
 *      pipeline in one CTA (2046 / 4092 samples per ms only) -- best when every cell has its own Doppler, as in
 *      the refinement passes of acquisition.py:81-101 (gb200_detect uses it);
 *  -1  (default) choose per call from the number of distinct Doppler values.
 * Results agree to float32 rounding.                                                                   */
int gb200_set_fused(gb200_engine* e, int mode);

/* Kernels launched by this engine so far (bench.py's gpu_launches). */
int gb200_launch_count(const gb200_engine* e, int64_t* out);

/* Measurement aid (bench.py roofline): when enabled, every doppler_spectra (which = 0) / correlate_cells
 * (which = 1) launch is bracketed by CUDA events on the engine's stream; gb200_kernel_timing synchronises and
 * returns the summed device time and the number of launches since timing was enabled.                 */
int gb200_enable_kernel_timing(gb200_engine* e, int on);
int gb200_kernel_timing(gb200_engine* e, int which, double* total_ms, int64_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* GYPSUM_B200_H */
