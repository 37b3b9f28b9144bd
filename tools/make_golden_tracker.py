"""Generate tests/golden/tracker_*.npz by running the LIVE reference tracker (/root/reference/gypsum/tracker.py).
Run:  python tools/make_golden_tracker.py [name ...]     (all cases: ~1 min; np.savez_compressed stamps the time, so
regenerate only the cases you add)"""
import os
import sys
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, "/root/reference")
warnings.filterwarnings("ignore", category=DeprecationWarning)

from gypsum.antenna_sample_provider import AntennaSampleChunk, SampleProviderAttributes  # noqa: E402
from gypsum.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals  # noqa: E402
from gypsum.satellite import GpsSatellite  # noqa: E402
from gypsum.tracker import GpsSatelliteTracker, GpsSatelliteTrackingParameters, LostSatelliteLockError  # noqa: E402

from oracle import tracker_oracle as t  # noqa: E402  (synthetic input + timestamps only)

OUT = os.path.join(ROOT, "tests", "golden")
N, FS = 2046, 2046000


def run(name, seed, n_ms, channel, init, sigma=0.02, N=N, FS=FS, ms_of=None):
    """ms_of(k): the stream millisecond whose timestamps chunk k carries (default k).  A case with ms_of records its
    start / end times, and its samples are synthesised from the first chunk's start time on (a later gap in the times
    is a gap in the timestamps only)."""
    codes = generate_replica_prn_signals()
    sv = channel[0]
    times = [t.chunk_times(k if ms_of is None else ms_of(k), FS, N) for k in range(n_ms)]
    x = t.synth_tracking_iq(seed, N, n_ms, FS, [channel], sigma, t0=times[0][0])
    # prn_as_complex is lru-cached per satellite id (satellite.py:20-21): a cached replica of another rate would collide
    GpsSatellite.prn_as_complex.fget.cache_clear()
    sat = GpsSatellite(GpsSatelliteId(sv), codes[GpsSatelliteId(sv)], N // 1023)
    params = GpsSatelliteTrackingParameters(satellite=sat, current_doppler_shift=init[0],
                                            current_carrier_wave_phase_shift=init[1],
                                            current_prn_code_phase_shift=init[2], doppler_shifts=[])
    trk = GpsSatelliteTracker(params, SampleProviderAttributes(FS, N))
    rows, lost_at = [], -1
    for k in range(n_ms):
        t0, t1 = times[k]
        try:
            ps = trk.process_samples(AntennaSampleChunk(t0, t1, x[k * N:(k + 1) * N]))
        except LostSatelliteLockError:
            lost_at = k
            break
        pk = params.correlation_peaks_rolling_buffer[-1]
        rows.append([pk.real, pk.imag, params.correlation_peak_strengths_rolling_buffer[-1], ps.pseudosymbol.as_val(),
                     params.carrier_wave_phase_errors[-1], params.discriminators[-2], params.current_doppler_shift,
                     params.current_carrier_wave_phase_shift, params.current_prn_code_phase_shift,
                     ps.start_of_pseudosymbol, ps.end_of_pseudosymbol, trk.phase,
                     # what the reference APPENDS to its histories (tracker.py:352-353): the values before the 6-second
                     # constellation adjustment of :370-387, which only the current_* fields above include
                     params.doppler_shifts[-1], params.carrier_wave_phases[-1]])
    extra = {} if ms_of is None else {"start_times": np.array(times, dtype=np.float64)[:, 0],
                                      "end_times": np.array(times, dtype=np.float64)[:, 1]}
    np.savez_compressed(os.path.join(OUT, f"tracker_{name}.npz"), seed=np.int64(seed), n_ms=np.int64(n_ms),
                        channel=np.array(channel, dtype=np.float64), init=np.array(init, dtype=np.float64),
                        sigma=np.float64(sigma), rows=np.array(rows, dtype=np.float64), lost_at=np.int64(lost_at),
                        n=np.int64(N), fs=np.int64(FS), **extra)
    r = np.array(rows)
    print(name, "ms", len(rows), "lost_at", lost_at, "final doppler", r[-1, 6], "symbols +/-", (r[:, 3] > 0).sum(), (r[:, 3] < 0).sum())


CASES = {
    # (sv, doppler, doppler rate, code phase, carrier phase, amplitude); init = (doppler, carrier phase, code phase)
    "short": lambda: run("short", 11, 700, (25, 1500.3, 0.0, 777, 0.3, 0.004), (1500.0, 0.0, 777)),
    "long": lambda: run("long", 12, 6300, (7, -2212.7, 0.5, 100, 1.0, 0.005), (-2210.0, 0.5, 100)),  # crosses the 6 s circularity check
    "noise": lambda: run("noise", 13, 6100, (3, 800.0, 0.0, 5, 0.0, 0.0), (800.0, 0.0, 5)),  # no signal: loses lock at the check
    # 4.092 Msps: the reference keeps its hard-wired 2046 (tracker.py:301-303, :319) -- SURVEY F12 -- so the code-phase
    # accumulator wraps at 2046 although a millisecond is 4092 samples; the planted phase stays below 2046
    # weak signal: circularity 0.89 at the 6-second check -> the -+5 Hz / +-pi/2 nudge of tracker.py:380-387 fires
    "adjust": lambda: run("adjust", 21, 6100, (9, 432.1, 0.0, 300, 0.4, 0.0016), (430.0, 0.0, 300)),
    "fs4": lambda: run("fs4", 14, 500, (12, 640.4, 0.0, 1501, 0.7, 0.004), (640.0, 0.0, 1501), N=4092, FS=4092000),
    # the other rates (same 2046 wrap).  1.023 Msps: the accumulator exceeds N = 1023 and np.roll is modular.
    "fs1": lambda: run("fs1", 31, 2000, (12, 640.4, 0.0, 1501, 0.7, 0.004), (640.0, 0.0, 1501), N=1023, FS=1023000),
    "fs8": lambda: run("fs8", 32, 2000, (12, 640.4, 0.0, 1501, 0.7, 0.002), (640.0, 0.0, 1501), N=8184, FS=8184000),
    # 16.368 Msps: the I-pole variance of is_locked() (tracker.py:184-192) sees the noise variance sigma^2 N / 2, so the
    # reference reports lock only at low sigma ...
    "fs16": lambda: run("fs16", 33, 1500, (12, 640.4, 0.0, 1501, 0.7, 0.001), (640.0, 0.0, 1501), sigma=0.01, N=16368,
                        FS=16368000),
    # ... and never at sigma = 0.02; this one crosses the 6-second constellation check
    "fs16_long": lambda: run("fs16_long", 34, 6100, (12, 640.4, 0.0, 1501, 0.7, 0.001), (640.0, 0.0, 1501), N=16368,
                             FS=16368000),
    # Channels that join late, and stream times far from 0.  The 6-second check compares a chunk's start time with the
    # time of the last check, which starts at 0 (tracker.py:221-222, :370-374).
    # joins at 5.5 s: the 6.0-s check sees the 501 peaks since the join and the -+5 Hz / +-pi/2 nudge fires
    "join55": lambda: run("join55", 21, 700, (9, 432.1, 0.0, 300, 0.4, 0.0016), (430.0, 0.0, 300), ms_of=lambda k: 5500 + k),
    # joins at exactly 6.0 s: the check runs on the first millisecond (one peak: nothing to do), then at 12.0 s (nudge)
    "join6": lambda: run("join6", 21, 6100, (9, 432.1, 0.0, 300, 0.4, 0.0016), (430.0, 0.0, 300), ms_of=lambda k: 6000 + k),
    # no signal, joins at 5.75 s: the 6.0-s check on 251 peaks loses it
    "join575_noise": lambda: run("join575_noise", 13, 300, (3, 800.0, 0.0, 5, 0.0, 0.0), (800.0, 0.0, 5),
                                 ms_of=lambda k: 5750 + k),
    # a 7-s gap in the start times after 600 ms: the check fires on the first millisecond after it (nudge)
    "gap": lambda: run("gap", 23, 1200, (9, 432.1, 0.0, 300, 0.4, 0.003), (430.0, 0.0, 300),
                       ms_of=lambda k: k if k < 600 else k + 7000),
    # stream times near one hour and one day: checks at the join (one peak) and 6 s later (nothing to do)
    "hour": lambda: run("hour", 24, 6100, (25, 1500.3, 0.0, 777, 0.3, 0.004), (1500.0, 0.0, 777),
                        ms_of=lambda k: 3599500 + k),
    "day": lambda: run("day", 25, 6100, (25, 1500.3, 0.0, 777, 0.3, 0.004), (1500.0, 0.0, 777),
                       ms_of=lambda k: 86399500 + k),
}

if __name__ == "__main__":
    for name in sys.argv[1:] or CASES:
        CASES[name]()
