"""GPU parity of the tracking path (tracker.cu + tracker_core.cuh through the C ABI) against trajectories recorded
from the live reference tracker (tests/golden/tracker_*.npz) and the tracker oracle.

Tolerances: correlator outputs (early / late / prompt peak) within 1e-5 of the prompt peak magnitude (float32 vs
float64); pseudosymbols exact; loop state (Doppler, carrier phase) within the stated bounds while the loop is in its
stable regime (SURVEY F11); code phase exact in the teacher-forced test."""
import os

import numpy as np
import pytest

from gpu_support import make_engine
from oracle import gypsum_oracle as o
from oracle import tracker_oracle as t

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
N, FS = 2046, 2046000


class Attrs:
    samples_per_second = FS
    samples_per_prn_transmission = N


def load_case(name):
    z = np.load(os.path.join(GOLDEN, f"tracker_{name}.npz"))
    ch = z["channel"]
    ch = (int(ch[0]), ch[1], ch[2], int(ch[3]), ch[4], ch[5])
    x = t.synth_tracking_iq(int(z["seed"]), N, int(z["n_ms"]), FS, [ch], float(z["sigma"]))
    return z, ch, x


@pytest.fixture(scope="module")
def engine(native_lib):
    e = make_engine(FS, N)
    yield e
    e.close()


def assert_symbols_and_code_phase_follow_reference(rec, rows):
    """Pseudosymbols and code phase are EXACT, bar per-millisecond proofs taken from the reference's own float64 trajectory:
    a symbol may differ only where the reference's in-phase prompt value is float32 noise around zero; the code phase
    (int() of the DLL accumulator, tracker.py:298-299) only where the reference's accumulator sits within 5e-3 of an integer
    and ours within 5e-3 of the reference's."""
    scale = np.abs(rows[:, 0]).max()
    for k in np.flatnonzero(rec["symbol"] != rows[:, 3].astype(int)):
        assert abs(rows[k, 0]) <= 1e-4 * scale, k
    for k in np.flatnonzero(rec["code_phase"] != rows[:, 8].astype(int)):
        frac = rows[k, 11] - np.floor(rows[k, 11])
        assert min(frac, 1 - frac) <= 5e-3 and abs(rec["phase_acc"][k] - rows[k, 11]) <= 5e-3, k


def times(n_ms):
    return np.array([t.chunk_times(k, FS, N)[0] for k in range(n_ms)])


def test_teacher_forced_correlators(engine):
    """Each millisecond starts from the oracle's loop state: early / late / prompt outputs and the updated state."""
    from gypsum_b200 import _native

    z, ch, x = load_case("short")
    init = z["init"]
    tr = t.TrackerOracle(ch[0], init[0], init[1], int(init[2]), FS, N)
    trk = _native.Tracker(engine, [ch[0] - 1], [init[0]], [init[1]], [int(init[2])])
    for k in range(300):
        a, b = t.chunk_times(k, FS, N)
        trk.set_state(0, tr.doppler, tr.carrier_phase, float(tr.phase), tr.code_phase)
        engine.upload_iq(x[k * N:(k + 1) * N])
        rec = trk.process(1, [a])[0, 0]
        r = tr.step(x[k * N:(k + 1) * N], a, b)
        scale = abs(r["peak"])
        assert abs(complex(rec["peak_re"], rec["peak_im"]) - r["peak"]) <= 1e-5 * scale, k
        assert abs(complex(rec["early_re"], rec["early_im"]) - r["early"]) <= 1e-5 * scale, k
        assert abs(complex(rec["late_re"], rec["late_im"]) - r["late"]) <= 1e-5 * scale, k
        assert abs(rec["strength"] - r["strength"]) <= 1e-4 * r["strength"], k
        assert rec["peak_offset"] == r["peak_offset"] and rec["symbol"] == r["symbol"], k
        assert rec["code_phase"] == r["code_phase"], k
        assert abs(rec["disc"] - r["disc"]) <= 1e-4 * max(1.0, abs(r["disc"])), k
        assert abs(rec["error"] - r["error"]) <= 1e-4 * max(1.0, abs(r["error"])), k
    trk.close()


@pytest.mark.parametrize("name", ["short", "long", "adjust"])
def test_free_running_matches_reference(engine, name):
    """One launch over the whole recording: the reference's pseudosymbol stream, Doppler and phase trajectories."""
    from gypsum_b200 import _native

    z, ch, x = load_case(name)
    init, rows = z["init"], z["rows"]
    n_ms = len(rows)
    trk = _native.Tracker(engine, [ch[0] - 1], [init[0]], [init[1]], [int(init[2])])
    engine.upload_iq(x)
    rec = trk.process(n_ms, times(n_ms))[0]
    trk.close()
    assert not rec["lost"].any()
    assert_symbols_and_code_phase_follow_reference(rec, rows)
    assert np.abs(rec["doppler"] - rows[:, 6]).max() <= 5e-3
    d = np.abs(rec["carrier_phase"] - rows[:, 7])
    assert np.minimum(d, 2 * np.pi - d).max() <= 2e-3
    assert np.abs(np.hypot(rec["peak_re"], rec["peak_im"]) - np.hypot(rows[:, 0], rows[:, 1])).max() <= 1e-3
    # histories (tracker.py:352-353) carry the value BEFORE the 6-second adjustment of :380-387 (recorded columns 12, 13)
    assert np.abs(rec["doppler_hist"] - rows[:, 12]).max() <= 5e-3
    d = np.abs(rec["carrier_phase_hist"] - rows[:, 13])
    assert np.minimum(d, 2 * np.pi - d).max() <= 2e-3
    fired = np.flatnonzero(rows[:, 6] != rows[:, 12])
    assert np.array_equal(np.flatnonzero(rec["doppler"] != rec["doppler_hist"]), fired)
    assert (len(fired) == 1 and fired[0] == 6000 and rec["doppler"][6000] - rec["doppler_hist"][6000] == 5.0) if name == "adjust" else len(fired) == 0
    assert rec["locked"].sum() > 0 and rec["locked"][:250].sum() == 0


def test_noise_channel_loses_lock_at_the_six_second_check(engine):
    from gypsum_b200 import _native

    z, ch, x = load_case("noise")
    init = z["init"]
    n_ms = int(z["n_ms"])
    trk = _native.Tracker(engine, [ch[0] - 1], [init[0]], [init[1]], [int(init[2])])
    engine.upload_iq(x)
    rec = trk.process(n_ms, times(n_ms))[0]
    assert int(np.flatnonzero(rec["lost"] == 1)[0]) == int(z["lost_at"]) == 6000
    assert (rec["lost"][6001:] == 2).all() and trk.get_state(0)["lost"] == 1
    trk.close()


def test_bank_of_channels_and_profiles(engine):
    """Several channels over one stream == each channel alone; |prompt profile| matches the oracle."""
    from gypsum_b200 import _native

    chans = [(25, 1500.3, 0.0, 777, 0.3, 0.004), (7, -2212.7, 0.0, 100, 1.0, 0.005), (31, 3000.2, 0.0, 2045, 2.0, 0.004)]
    x = t.synth_tracking_iq(21, N, 60, FS, chans)
    prn = [c[0] - 1 for c in chans]
    dop = [1500.0, -2210.0, 3000.0]
    engine.upload_iq(x)
    bank = _native.Tracker(engine, prn, dop, [0.0, 0.5, 0.0], [777, 100, 2045])
    rec, prof = bank.process(60, times(60), want_profiles=True)
    bank.close()
    for c in range(3):
        one = _native.Tracker(engine, [prn[c]], [dop[c]], [[0.0, 0.5, 0.0][c]], [[777, 100, 2045][c]])
        r1 = one.process(60, times(60))[0]
        one.close()
        for k in ("doppler", "carrier_phase", "peak_re", "code_phase", "symbol"):
            assert np.array_equal(rec[c][k], r1[k]), (c, k)
        assert (prof[c].argmax(axis=1) == rec[c]["peak_offset"]).all()
    tr = t.TrackerOracle(25, 1500.0, 0.0, 777, FS, N)
    y = x[:N] * np.exp(-1j * (2 * np.pi * 1500.0 * (np.arange(N) / FS)))
    ref = np.abs(o.correlate_1ms(y, np.roll(tr.prn, 777)))
    assert np.abs(prof[0][0] - ref).max() <= 1e-5 * ref.max()


def test_drop_in_tracker_class(engine):
    """GpsSatelliteTracker.process_samples, one call per millisecond, fills the reference's histories and returns the
    reference's pseudosymbols; LostSatelliteLockError surfaces from the device flag."""
    from gypsum_b200.antenna_sample_provider import AntennaSampleChunk
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import (GpsSatelliteTracker, GpsSatelliteTrackingParameters, NavigationBitPseudosymbol)

    z, ch, x = load_case("short")
    init, rows = z["init"], z["rows"]
    codes = generate_replica_prn_signals()
    sat = GpsSatellite(GpsSatelliteId(ch[0]), codes[GpsSatelliteId(ch[0])], 2)
    params = GpsSatelliteTrackingParameters(satellite=sat, current_doppler_shift=init[0],
                                            current_carrier_wave_phase_shift=init[1],
                                            current_prn_code_phase_shift=int(init[2]), doppler_shifts=[])
    trk = GpsSatelliteTracker(params, Attrs())
    for k in range(320):
        a, b = t.chunk_times(k, FS, N)
        ps = trk.process_samples(AntennaSampleChunk(a, b, x[k * N:(k + 1) * N]))
        assert ps.pseudosymbol == NavigationBitPseudosymbol.from_val(int(rows[k, 3]))
        assert abs(ps.start_of_pseudosymbol - rows[k, 9]) <= 1e-9 and abs(ps.end_of_pseudosymbol - rows[k, 10]) <= 1e-9
    assert len(params.doppler_shifts) == 320 and len(params.discriminators) == 640
    assert len(params.non_coherent_correlation_profiles) == 250 and params.non_coherent_correlation_profiles[-1].shape == (N,)
    assert abs(params.current_doppler_shift - rows[319, 6]) <= 5e-3
    assert abs(params.correlation_peaks_rolling_buffer[-1] - complex(rows[319, 0], rows[319, 1])) <= 1e-3
    assert isinstance(params.is_locked(), bool)
    with pytest.raises(RuntimeError):
        GpsSatelliteTrackingParameters(satellite=sat, current_doppler_shift=0, current_carrier_wave_phase_shift=0,
                                       current_prn_code_phase_shift=0, doppler_shifts=[], carrier_wave_phases=[])


def test_tracker_bank_class(engine):
    """gypsum_b200.tracker.TrackerBank: channels given as (satellite, doppler, phase, code phase) like
    pipeline.py:56-62 seeds them; one launch for the whole block of milliseconds == the per-millisecond drop-in."""
    from gypsum_b200.antenna_sample_provider import AntennaSampleChunk
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import GpsSatelliteTracker, GpsSatelliteTrackingParameters, TrackerBank

    chans = [(25, 1500.3, 0.0, 777, 0.3, 0.004), (7, -2212.7, 0.0, 100, 1.0, 0.005)]
    x = t.synth_tracking_iq(33, N, 40, FS, chans)
    codes = generate_replica_prn_signals()
    sats = {sv: GpsSatellite(GpsSatelliteId(sv), codes[GpsSatelliteId(sv)], 2) for sv in (25, 7)}
    bank = TrackerBank([(sats[25], 1500.0, 0.0, 777), (sats[7], -2210.0, 0.5, 100)], Attrs())
    rec = bank.process(x, times(40))
    assert rec.shape == (2, 40)
    for c, (sv, f0, p0, cp0) in enumerate([(25, 1500.0, 0.0, 777), (7, -2210.0, 0.5, 100)]):
        params = GpsSatelliteTrackingParameters(satellite=sats[sv], current_doppler_shift=f0,
                                                current_carrier_wave_phase_shift=p0, current_prn_code_phase_shift=cp0,
                                                doppler_shifts=[])
        trk = GpsSatelliteTracker(params, Attrs(), keep_correlation_profiles=False)
        for k in range(40):
            a, b = t.chunk_times(k, FS, N)
            ps = trk.process_samples(AntennaSampleChunk(a, b, x[k * N:(k + 1) * N]))
            assert ps.pseudosymbol.as_val() == rec[c, k]["symbol"]
        assert params.current_doppler_shift == rec[c, -1]["doppler"]
        assert len(params.non_coherent_correlation_profiles) == 0


_FS4_SCRIPT = r"""
import os, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from gypsum_b200 import _native
from oracle import gypsum_oracle as o
from oracle import tracker_oracle as t

z = np.load(os.path.join(sys.argv[1], "tests", "golden", "tracker_fs4.npz"))
n, fs = int(z["n"]), int(z["fs"])
ch = z["channel"]
ch = (int(ch[0]), ch[1], ch[2], int(ch[3]), ch[4], ch[5])
x = t.synth_tracking_iq(int(z["seed"]), n, int(z["n_ms"]), fs, [ch], float(z["sigma"]))
init, rows = z["init"], z["rows"]
eng = _native.Engine(fs, n)
eng.set_replicas(np.stack([o.ca_code(sv) for sv in range(1, 33)]).astype(np.uint8))
eng.upload_iq(x)
trk = _native.Tracker(eng, [ch[0] - 1], [init[0]], [init[1]], [int(init[2])])
tt = np.array([t.chunk_times(k, fs, n)[0] for k in range(len(rows))])
rec = trk.process(len(rows), tt)[0]
assert not rec["lost"].any()
scale = np.abs(rows[:, 0]).max()
for k in np.flatnonzero(rec["symbol"] != rows[:, 3].astype(int)):
    assert abs(rows[k, 0]) <= 1e-4 * scale, k
for k in np.flatnonzero(rec["code_phase"] != rows[:, 8].astype(int)):
    frac = rows[k, 11] - np.floor(rows[k, 11])
    assert min(frac, 1 - frac) <= 5e-3 and abs(rec["phase_acc"][k] - rows[k, 11]) <= 5e-3, k
assert np.abs(rec["doppler"] - rows[:, 6]).max() <= 5e-3
d = np.abs(rec["carrier_phase"] - rows[:, 7])
assert np.minimum(d, 2 * np.pi - d).max() <= 2e-3
print("fs4 ok")
"""


def test_free_running_at_4092_ksps_matches_reference(native_lib):
    """The reference at 4.092 Msps keeps its hard-wired 2046 (tracker.py:301-303, :319; SURVEY F12): the code-phase
    accumulator wraps at 2046 although a millisecond is 4092 samples.  Same bounds as the 2.046 Msps trajectories.
    Runs in its own process (last test of the last GPU file) so that a fault on this never-exercised path cannot
    disturb the CUDA context of the other tests."""
    import subprocess
    import sys

    proc = subprocess.run([sys.executable, "-c", _FS4_SCRIPT, ROOT], capture_output=True, text=True, timeout=300)
    assert proc.returncode == 0 and "fs4 ok" in proc.stdout, proc.stderr[-2000:]
