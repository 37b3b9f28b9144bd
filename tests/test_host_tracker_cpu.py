"""Host-side tracking glue without a GPU: GpsSatelliteTracker.process_samples (tracker.py:331-389 as seen by the caller:
pseudosymbol with the code-phase delay, the histories the visualiser reads, host edits of the loop state pushed to the
device, LostSatelliteLockError) through a stand-in for the native channel whose milliseconds are computed by the tracker
oracle, against the trajectories recorded from the live reference.  The stand-in is test infrastructure."""
import os

import numpy as np
import pytest

from gpu_support import Attrs
from gypsum_b200 import _native
from oracle import tracker_oracle as t

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, FS = 2046, 2046000


class StandInEngine:
    iq_tag = None

    def upload_iq(self, x, tag=None):
        self.x = np.asarray(x)
        self.iq_tag = tag
        self.uploads = getattr(self, "uploads", 0) + 1

    def set_replicas(self, chips):
        self.chips = np.asarray(chips)


class StandInPool:
    """_native.Tracker.pool(...): every seeded slot is a TrackerOracle stepped on the engine's current chunk; keep_undo
    launches remember a deep copy of each launched channel, undo_channel puts it back."""

    @classmethod
    def pool(cls, engine, capacity):
        self = cls()
        self.engine, self.capacity = engine, capacity
        self.ch, self.undo = {}, {}
        self.set_calls, self.launches, self.undos = [], [], []
        return self

    def reset_channel(self, channel, prn_idx, doppler, carrier_phase, code_phase):
        sv = 1 + int(prn_idx)  # row r of the table holds SV r + 1 in these tests
        self.ch[channel] = t.TrackerOracle(sv, doppler, carrier_phase, int(code_phase), FS, N)

    def set_state(self, channel, doppler, carrier_phase, phase_acc, code_phase):
        self.set_calls.append((doppler, carrier_phase, phase_acc, code_phase))
        o_ = self.ch[channel]
        o_.doppler, o_.carrier_phase, o_.phase, o_.code_phase = doppler, carrier_phase, phase_acc, code_phase

    def undo_channel(self, channel):
        self.undos.append(channel)
        self.ch[channel] = self.undo.pop(channel)

    def process_channels(self, channels, n_ms, start_times, want_profiles=False, keep_undo=False):
        import copy

        assert n_ms == 1
        self.launches.append(list(channels))
        t0 = float(start_times[0])
        rec = np.zeros((len(channels), 1), dtype=_native.TRACK_DTYPE)
        for i, c in enumerate(channels):
            if keep_undo:
                self.undo[c] = copy.deepcopy(self.ch[c])
            orc, lost = self.ch[c], 0
            try:
                r = orc.step(self.engine.x, t0, round(t0 + N / FS, 6))
            except t.LostLock as exc:
                r, lost = exc.args[0], 1
                r.update(doppler=orc.doppler, carrier_phase=orc.carrier_phase)
            for k in ("doppler", "carrier_phase", "doppler_hist", "carrier_phase_hist", "error", "disc", "strength",
                      "code_phase", "symbol", "peak_offset"):
                rec[k][i, 0] = r[k]
            rec["phase_acc"][i, 0], rec["locked"][i, 0], rec["lost"][i, 0] = orc.phase, int(r["locked"]), lost
            rec["peak_re"][i, 0], rec["peak_im"][i, 0] = r["peak"].real, r["peak"].imag
        prof = np.zeros((len(channels), 1, N), dtype=np.float32)
        return (rec, prof) if want_profiles else rec


class Chunk:
    def __init__(self, k, x):
        self.start_time, self.end_time = t.chunk_times(k, FS, N)
        self.samples = x[k * N:(k + 1) * N]


def _world(monkeypatch):
    from gypsum_b200 import tracker as trk_mod
    from gypsum_b200 import utils
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals

    ent = {"engine": StandInEngine(), "codes": {}, "table": []}
    monkeypatch.setattr(utils.POOL, "get", lambda fs, n, device=0: ent)
    monkeypatch.setattr(trk_mod._native, "Tracker", StandInPool)
    codes = generate_replica_prn_signals()
    # register SVs 1..32 so that table row r is SV r + 1 (what the stand-in assumes)
    for s in range(1, 33):
        utils.POOL.replica_index(ent, np.ascontiguousarray(np.asarray(codes[GpsSatelliteId(s)].inner) != 0, dtype=np.uint8))
    return ent, codes, trk_mod


def _add_tracker(world, sv, init, profiles=True):
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId
    from gypsum_b200.satellite import GpsSatellite

    ent, codes, trk_mod = world
    params = trk_mod.GpsSatelliteTrackingParameters(
        satellite=GpsSatellite(GpsSatelliteId(sv), codes[GpsSatelliteId(sv)], 2), current_doppler_shift=init[0],
        current_carrier_wave_phase_shift=init[1], current_prn_code_phase_shift=int(init[2]), doppler_shifts=[])
    return trk_mod.GpsSatelliteTracker(params, Attrs(FS, N), keep_correlation_profiles=profiles), params


def _tracker(monkeypatch, sv, init):
    world = _world(monkeypatch)
    trk, params = _add_tracker(world, sv, init)
    return trk, params, world[2]


def _case(name):
    z = np.load(os.path.join(ROOT, "tests", "golden", f"tracker_{name}.npz"))
    ch = z["channel"]
    ch = (int(ch[0]), ch[1], ch[2], int(ch[3]), ch[4], ch[5])
    return z, ch, t.synth_tracking_iq(int(z["seed"]), N, int(z["n_ms"]), FS, [ch], float(z["sigma"]))


def test_process_samples_fills_the_reference_histories(monkeypatch):
    z, ch, x = _case("short")
    trk, params, _ = _tracker(monkeypatch, ch[0], z["init"])
    rows = z["rows"]
    for k in range(300):
        ps = trk.process_samples(Chunk(k, x))
        g = rows[k]
        assert (ps.pseudosymbol.as_val(), ps.start_of_pseudosymbol, ps.end_of_pseudosymbol) == (int(g[3]), g[9], g[10])
        assert (params.current_doppler_shift, params.current_carrier_wave_phase_shift,
                params.current_prn_code_phase_shift, trk.phase) == (g[6], g[7], int(g[8]), g[11])
    # what tracker.py:299-353 appends per millisecond
    assert len(params.doppler_shifts) == len(params.carrier_wave_phases) == len(params.carrier_wave_phase_errors) == 300
    assert len(params.correlation_peaks_rolling_buffer) == len(params.correlation_peak_angles) == 300
    assert len(params.discriminators) == 600 and len(params.non_coherent_correlation_profiles) == 250
    assert params.doppler_shifts[-1] == rows[299, 6] and params.carrier_wave_phase_errors[-1] == rows[299, 4]
    assert abs(params.correlation_peaks_rolling_buffer[-1] - complex(rows[299, 0], rows[299, 1])) <= 1e-6 * abs(rows[299, 0])
    assert trk._pool.native.set_calls == []  # no host edits: nothing pushed


def test_host_edits_of_the_loop_state_reach_the_channel(monkeypatch):
    z, ch, x = _case("short")
    trk, params, _ = _tracker(monkeypatch, ch[0], z["init"])
    trk.process_samples(Chunk(0, x))
    params.current_doppler_shift += 2.5  # e.g. the pipeline's re-acquisition path (pipeline.py:104-147)
    trk.process_samples(Chunk(1, x))
    calls = trk._pool.native.set_calls
    assert len(calls) == 1 and calls[0][0] == pytest.approx(float(z["rows"][0, 6]) + 2.5)
    trk.process_samples(Chunk(2, x))
    assert len(calls) == 1


def test_lost_lock_surfaces_as_the_reference_exception(monkeypatch):
    z, ch, x = _case("noise")
    trk, params, trk_mod = _tracker(monkeypatch, ch[0], z["init"])
    lost_at = int(z["lost_at"])
    with pytest.raises(trk_mod.LostSatelliteLockError):
        for k in range(lost_at + 1):
            trk.process_samples(Chunk(k, x))
    assert len(params.doppler_shifts) == lost_at + 1  # the failing millisecond's histories were appended first (tracker.py:346-353, :378)


def test_histories_hold_the_state_before_the_six_second_adjustment(monkeypatch):
    """tracker.py:352-353 append to doppler_shifts / carrier_wave_phases before :380-387 nudge current_*: on the
    millisecond of the adjustment the two differ by 5 Hz / pi/2, exactly as recorded from the live reference."""
    z, ch, x = _case("adjust")
    trk, params, _ = _tracker(monkeypatch, ch[0], z["init"])
    rows = z["rows"]
    for k in range(6001):
        trk.process_samples(Chunk(k, x))
    g = rows[6000]
    assert (params.current_doppler_shift, params.current_carrier_wave_phase_shift) == (g[6], g[7])
    assert (params.doppler_shifts[-1], params.carrier_wave_phases[-1]) == (g[12], g[13])
    assert params.current_doppler_shift - params.doppler_shifts[-1] == 5.0


def test_trackers_sharing_a_chunk_share_one_launch_and_one_upload(monkeypatch):
    """receiver.py:237-257 hands one chunk to every tracked satellite in turn: the first call advances every channel, the
    others find their millisecond computed; results equal each tracker run on its own."""
    za, cha, xa = _case("short")
    world = _world(monkeypatch)
    ta, pa = _add_tracker(world, cha[0], za["init"], profiles=False)
    tb, pb = _add_tracker(world, 7, (-2210.0, 0.5, 100), profiles=False)
    native, eng = ta._pool.native, world[0]["engine"]
    syms = []
    for k in range(30):
        c = Chunk(k, xa)
        syms.append((ta.process_samples(c).pseudosymbol.as_val(), tb.process_samples(c).pseudosymbol.as_val()))
    assert len(native.launches) == 30 and all(sorted(l) == sorted([ta._channel, tb._channel]) for l in native.launches)
    assert eng.uploads == 30 and native.undos == []
    assert [s[0] for s in syms] == [int(v) for v in za["rows"][:30, 3]]
    solo = t.TrackerOracle(7, -2210.0, 0.5, 100, FS, N)
    want = [solo.step(xa[k * N:(k + 1) * N], *t.chunk_times(k, FS, N))["symbol"] for k in range(30)]
    assert [s[1] for s in syms] == want and pb.current_doppler_shift == solo.doppler


def test_a_step_computed_ahead_is_taken_back_when_it_was_not_asked_for(monkeypatch):
    """Channel B is advanced together with A through chunk 0, but is then asked about chunk 1 (it skipped 0), and later
    has its loop state edited while a step is waiting: both times the step is undone and recomputed from the right
    state, so B's results equal B run alone on exactly the chunks it was asked about."""
    za, cha, xa = _case("short")
    world = _world(monkeypatch)
    ta, _ = _add_tracker(world, cha[0], za["init"], profiles=False)
    tb, pb = _add_tracker(world, 7, (-2210.0, 0.5, 100), profiles=False)
    native = ta._pool.native
    solo = t.TrackerOracle(7, -2210.0, 0.5, 100, FS, N)
    ta.process_samples(Chunk(0, xa))                      # B computed ahead for chunk 0 ...
    got = tb.process_samples(Chunk(1, xa))                # ... but asked about chunk 1
    assert native.undos == [tb._channel]
    assert got.pseudosymbol.as_val() == solo.step(xa[N:2 * N], *t.chunk_times(1, FS, N))["symbol"]
    assert pb.current_doppler_shift == solo.doppler
    ta.process_samples(Chunk(2, xa))                      # (A itself was computed ahead for chunk 1, never asked: undone) B ahead for chunk 2
    pb.current_doppler_shift += 1.25                      # host edit before B is asked
    solo.doppler += 1.25
    got = tb.process_samples(Chunk(2, xa))
    assert native.undos == [tb._channel, ta._channel, tb._channel] and len(native.set_calls) == 1
    assert got.pseudosymbol.as_val() == solo.step(xa[2 * N:3 * N], *t.chunk_times(2, FS, N))["symbol"]
    assert pb.current_doppler_shift == solo.doppler


def test_tracker_keeps_working_after_it_raised_lost_lock(monkeypatch):
    """The reference object simply processes the next chunk after raising (tracker.py:378 has no latch)."""
    z, ch, x = _case("noise")
    trk, params, trk_mod = _tracker(monkeypatch, ch[0], z["init"])
    lost_at = int(z["lost_at"])
    for k in range(lost_at):
        trk.process_samples(Chunk(k, x))
    with pytest.raises(trk_mod.LostSatelliteLockError):
        trk.process_samples(Chunk(lost_at, x))
    # the noise golden stops at the raise; the next chunk of the same stream is still processed
    x2 = t.synth_tracking_iq(99, N, 2, FS, [ch], float(z["sigma"]))
    c = Chunk(0, x2)
    c.start_time, c.end_time = t.chunk_times(lost_at + 1, FS, N)
    ps = trk.process_samples(c)
    assert ps.pseudosymbol.as_val() in (-1, 1) and len(params.doppler_shifts) == lost_at + 2
