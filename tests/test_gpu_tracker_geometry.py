"""Tracking at the edges the golden trajectories never reach: a DLL step of more than a sample, exact ties in the prompt
profile, channels that join late or see a gap in the start times, a pool slot handed to another satellite, banks larger
than one wave of the persistent kernel, unsorted channel subsets and a device ring read at odd slots when N is odd.
k_track_channels / k_track_channels_wide (tracker.cu) and track_update (tracker_core.cuh) against the float64 tracker
oracle and the live reference's trajectories (tests/golden/tracker_*.npz); bounds as in tests/tracker_support.py."""
import numpy as np
import pytest

from gpu_support import Attrs, EngineCache
from oracle import tracker_oracle as t
from tracker_support import (assert_follows_reference, assert_ms_matches_oracle, load_tracker_case, oracle_row,
                             start_times)

pytestmark = pytest.mark.gpu
ALL_RATES = [1, 2, 3, 4, 5, 6, 8, 10, 12, 16]


@pytest.fixture(scope="module")
def engines(native_lib):
    cache = EngineCache()
    yield cache
    cache.close()


def _sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def _same_records(a, b):
    return a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("s", ALL_RATES)
def test_dll_overshoot_reaches_negative_and_past_2046_code_phases(engines, s):
    """Free-running oracle, teacher-forced device, at an amplitude where one DLL step is several samples: each
    millisecond's signal sits one sample late of the oracle's code phase until the phase has gone negative, then one
    sample early until int() of the accumulator has reached 2046 or more (tracker.py:298-303)."""
    from gypsum_b200 import _native

    n, fs = 1023 * s, 1023000 * s
    amp = 150.0 / n
    eng = engines(n)
    trk = _native.Tracker(eng, [24], [1500.0], [0.0], [0])
    tr = t.TrackerOracle(25, 1500.0, 0.0, 0, fs, n)
    tr.phase = 0.5
    seen = []
    for k in range(60):
        down = not any(p < 0 for p in seen)
        lag = tr.code_phase + (1 if down else -1)
        a, b = t.chunk_times(k, fs, n)
        xk = t.synth_tracking_iq(900 + k, n, 1, fs, [(25, 1500.0, 0.0, lag, 0.3, amp)], t0=a)
        trk.set_state(0, tr.doppler, tr.carrier_phase, float(tr.phase), tr.code_phase)
        eng.upload_iq(xk)
        rec = trk.process(1, [a])[0, 0]
        r = tr.step(xk, a, b)
        assert_ms_matches_oracle(rec, r, k)
        seen.append(r["code_phase"])
        if min(seen) < 0 and max(seen) >= 2046:
            break
    assert min(seen) < 0 and max(seen) >= 2046, seen
    trk.close()


@pytest.mark.parametrize("s", ALL_RATES)
def test_all_zero_input_ties_resolve_to_the_first_rolled_index(engines, s):
    """All-zero IQ: every lag of the prompt profile ties at 0, so np.argmax gives rolled index 0 (which sits on branch
    p mod S, usually not the first task), symbol 0 and zero correlators.  One channel per branch, 300 ms; strength (NaN)
    and lock (from ms 250: zero error variance and an empty negative pole) from the oracle."""
    from gypsum_b200 import _native

    n, fs = 1023 * s, 1023000 * s
    phases = [s * ((37 + 11 * r) % (2046 // s - 1)) + r for r in range(s)]  # below 2046: the DLL keeps them
    assert sorted(p % s for p in phases) == list(range(s)) and max(phases) < 2046
    eng = engines(n)
    eng.upload_iq(np.zeros(300 * n, dtype=np.complex64))
    bank = _native.Tracker(eng, [4] * s, [1000.0] * s, [0.0] * s, phases)
    rec = bank.process(300, start_times(300, fs, n))
    tr = t.TrackerOracle(5, 1000.0, 0.0, phases[0], fs, n)
    want = [tr.step(np.zeros(n, dtype=np.complex64), *t.chunk_times(k, fs, n)) for k in range(300)]
    assert all(w["peak_offset"] == 0 and w["symbol"] == 0 and np.isnan(w["strength"]) for w in want)
    locked = np.array([w["locked"] for w in want])
    assert not locked[:250].any() and locked[250:].all()
    for c in range(s):
        r = rec[c]
        assert (r["peak_offset"] == 0).all() and (r["symbol"] == 0).all(), c
        for f in ("peak_re", "peak_im", "early_re", "early_im", "late_re", "late_im", "disc", "error"):
            assert (r[f] == 0).all(), (c, f)
        assert np.isnan(r["strength"]).all() and np.array_equal(r["locked"].astype(bool), locked), c
        assert (r["code_phase"] == phases[c]).all() and not r["lost"].any(), c
    bank.close()
    one = _native.Tracker(eng, [4] * s, [1000.0] * s, [0.0] * s, phases)
    rec1, prof = one.process(2, start_times(2, fs, n), want_profiles=True)
    assert (prof == 0).all() and (rec1["peak_offset"] == 0).all()
    one.close()


LATE = ["join55", "join6", "join575_noise", "gap"]


def _late_expectations(rec, rows, lost_at):
    """Lost and nudge milliseconds exact: the device stops where the reference raised, and its record carries both the
    history value and the nudged one exactly where the reference's does."""
    fired = np.flatnonzero(rows[:, 6] != rows[:, 12])
    assert np.array_equal(np.flatnonzero(rec["doppler"][:len(rows)] != rec["doppler_hist"][:len(rows)]), fired)
    if lost_at >= 0:
        assert int(np.flatnonzero(rec["lost"] == 1)[0]) == lost_at and (rec["lost"][lost_at + 1:] == 2).all()
    else:
        assert not rec["lost"].any()


@pytest.mark.parametrize("name", LATE)
def test_late_start_matches_reference_at_2046_ksps(engines, name):
    """Channels that join at 5.5, 6.0 and 5.75 s (no signal) and a 7-s gap in the start times, against the live
    reference's trajectories: the 6-second check (tracker.py:370-387) fires on the reference's milliseconds."""
    from gypsum_b200 import _native

    z, ch, x, n, fs, tt = load_tracker_case(name)
    init, rows, lost_at = z["init"], z["rows"], int(z["lost_at"])
    eng = engines(n)
    trk = _native.Tracker(eng, [ch[0] - 1], [init[0]], [init[1]], [int(init[2])])
    n_ms = len(rows) + (1 if lost_at >= 0 else 0)
    eng.upload_iq(x[:n_ms * n])
    rec = trk.process(n_ms, tt[:n_ms, 0])[0]
    trk.close()
    assert_follows_reference(rec[:len(rows)], rows, histories=True)
    _late_expectations(rec, rows, lost_at)


@pytest.mark.parametrize("name", LATE)
def test_late_start_matches_oracle_on_the_wide_kernel(engines, name):
    """The same start times at 5.115 Msps (k_track_channels_wide, odd N) against the float64 oracle's trajectory."""
    from gypsum_b200 import _native

    z, ch, _, _, _, tt = load_tracker_case(name)
    init = z["init"]
    n, fs = 5115, 5115000
    n_ms = len(tt)
    x = t.synth_tracking_iq(int(z["seed"]), n, n_ms, fs, [ch], float(z["sigma"]), t0=float(tt[0, 0]))
    tr = t.TrackerOracle(ch[0], init[0], init[1], int(init[2]), fs, n)
    rows, lost_at = [], -1
    for k in range(n_ms):
        try:
            rows.append(oracle_row(tr, tr.step(x[k * n:(k + 1) * n], *tt[k])))
        except t.LostLock:
            lost_at = k
            break
    rows = np.array(rows)
    n_run = len(rows) + (1 if lost_at >= 0 else 0)
    eng = engines(n)
    trk = _native.Tracker(eng, [ch[0] - 1], [init[0]], [init[1]], [int(init[2])])
    eng.upload_iq(x[:n_run * n])
    rec = trk.process(n_run, tt[:n_run, 0])[0]
    trk.close()
    assert_follows_reference(rec[:len(rows)], rows, histories=True)
    _late_expectations(rec, rows, lost_at)
    assert (lost_at >= 0) == (name == "join575_noise")


@pytest.mark.parametrize("name", ["hour", "day"])
def test_stream_times_of_an_hour_and_a_day_teacher_forced(engines, name):
    """At 3599.5 s and 86399.5 s the reference loop cannot hold lock: a Doppler update df moves the wiped-off phase by
    2 pi df t, so float32 correlators cannot follow its free-running trajectory.  Teacher-forced, every millisecond's
    wipe-off, correlators and loop update match the oracle, and the 6-second check loses the channel on the reference's
    millisecond (the second check, 6 s after the one at the join)."""
    from gypsum_b200 import _native

    z, ch, x, n, fs, tt = load_tracker_case(name)
    init, lost_at = z["init"], int(z["lost_at"])
    tr = t.TrackerOracle(ch[0], init[0], init[1], int(init[2]), fs, n)
    eng = engines(n)
    trk = _native.Tracker(eng, [ch[0] - 1], [init[0]], [init[1]], [int(init[2])])
    for k in range(lost_at + 1):
        a, b = tt[k]
        trk.set_state(0, tr.doppler, tr.carrier_phase, float(tr.phase), tr.code_phase)
        eng.upload_iq(x[k * n:(k + 1) * n])
        rec = trk.process(1, [a])[0, 0]
        try:
            r = tr.step(x[k * n:(k + 1) * n], a, b)
        except t.LostLock as exc:
            r = exc.args[0]
            assert k == lost_at and rec["lost"] == 1
        assert_ms_matches_oracle(rec, r, k)
        assert rec["lost"] == (k == lost_at), k
    trk.close()


def test_pool_slot_reused_for_another_satellite(engines):
    """A pool slot tracks satellite A past its 6-second check, then is reset to satellite B at t = 20 s: B's records
    equal a fresh single-channel tracker of B bit for bit (nothing of A's lock windows, peak ring or check time is kept)
    and follow the oracle."""
    from gypsum_b200 import _native

    n, fs = 2046, 2046000
    eng = engines(n)
    pool = _native.Tracker.pool(eng, 4)
    xa = t.synth_tracking_iq(61, n, 6300, fs, [(7, -2212.7, 0.5, 100, 1.0, 0.005)])
    pool.reset_channel(1, 6, -2210.0, 0.5, 100)
    eng.upload_iq(xa)
    ra = pool.process_channels([1], 6300, start_times(6300, fs, n))[0]
    assert ra["locked"].sum() > 0 and not ra["lost"].any()
    tb = np.array([t.chunk_times(20000 + k, fs, n) for k in range(700)])
    xb = t.synth_tracking_iq(62, n, 700, fs, [(25, 1500.3, 0.0, 777, 0.3, 0.004)], t0=20.0)
    pool.reset_channel(1, 24, 1500.0, 0.0, 777)
    eng.upload_iq(xb)
    rb = pool.process_channels([1], 700, tb[:, 0])[0]
    fresh = _native.Tracker(eng, [24], [1500.0], [0.0], [777])
    rf = fresh.process(700, tb[:, 0])[0]
    fresh.close()
    pool.close()
    assert _same_records(rb, rf)
    assert rb["locked"][:250].sum() == 0 and rb["locked"].sum() > 0
    tr = t.TrackerOracle(25, 1500.0, 0.0, 777, fs, n)
    rows = np.array([oracle_row(tr, tr.step(xb[k * n:(k + 1) * n], *tb[k])) for k in range(700)])
    assert_follows_reference(rb, rows, histories=True)


def _mixed_bank(n_ch, s):
    """n_ch channels over four planted satellites: repeated PRNs, Dopplers of both signs, code phases on every branch."""
    planted = [(25, 1500.3, 0.0, 777, 0.3, 0.004), (7, -2212.7, 0.0, 101, 1.0, 0.004), (25, -800.2, 0.0, 1900, 2.0, 0.004),
               (12, 640.4, 0.0, 3, 0.7, 0.004)]  # below 2046, the only code phases the DLL keeps
    seeds = [(sv - 1, round(f), 0.0, cp) for sv, f, _, cp, _, _ in planted]
    rng = np.random.default_rng(s)
    for c in range(4, n_ch):
        seeds.append((int(rng.choice([6, 24, 24, 11, 30])), float(rng.choice([-1, 1]) * rng.integers(0, 5000)), 0.0,
                      int(s * rng.integers(0, 1023) + c % s)))
    return planted, seeds


@pytest.mark.parametrize("s", [2, 16])
def test_bank_larger_than_one_wave(engines, s):
    """SMs + 5 channels in one launch (more CTAs than SMs) == the same channels in banks of 7; the four planted ones
    follow the oracle."""
    from gypsum_b200 import _native

    n, fs, n_ms = 1023 * s, 1023000 * s, 30
    n_ch = _sm_count() + 5
    planted, seeds = _mixed_bank(n_ch, s)
    assert n_ch > _sm_count() and len({c[3] % s for c in seeds}) == s
    x = t.synth_tracking_iq(70 + s, n, n_ms, fs, planted)
    ts = start_times(n_ms, fs, n)
    eng = engines(n)
    eng.upload_iq(x)
    big = _native.Tracker(eng, *[list(v) for v in zip(*seeds)])
    rec = big.process(n_ms, ts)
    big.close()
    for c0 in range(0, n_ch, 7):
        small = _native.Tracker(eng, *[list(v) for v in zip(*seeds[c0:c0 + 7])])
        assert _same_records(rec[c0:c0 + 7], small.process(n_ms, ts)), c0
        small.close()
    for c, (sv, *_r) in enumerate(planted):
        tr = t.TrackerOracle(sv, *seeds[c][1:], fs, n)
        rows = np.array([oracle_row(tr, tr.step(x[k * n:(k + 1) * n], *t.chunk_times(k, fs, n))) for k in range(n_ms)])
        assert_follows_reference(rec[c], rows, histories=True)


def test_process_channels_with_an_unsorted_subset(engines):
    """An unsorted subset reaching past the SM count: each record goes to its own slot (== that channel alone), the other
    channels' states stay, and keep_undo + undo_channel + a rerun gives the same records bit for bit."""
    from gypsum_b200 import _native

    s, n_ms = 2, 20
    n, fs = 1023 * s, 1023000 * s
    sm = _sm_count()
    n_ch = sm + 5
    planted, seeds = _mixed_bank(n_ch, s)
    x = t.synth_tracking_iq(80, n, n_ms, fs, planted)
    ts = start_times(n_ms, fs, n)
    eng = engines(n)
    eng.upload_iq(x)
    bank = _native.Tracker(eng, *[list(v) for v in zip(*seeds)])
    sel = [sm + 3, 2, sm + 1, 0, 7, sm + 4, 1]
    before = [bank.get_state(c) for c in range(n_ch)]
    rec = bank.process_channels(sel, n_ms, ts, keep_undo=True)
    for i, c in enumerate(sel):
        one = _native.Tracker(eng, *[[v] for v in seeds[c]])
        assert _same_records(rec[i], one.process(n_ms, ts)[0]), c
        one.close()
    after = [bank.get_state(c) for c in range(n_ch)]
    for c in range(n_ch):
        if c not in sel:
            assert after[c] == before[c], c
        else:
            assert after[c]["code_phase"] == rec[sel.index(c), -1]["code_phase"], c
    for c in sel:
        bank.undo_channel(c)
    assert [bank.get_state(c) for c in range(n_ch)] == before
    again = bank.process_channels(sel, n_ms, ts, keep_undo=True)
    assert _same_records(rec, again)
    bank.close()


def test_process_ring_at_odd_and_even_slots_at_5115_ksps(native_lib):
    """N = 5115 is odd, so every other slot of a DeviceSampleRing starts 8 bytes past a 16-byte boundary.
    TrackerBank.process_ring over 3-ms windows starting at odd and even slots, and across the ring's end, == the same
    bank fed through upload_iq, bit for bit."""
    from gypsum_b200.antenna_sample_provider import AntennaSampleChunk, DeviceSampleRing
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import TrackerBank

    s, n_ms = 5, 45
    n, fs = 1023 * s, 1023000 * s
    attrs = Attrs(fs, n)
    x = t.synth_tracking_iq(90, n, n_ms, fs, [(25, 1500.3, 0.0, 777, 0.3, 0.004), (7, -2212.7, 0.0, 1901, 1.0, 0.004)])
    tt = np.array([t.chunk_times(k, fs, n) for k in range(n_ms)])
    codes = generate_replica_prn_signals()
    sats = {sv: GpsSatellite(GpsSatelliteId(sv), codes[GpsSatelliteId(sv)], s) for sv in (25, 7)}
    seeds = [(sats[25], 1500.0, 0.0, 777), (sats[7], -2210.0, 0.5, 1901)]
    ring_bank, upload_bank = TrackerBank(seeds, attrs), TrackerBank(seeds, attrs)
    ring = DeviceSampleRing(attrs, 10)
    firsts = []
    for k in range(n_ms):
        ring.append(AntennaSampleChunk(tt[k, 0], tt[k, 1], x[k * n:(k + 1) * n]))
        if (k + 1) % 3 == 0:
            w = slice(k - 2, k + 1)
            firsts.append((k - 2) % 10)
            got = ring_bank.process_ring(ring, 3, tt[w, 0])
            want = upload_bank.process(x[w.start * n:w.stop * n], tt[w, 0])
            assert _same_records(got, want), k
    assert {f % 2 for f in firsts} == {0, 1} and 9 in firsts
    ring.native.close()
