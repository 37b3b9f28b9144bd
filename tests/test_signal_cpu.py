"""The C/N0 and phase-lock estimator on the CPU: the host build of gypsum_b200/csrc/signal_core.cuh against the float64
oracle (tests/signal_oracle.py) on the prompts the live reference tracker recorded (tests/golden/tracker_*.npz), its
independence from how calls split the stream, its stop rule, the C/N0 it recovers against what the IQ planted, its
noise floor, and the record layout."""
import ctypes as C
import math

import numpy as np
import pytest

import signal_oracle as so
from oracle import tracker_oracle as t
from signal_support import (NOISE_CASES, SIGNAL_CASES, SignalEmulator, assert_windows_match, golden_records,
                            oracle_windows, signal_dtype, track_dtype, without_ms_index)

ALL_CASES = SIGNAL_CASES + NOISE_CASES


@pytest.mark.parametrize("w", [20, 100, 1000])
@pytest.mark.parametrize("name", ALL_CASES)
def test_host_core_equals_oracle_on_golden_rows(name, w):
    rec, ts, n, _ = golden_records(name)
    emu = SignalEmulator(w, n)
    assert emu.floor == so.noise_floor_dbhz(n)
    got = emu.run(rec, ts)
    want = oracle_windows(rec, ts, w, emu.floor)
    assert_windows_match(got, want, name)
    assert len(got) >= min(1, len(rec) // w)


@pytest.mark.parametrize("w", [20, 37, 1000])
@pytest.mark.parametrize("name", ["long", "day", "join575_noise", "gap"])
def test_split_calls_are_byte_identical(name, w):
    """The rows cut at random points into calls (ones of a single millisecond among them) give the windows of one call,
    byte for byte apart from ms_index, which counts within each call."""
    rec, ts, n, _ = golden_records(name)
    whole = SignalEmulator(w, n).run(rec, ts)
    rng = np.random.default_rng(len(name) * 1000 + w)
    for trial in range(3):
        cuts = np.sort(rng.choice(np.arange(1, len(rec)), size=12 + 8 * trial, replace=False))
        cuts = np.unique(np.concatenate([cuts, cuts[:4] + 1]))
        cuts = cuts[cuts < len(rec)]
        emu = SignalEmulator(w, n)
        parts, bounds = [], [0, *cuts, len(rec)]
        for a, b in zip(bounds[:-1], bounds[1:]):
            got = emu.run(rec[a:b], ts[a:b])
            # ms_index is the call's own millisecond of the window's last record, or -1 for an earlier call
            last = got["first_ms"] + got["n_ms"] - 1
            idx = np.where(last >= a, last - a, -1)
            assert np.array_equal(got["ms_index"], idx)
            parts.append(got)
        split = np.concatenate(parts) if parts else np.zeros(0, signal_dtype())
        assert without_ms_index(split) == without_ms_index(whole), trial


def _stop_case(name, w):
    rec, ts, n, _ = golden_records(name)
    return rec, ts, SignalEmulator(w, n)


@pytest.mark.parametrize("w", [20, 100, 700, 1000])
@pytest.mark.parametrize("name,lost_at", [("day", 6000), ("join575_noise", 250)])
def test_stop_rule(name, lost_at, w):
    """A channel stops at its first lost record, which is not counted; the open window is emitted at once if it holds a
    record (status 0 below 20 of them), and nothing follows, in that call or any later one."""
    rec, ts, emu = _stop_case(name, w)
    assert rec["lost"][lost_at] and not rec["lost"][:lost_at].any()
    got = emu.run(rec, ts)
    full, cut = divmod(lost_at, w)
    assert len(got) == full + (1 if cut else 0)
    assert (got["n_ms"][:full] == w).all()
    assert np.array_equal(got["first_ms"], np.arange(len(got)) * w)
    if cut:
        assert got["n_ms"][-1] == cut and got["ms_index"][-1] == lost_at - 1
        if cut < so.MIN_MS:
            assert got["status"][-1] == so.NONE and np.isnan(got["cn0_dbhz"][-1])
        else:
            assert got["status"][-1] != so.NONE
    # nothing after the stop, even with records that are not lost
    more = rec.copy()
    more["lost"] = 0
    assert len(emu.run(more[:300], ts[:300])) == 0
    # the stop at the first millisecond of a later call: the window carried in is emitted with ms_index -1
    emu2 = SignalEmulator(w, 2046)
    first = emu2.run(rec[:lost_at], ts[:lost_at])
    tail = emu2.run(rec[lost_at:], ts[lost_at:])
    assert len(first) == full
    assert len(tail) == (1 if cut else 0)
    if cut:
        assert tail["ms_index"][0] == -1 and tail["n_ms"][0] == cut
        assert without_ms_index(tail) == without_ms_index(got[-1:])


@pytest.mark.parametrize("name", SIGNAL_CASES)
def test_planted_cn0_recovered(name):
    """The mean estimate is within 0.8 dB of the C/N0 the IQ planted (the largest miss, 0.6 dB low at 52 dB-Hz, is the
    signal's own off-peak correlation raising the noise estimate), every window of at least 20 ms reports a signal,
    and windows of 1000 ms vary by under 0.1 dB."""
    rec, ts, n, planted = golden_records(name)
    for w in (20, 100, 1000):
        got = SignalEmulator(w, n).run(rec, ts)
        est = got[got["n_ms"] >= so.MIN_MS]
        if len(est) == 0:
            continue
        assert (est["status"] == so.SIGNAL).all(), (w, est["cn0_dbhz"].min())
        assert abs(est["cn0_dbhz"].mean() - planted) <= 0.8, (w, est["cn0_dbhz"].mean(), planted)
        if w == 1000 and len(est) > 1:
            assert est["cn0_dbhz"].std() <= 0.1


@pytest.mark.parametrize("name", NOISE_CASES)
def test_noise_only_sits_at_the_floor(name):
    """Every window of at least 20 ms of noise alone has status 2, and the mean estimate is the H_N floor within 0.1 dB."""
    rec, ts, n, planted = golden_records(name)
    assert planted is None
    floor = so.noise_floor_dbhz(n)
    for w in (20, 100, 1000):
        got = SignalEmulator(w, n).run(rec, ts)
        est = got[got["n_ms"] >= so.MIN_MS]
        assert (est["status"] == so.NOISE).all(), w
        vals = est["cn0_dbhz"][~np.isnan(est["cn0_dbhz"])]
        if w >= 100 and len(vals):
            assert abs(vals.mean() - floor) <= 0.1, (w, vals.mean(), floor)


def _oracle_stream(n, cn0, n_ms, seed, sigma=0.02):
    """The prompts of the float64 tracker oracle over synthetic IQ with a signal at cn0 dB-Hz (None: noise alone)."""
    fs = 1000 * n
    amp = 0.0 if cn0 is None else math.sqrt(10 ** (cn0 / 10) * sigma * sigma / fs)
    x = t.synth_tracking_iq(seed, n, n_ms, fs, [(5, 1200.0, 0.0, 300, 0.7, amp)], sigma)
    tr = t.TrackerOracle(5, 1200.0, 0.7, 300, fs, n)
    rec = np.zeros(n_ms, dtype=track_dtype())
    ts = np.empty(n_ms)
    for k in range(n_ms):
        a, b = t.chunk_times(k, fs, n)
        r = tr.step(x[k * n:(k + 1) * n], a, b)
        rec[k]["peak_re"], rec[k]["peak_im"], rec[k]["strength"] = r["peak"].real, r["peak"].imag, r["strength"]
        rec[k]["locked"] = int(r["locked"])
        ts[k] = a
    return rec, ts


# measured on these streams (DESIGN.md §8e): the estimate reads high near the floor, where the noise's own peak
# adds to the signal's, and low at high C/N0, where the signal's off-peak correlation raises the noise estimate
SWEEP = [(40, 0.8), (45, 0.4), (50, 0.6), (55, 1.2)]


@pytest.mark.parametrize("n", [2046, 16368])
def test_tracker_oracle_sweep(n):
    """40 to 55 dB-Hz through the float64 tracker oracle at 2.046 and 16.368 Msps, each within its measured bias; the
    estimates rise with the planted C/N0, and from 45 dB-Hz every window reports a signal with the phase locked."""
    means = []
    for i, (cn0, tol) in enumerate(SWEEP):
        rec, ts = _oracle_stream(n, cn0, 600, seed=40 + i)
        emu = SignalEmulator(200, n)
        got = emu.run(rec, ts)
        assert_windows_match(got, oracle_windows(rec, ts, 200, emu.floor))
        m = got["cn0_dbhz"].mean()
        assert abs(m - cn0) <= tol, (cn0, m)
        if cn0 >= 45:
            assert (got["status"] == so.SIGNAL).all() and (got["pll_lock"] >= 0.9).all(), got
        means.append(m)
    assert all(b > a + 3 for a, b in zip(means, means[1:])), means


def test_noise_floor_at_16368():
    """Noise alone at 16.368 Msps: every window has status 2.  At 16 samples per chip neighbouring lags are correlated,
    so the largest of N lags is a little smaller than the H_N of independent ones: the estimate sits 0.2 to 0.5 dB
    below the floor formula, never above it."""
    n = 16368
    rec, ts = _oracle_stream(n, None, 600, seed=9)
    emu = SignalEmulator(200, n)
    got = emu.run(rec, ts)
    floor = so.noise_floor_dbhz(n)
    assert (got["status"] == so.NOISE).all()
    assert floor - 0.5 <= got["cn0_dbhz"].mean() <= floor - 0.2, (got["cn0_dbhz"], floor)


def test_noise_floor_helpers():
    from gypsum_b200.tracker import cn0_noise_floor_dbhz

    for n in (1023, 2046, 4092, 16368):
        assert cn0_noise_floor_dbhz(n) == so.noise_floor_dbhz(n) == SignalEmulator(20, n).floor
    assert round(cn0_noise_floor_dbhz(2046), 2) == 38.57 and round(cn0_noise_floor_dbhz(16368), 2) == 39.68


def test_status_rules():
    """Too few records and non-finite sums are status 0; M2 <= Pn is status 2 with NaN C/N0; the 1-dB margin."""
    floor = so.noise_floor_dbhz(2046)
    assert so.estimate(1.0, 1.0, 1.0, 19, floor)[4] == so.NONE
    assert so.estimate(math.inf, 1.0, 1.0, 20, floor)[4] == so.NONE
    cn0, _, _, _, status = so.estimate(0.0, 0.0, 1.0, 20, floor)
    assert status == so.NOISE and math.isnan(cn0)
    rec = np.zeros(20, dtype=track_dtype())
    rec["peak_re"], rec["strength"] = 1.0, 1.0  # zero-strength records make every sum infinite: not estimated
    rec["strength"][3] = 0.0
    emu = SignalEmulator(20, 2046)
    got = emu.run(rec, np.arange(20) * 1e-3)
    assert got["status"][0] == so.NONE and np.isnan(got["cn0_dbhz"][0])
    assert_windows_match(got, oracle_windows(rec, np.arange(20) * 1e-3, 20, emu.floor))


def test_record_layout_matches_header():
    from hostbuild import host_library

    lib = host_library("signal_emu")
    out = np.zeros(11, dtype=np.int64)
    lib.signal_emu_layout(out.ctypes.data_as(C.c_void_p))
    dt = signal_dtype()
    assert [dt.fields[f][1] for f in dt.names] == list(out[:10])
    assert dt.itemsize == out[10] == 64
