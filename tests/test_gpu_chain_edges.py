"""The receiver chain's warp scans at every lane, span and call edge.  Three kernels decide things at the edges of fixed
partitions: k_fix_plan (fix.cu) walks a call 32 milliseconds at a time and carries by warp ballots the segment's slide,
the previous fix a pass-2 fix chains from, the link into the next chunk and the first five-ready millisecond, and
k_fix_finish picks the slide the next call starts from; k_signal_stop (signal.cu) scans 1024-record spans, four warps
per block, and joins them with atomicMin; k_parse_subframes (orbit.cu) takes a chain-mode drop by a 32-lane ballot.

The position-fix tests re-split the 14 recorded timelines and the scripted least-squares one (resplit()): every
millisecond where the plan decides something is put at in-call indices 0, 1, 30, 31, 32, 33, 63 and 64, at the end of
its call and alone in a one-millisecond call, and every timeline runs in 33-ms calls at each offset 0 to 32.  Each call
goes through fix_support.ChainCheck against one oracle run sliced to it (tests/test_fix_splits_cpu.py shows the oracle
does not depend on the split) and against the model of the passes bit for bit, the carried slide exactly."""
import os
import time

import numpy as np
import pytest

import fix_lsq_oracle as lo
from fix_support import (ChainCheck, OracleTimeline, call_starts, edge_ms, edge_splits, fix_emulator, resplit, run_calls,
                         scripted_timeline, sweep_cuts)
from gpu_support import make_engine
from oracle import fix_oracle as fx
from signal_support import SignalEmulator, assert_windows_match
from tracker_support import load_tracker_case

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, FS = 2046, 2046000
TIMELINES = [("fix", n) for n in ("realistic", "three", "gate", "lost", "five", "raise")] + \
            [("fix_repair", n) for n in ("gap_mid", "gap_two", "gap_back", "gap_first", "gap_carry", "gap_five",
                                         "gap_raise", "singular")]
IDS = [n for _, n in TIMELINES]


@pytest.fixture(scope="module")
def engine(native_lib):
    e = make_engine(FS, N)
    yield e
    e.close()


@pytest.fixture(scope="module")
def fix_emu():
    return fix_emulator()


_TIMELINES = {}


def _timeline(group, name, fix_emu):
    """(calls, oracle timeline, edge milliseconds, solver) of one timeline, the oracle run once per module."""
    if (group, name) not in _TIMELINES:
        if group is None:
            calls, oracle, solver = scripted_timeline(), lo, "least_squares"
        else:
            z = np.load(os.path.join(ROOT, "tests", "golden", f"{group}.npz"))
            calls, oracle, solver = fx.golden_calls(z, name), fx, "reference"
        tl = OracleTimeline(oracle, calls)
        bounds, _ = call_starts(calls)
        misses = [b + d["first_miss"] for b, d in zip(bounds, tl.model(fix_emu, calls)) if d["first_miss"] is not None]
        _TIMELINES[group, name] = (calls, tl, edge_ms(calls, tl, misses), solver)
    return _TIMELINES[group, name]


def _run_split(engine, fix_emu, calls, tl, solver, cuts, what):
    """The timeline cut at `cuts` on the device, every call through ChainCheck; returns the check."""
    split = resplit(calls, cuts)
    starts, _ = call_starts(split)
    chk = ChainCheck(fix_emu, solver)
    for s, (rx, _), (got, obs, state) in zip(starts, split, run_calls(engine, split, solver=solver)):
        want, resets, order, stopped = tl.call(s, s + len(rx))
        chk(want, resets, order, stopped, got, obs, state, what=(what, s))
    return chk, starts


def _edge_placements(engine, fix_emu, group, name):
    calls, tl, edges, solver = _timeline(group, name, fix_emu)
    t0, n_runs, repaired, worst = time.time(), 0, set(), 0.0
    placed = {p: 0 for p in ("last", "alone", 0, 1, 30, 31, 32, 33, 63, 64)}
    _, total = call_starts(calls)
    for p, cuts, on in edge_splits(calls, edges):
        chk, starts = _run_split(engine, fix_emu, calls, tl, solver, cuts, (name, p))
        ends = starts[1:] + [total]
        for e in on:  # each edge sits where it was placed
            k = max(i for i, s in enumerate(starts) if s <= e)
            if p == "last":
                assert e == ends[k] - 1
            elif p == "alone":
                assert starts[k] == e and ends[k] == e + 1
            else:
                assert e - starts[k] == p
        placed[p] += len(on)
        n_runs += 1
        repaired.add(chk.repaired)
        worst = max(worst, chk.worst[0])
    assert placed["last"] == placed["alone"] == len(edges) and placed[0] == len(edges)
    print(f"{name}: {len(edges)} edges {edges}, placed {placed} in {n_runs} runs; repair counts {sorted(repaired)}; "
          f"worst slide {worst:.3g} ulp; {time.time() - t0:.1f} s")
    return repaired


def _lane_sweep(engine, fix_emu, group, name):
    calls, tl, _, solver = _timeline(group, name, fix_emu)
    t0, repaired = time.time(), []
    for o in range(33):
        chk, _ = _run_split(engine, fix_emu, calls, tl, solver, sweep_cuts(calls, o), (name, "sweep", o))
        repaired.append(chk.repaired)
    print(f"{name}: 33-ms calls at offsets 0-32, repaired {repaired}; {time.time() - t0:.1f} s")
    return repaired


@pytest.mark.parametrize("group,name", TIMELINES, ids=IDS)
def test_edge_placements(engine, fix_emu, group, name):
    """Every edge millisecond of the timeline at every placement, in the reference mode."""
    _edge_placements(engine, fix_emu, group, name)


@pytest.mark.parametrize("group,name", TIMELINES, ids=IDS)
def test_lane_sweep(engine, fix_emu, group, name):
    """33-ms calls at every offset 0 to 32: every millisecond at every lane of chunk 0 and at lane 0 of chunk 1."""
    repaired = _lane_sweep(engine, fix_emu, group, name)
    if name == "gap_first":
        assert len(set(repaired)) > 1  # the split decides how much the serial repair recomputes


def test_least_squares_edge_placements(engine, fix_emu):
    """The scripted six-channel timeline (ready set 6 -> 5 -> 4 inside a segment, a jump repaired over six rows) in the
    least-squares mode, every edge at every placement."""
    _edge_placements(engine, fix_emu, None, "scripted")


def test_least_squares_lane_sweep(engine, fix_emu):
    _lane_sweep(engine, fix_emu, None, "scripted")


# ---- k_signal_stop: 1024-record spans, four warps per block, joined by atomicMin

SIGNAL_FIRST_LOST = (1023, 1024, 1025, 4095, 4096, 4097)


def _device(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def _records(rng, n_ch, n_ms, first_lost):
    """Seeded TRACK_DTYPE records; channel c loses lock at first_lost[c] (None: never) as the tracker writes it: `lost`
    1 there and 2 on every record after it."""
    from gypsum_b200 import _native

    rec = np.zeros((n_ch, n_ms), dtype=_native.TRACK_DTYPE)
    rec["peak_re"] = rng.normal(0.0, 1.0, (n_ch, n_ms)) + 3.0
    rec["peak_im"] = rng.normal(0.0, 1.0, (n_ch, n_ms))
    rec["strength"] = rng.uniform(0.5, 10.0, (n_ch, n_ms))
    rec["locked"] = rng.integers(0, 2, (n_ch, n_ms))
    for c, k in enumerate(first_lost):
        if k is not None:
            rec["lost"][c, k] = 1
            rec["lost"][c, k + 1:] = 2
    return rec


@pytest.mark.parametrize("n_ms", [1024, 4096, 4097, 9000])
def test_signal_stop_spans(engine, n_ms):
    """Four channels of synthetic records, three of them losing lock at span and block edges (1023 to 1025, 4095 to
    4097, the last record) and one never: in one call and in calls cut at 1024 and 4096, at W = 20, 1000 and 1024, every
    channel's windows are the host core's, a stopped channel's last window ends just before its first lost record, and a
    further call emits nothing for the stopped channels."""
    import torch

    from gypsum_b200 import _native

    rng = np.random.default_rng(n_ms)
    firsts = sorted({k for k in SIGNAL_FIRST_LOST + (n_ms - 1,) if k < n_ms})
    ts = 0.001 * np.arange(n_ms)
    n_checked = 0
    for i in range(0, len(firsts), 3):
        first_lost = firsts[i:i + 3] + [None] * (4 - len(firsts[i:i + 3]))
        rec = _records(rng, 4, n_ms, first_lost)
        more = _records(rng, 4, 1024, [None] * 4)
        ts_more = 0.001 * (n_ms + np.arange(1024))
        for w in (20, 1000, 1024):
            for cuts in ([], [1024, 4096]):
                bounds = [0] + [c for c in cuts if c < n_ms] + [n_ms]
                trk = _native.Tracker(engine, [0, 1, 2, 3], [0.0] * 4, [0.0] * 4, [0] * 4)
                emus = [SignalEmulator(w, N) for _ in range(4)]
                got = [[] for _ in range(4)]
                for a, b in zip(bounds[:-1], bounds[1:]):
                    d = _device(rec[:, a:b])
                    out = trk.signal_windows(b - a, ts[a:b], w, records_device_ptr=d.data_ptr())
                    torch.cuda.synchronize()
                    for c in range(4):
                        assert_windows_match(out[c], emus[c].run(rec[c, a:b], ts[a:b]), (first_lost, w, cuts, a, c))
                        got[c].append(out[c])
                for c, k in enumerate(first_lost):
                    win = np.concatenate(got[c])
                    if k is None:
                        assert len(win) == n_ms // w, (w, c)
                    else:
                        assert len(win) == k // w + (1 if k % w else 0), (first_lost, w, cuts, c)
                        assert win[-1]["first_ms"] + win[-1]["n_ms"] == k, (first_lost, w, cuts, c)
                d = _device(more)
                out = trk.signal_windows(1024, ts_more, w, records_device_ptr=d.data_ptr())
                torch.cuda.synchronize()
                for c, k in enumerate(first_lost):
                    assert_windows_match(out[c], emus[c].run(more[c], ts_more), (first_lost, w, cuts, "more", c))
                    assert (len(out[c]) == 0) == (k is not None), (first_lost, w, cuts, c)
                trk.close()
                n_checked += 1
    print(f"n_ms {n_ms}: first lost records {firsts}, {n_checked} runs")


# ---- k_parse_subframes in chain mode: the drop millisecond by a 32-lane ballot


@pytest.mark.parametrize("p", [0, 1, 31, 32, 33])
def test_chain_drop_scan(native_lib, p):
    """The recorded noise channel loses lock at ms 6000.  Tracked through TrackerBank in two calls split at 6000 - p,
    each followed by integrate_bits -> decode_subframes -> parse_subframes: the first call drops nothing and counts
    every millisecond; the second counts up to in-call index p and is dropped (prn_count -1) from p on."""
    from gypsum_b200.antenna_sample_provider import SampleProviderAttributes
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import TrackerBank

    z, ch, x, n, fs, tt = load_tracker_case("noise")
    init = z["init"]
    lost_at, n_ms = int(z["lost_at"]), int(z["n_ms"])
    sv = GpsSatelliteId(ch[0])
    bank = TrackerBank([(GpsSatellite(sv, generate_replica_prn_signals()[sv], n // 1023), init[0], init[1], int(init[2]))],
                       SampleProviderAttributes(fs, n))
    cut = lost_at - p
    recs, counts = [], []
    for a, b in ((0, cut), (cut, n_ms)):
        recs.append(bank.process(x[a * n:b * n], tt[a:b, 0])[0])
        bank.integrate_bits(tt[a:b, 0], tt[a:b, 1])
        bank.decode_subframes()
        bank.parse_subframes()
        counts.append(bank.observations()["prn_count"][0])
    bank.native.close()
    assert not recs[0]["lost"].any() and (counts[0] > 0).all()
    assert int(np.flatnonzero(recs[1]["lost"])[0]) == p
    assert (counts[1][:p] > 0).all() and (counts[1][p:] == -1).all(), (p, counts[1][max(p - 2, 0):p + 3])
