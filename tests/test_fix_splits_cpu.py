"""The position fix under any split of a timeline into calls, on the CPU.  tests/test_gpu_chain_edges.py cuts the recorded
timelines so that every decision of k_fix_plan falls on every edge of its 32-millisecond chunks and of a call, and checks
each call against one oracle run sliced to it.  That rests on what this file shows: resplit() moves events and drops to
the calls that hold them, the receiver oracle gives the same records byte for byte however the timeline is cut (and
OracleTimeline's slices are what it says of each call), the model of the device's passes stays within the bounds of
DESIGN.md §6 on every split, and the repair the device runs depends on the split."""
import os

import numpy as np
import pytest

import fix_lsq_oracle as lo
from fix_support import (FIXING, MANY_BIAS_S, MANY_POS_M, MANY_SLIDE_ULPS, BIAS_S, POS_M, SLIDE_ULPS, OracleTimeline,
                         call_starts, edge_ms, edge_splits, fix_emulator, resplit, scripted_timeline, sweep_cuts)
from oracle import fix_oracle as fx

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIMELINES = [("fix", n) for n in ("realistic", "three", "gate", "lost", "five", "raise")] + \
            [("fix_repair", n) for n in ("gap_mid", "gap_two", "gap_back", "gap_first", "gap_carry", "gap_five",
                                         "gap_raise", "singular")]
CASES = [(fx, g, n) for g, n in TIMELINES] + [(lo, None, "scripted"), (lo, "fix", "five")]


def timeline(group, name):
    if group is None:
        return scripted_timeline()
    return fx.golden_calls(np.load(os.path.join(ROOT, "tests", "golden", f"{group}.npz")), name)


@pytest.fixture(scope="module")
def fix_emu():
    return fix_emulator()


def _events(calls):
    """Per channel: [(kind, words, trailing edge, global ms)] and the global drops of each original call."""
    bounds, _ = call_starts(calls)
    n_ch = len(calls[0][1])
    ev = [[(k, w, te, b + m) for b, (_, chans) in zip(bounds, calls) for k, w, te, m in chans[ch][0]] for ch in range(n_ch)]
    drops = [[b + chans[ch][1] for b, (_, chans) in zip(bounds, calls) if chans[ch][1] >= 0] for ch in range(n_ch)]
    return ev, drops


@pytest.mark.parametrize("group,name", TIMELINES + [(None, "scripted")])
def test_resplit_moves_every_event_and_drop(group, name):
    calls = timeline(group, name)
    bounds, total = call_starts(calls)
    same = resplit(calls, [])
    assert len(same) == len(calls)
    for (a, ca), (b, cb) in zip(same, calls):
        assert np.array_equal(a, b) and ca == cb
    cuts = sorted(set(sweep_cuts(calls, 11)) | {1, total - 1, *(b + 1 for b in bounds), *(b - 1 for b in bounds[1:])})
    split = resplit(calls, cuts)
    starts, total2 = call_starts(split)
    assert total2 == total and starts == sorted(set(bounds) | {c for c in cuts if 0 < c < total})
    assert np.array_equal(np.concatenate([rx for rx, _ in split]), np.concatenate([rx for rx, _ in calls]))
    ev, drops = _events(calls)
    ev2, _ = _events(split)
    assert ev2 == ev  # every event once, in its channel's order, at its own millisecond
    for s, (rx, chans) in zip(starts, split):
        b = max(x for x in bounds if x <= s)  # the original call this piece belongs to
        e_orig = b + len(calls[bounds.index(b)][0])
        for ch, (events, d) in enumerate(chans):
            assert all(0 <= m < len(rx) for _, _, _, m in events)
            drop = [x for x in drops[ch] if b <= x < e_orig]
            if not drop or drop[0] >= s + len(rx):
                assert d == -1, (s, ch)
            else:
                assert d == max(drop[0] - s, 0), (s, ch)  # the piece holding the drop, or one after it: at 0


def _bounds_check(oracle, rec, d, many_from):
    """The model's records of one call against the oracle's within the §6 bounds (MANY_* from index many_from on)."""
    fixing = np.flatnonzero(np.isin(rec["status"], FIXING))
    assert sorted(d["out"]) == list(fixing)
    worst = 0.0
    for m in fixing:
        got, want = d["out"][m], rec[m]
        many = m >= many_from
        ulps, bias, pos = (MANY_SLIDE_ULPS, MANY_BIAS_S, MANY_POS_M) if many else (SLIDE_ULPS, BIAS_S, POS_M)
        assert got["status"] == want["status"], m
        for k in ("slide_in", "slide_out"):
            u = abs(got[k] - want[k]) / (2.0 ** -52 * abs(want[k]))
            assert u <= ulps, (m, k, u)
            worst = max(worst, u)
        if want["status"] == fx.FIX_SOLVED:
            assert np.abs(got["pseudorange"] - want["pseudorange"]).max() <= ulps * 2.0 ** -52 * abs(want["slide_in"])
            assert abs(got["clock_bias"] - want["clock_bias"]) <= bias, m
            assert max(abs(got[k] - want[k]) for k in "xyz") <= pos, m
    return worst


@pytest.mark.parametrize("oracle,group,name", CASES, ids=[f"{o.__name__.split('.')[-1]}-{n}" for o, _, n in CASES])
def test_oracle_is_split_invariant(fix_emu, oracle, group, name):
    """Two splits per timeline, a 33-ms sweep and the union of every edge placement: the oracle's records are the one
    run's byte for byte, OracleTimeline's slices are the oracle's resets, order and stop of every call, and the model
    of the device's passes on the oracle's rows is within the §6 bounds, its carried slide too."""
    calls = timeline(group, name)
    tl = OracleTimeline(oracle, calls)
    bounds, total = call_starts(calls)
    misses = [b + d["first_miss"] for b, d in zip(bounds, tl.model(fix_emu, calls)) if d["first_miss"] is not None]
    edges = edge_ms(calls, tl, misses)
    union = sorted({c for _, cuts, _ in edge_splits(calls, edges) for c in cuts})
    offset = (7 * len(name) + len(edges)) % 33
    five = np.flatnonzero((tl.records["n_ready"] > 4) & np.isin(tl.records["status"], FIXING))
    many_from = five[0] if oracle is lo and len(five) else total
    worst = 0.0
    for cuts in (sweep_cuts(calls, offset), union):
        split = resplit(calls, cuts)
        starts, _ = call_starts(split)
        rcv = oracle.ReceiverOracle(len(calls[0][1]))
        carried, recs = None, []
        for s, (rx, chans) in zip(starts, split):
            rec = rcv.call(chans, rx)
            want, resets, order, stopped = tl.call(s, s + len(rx))
            assert rec.tobytes() == want.tobytes(), s
            assert rcv.resets == resets and rcv.order == order and rcv.stopped == stopped, s
            d = oracle.device_passes(fix_emu, rec, rcv.rows, rcv.resets, carried)
            carried = d["slide"]
            worst = max(worst, _bounds_check(oracle, rec, d, many_from - s))
            recs.append(rec)
        assert np.concatenate(recs).tobytes() == tl.records.tobytes()
        if tl.slide is not None:
            ulps = MANY_SLIDE_ULPS if many_from < total else SLIDE_ULPS
            assert abs(carried - tl.slide) <= ulps * 2.0 ** -52 * abs(tl.slide)
        else:
            assert carried is None
    print(f"{name}: {len(edges)} edges, sweep offset {offset}, {len(union)} edge cuts; model within {worst:.3g} ulp "
          f"of the oracle's slides")


def test_repair_depends_on_the_split(fix_emu):
    """gap_first in 33-ms calls: how many fixes the device's serial repair recomputes depends on where the calls are
    cut, so the re-split timelines drive k_fix_repair and the carried slide through states the recorded split does not."""
    calls = timeline("fix_repair", "gap_first")
    tl = OracleTimeline(fx, calls)
    counts = [sum(len(d["repaired"]) for d in tl.model(fix_emu, resplit(calls, sweep_cuts(calls, o))))
              for o in (0, 5, 17, 31)]
    print(f"gap_first in 33-ms calls at offsets 0, 5, 17, 31: repaired {counts}")
    assert len(set(counts)) >= 2, counts
