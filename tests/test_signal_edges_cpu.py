"""The C/N0 window plans of tests/test_gpu_signal_edges.py on the CPU: the call sizes and stop placements that put
k_signal_windows (signal.cu) at its edges, shown to reach them through the host build of signal_core.cuh, which
equals the float64 oracle on them.

Window j of a call covers the call's milliseconds [start_j, end_j): window 0 continues the window the last call left
open with open.n records and ends after r = W - open.n of them, window j > 0 is [r + (j-1) W, r + j W).  A thread sums
its window in batches of 8 records with a scalar tail, so window 0's length mod 8 decides the tail; a stop (the first
lost record) at in-call index s cuts window j with start_j <= s."""
import numpy as np
import pytest

import signal_support as ss

W_SIZES = (20, 21, 27, 1000, 1024, 60000)
N = 2046


def carry_sizes(w):
    """Call sizes that carry every open.n from 0 to W - 1 into a call (W <= 27), or 0 to 8 and W - 8 to W - 1, so that
    window 0's length r takes every value mod 8 (r = 1 included); calls of 1 to 9, W - 1, W and W + 1 ms; and for
    W <= 27 a last call of more than 128 windows.  At W = 60 000, calls that cross windows."""
    if w == 60000:
        return [59999, 1, 7, 59990, 30000, 40000, 60001]
    sizes = list(range(1, 10)) + [w - 1, w, w + 1]
    want = set(range(w)) if w <= 27 else set(range(9)) | set(range(w - 8, w))
    while want - set(open_at(sizes, w)):
        o = sum(sizes) % w
        t = min(want - set(open_at(sizes, w)), key=lambda t: (t - o) % w or w)
        sizes.append((t - o) % w or w)
    if w <= 27:
        sizes.append(130 * w + 5)
    return sizes


def open_at(sizes, w):
    """open.n at the start of every call of these sizes (and one after them), with no stop."""
    return [int(s) % w for s in np.cumsum([0] + list(sizes))]


def stop_plan(w):
    """(cuts, n_ms, stops): a stream of 4 W + 7 ms cut at b1 = W + W/2 + 3 (so the call from b1 opens with a carried
    window) and b2 = 3 W + 5, and the first lost records placed at offsets 0 to 8 of window 2's first batch (offset 0:
    start == stop of window j = 1 of the call from b1), offsets 0 to 8 of the call from b1 (offset 0: a stop at ms 0 of
    a call with an open window), the last record of window 2 (end - 1), its end, and the last ms of the call to b2."""
    b1, b2 = w + w // 2 + 3, 3 * w + 5
    stops = sorted({2 * w + q for q in range(9)} | {b1 + q for q in range(9)} | {3 * w - 1, 3 * w, b2 - 1})
    return [b1, b2], 4 * w + 7, stops


def stop_edge(k, w, cuts):
    """Where a first lost record at stream ms k falls: (call start, in-call index s, window j, offset of s in window j,
    r, windows the call emits)."""
    a = max([0] + [c for c in cuts if c <= k])
    s, o = k - a, a % w
    r = w - o
    j = 0 if s < r else 1 + (s - r) // w
    start = 0 if j == 0 else r + (j - 1) * w
    held = s - start + (o if j == 0 else 0)  # records the cut window holds
    return a, s, j, s - start, r, j + (1 if held > 0 else 0)


def records(seed, n_ch, n_ms, first_lost):
    """Seeded TRACK_DTYPE records; channel c loses lock at first_lost[c] (None: never), `lost` 2 after it."""
    rng = np.random.default_rng(seed)
    rec = np.zeros((n_ch, n_ms), dtype=ss.track_dtype())
    rec["peak_re"] = rng.normal(0.0, 1.0, (n_ch, n_ms)) + 3.0
    rec["peak_im"] = rng.normal(0.0, 1.0, (n_ch, n_ms))
    rec["strength"] = rng.uniform(0.5, 10.0, (n_ch, n_ms))
    rec["locked"] = rng.integers(0, 2, (n_ch, n_ms))
    for c, k in enumerate(first_lost):
        if k is not None:
            rec["lost"][c, k] = 1
            rec["lost"][c, k + 1:] = 2
    return rec


def stop_runs(w):
    """The stops of stop_plan in runs of four channels (the last padded with channels that never stop)."""
    cuts, n_ms, stops = stop_plan(w)
    runs = [stops[i:i + 4] for i in range(0, len(stops), 4)]
    return cuts, n_ms, [r + [None] * (4 - len(r)) for r in runs]


def emulate(rec, ts, w, bounds):
    """Each channel's windows per call through the host build, calls [bounds[i], bounds[i + 1])."""
    out = []
    for c in range(rec.shape[0]):
        emu = ss.SignalEmulator(w, N)
        out.append([emu.run(rec[c, a:b], ts[a:b]) for a, b in zip(bounds[:-1], bounds[1:])])
    return out


@pytest.mark.parametrize("w", W_SIZES)
def test_carry_sizes_reach_every_open_count(w):
    sizes = carry_sizes(w)
    opens = open_at(sizes, w)[:-1]
    if w <= 27:
        assert set(opens) == set(range(w)) and max(sizes) // w > 128
    assert w - 1 in opens  # r = 1
    if w < 60000:
        assert {(w - o) % 8 for o in opens} == set(range(8))
        assert set(range(1, 10)) | {w - 1, w, w + 1} <= set(sizes)
    else:
        assert any(int(a) // w != int(a + s - 1) // w for a, s in zip(np.cumsum([0] + sizes), sizes))


@pytest.mark.parametrize("w", W_SIZES)
def test_stop_plan_reaches_every_edge(w):
    """Each placement is where its name says, and the host build emits the windows stop_edge counts, the last ending
    at the stop."""
    cuts, n_ms, runs = stop_runs(w)
    offs, zero_open, start_eq = set(), False, False
    for k in (k for run in runs for k in run if k is not None):
        a, s, j, off, r, emitted = stop_edge(k, w, cuts)
        if j > 0 or a == cuts[0]:
            offs.add((j > 0, off))
        zero_open |= s == 0 and a % w > 0
        start_eq |= j > 0 and off == 0 and emitted == j
    r0 = w - cuts[0] % w  # window 0's length in the call from b1
    assert {(True, q) for q in range(9)} | {(False, q) for q in range(min(9, r0))} <= offs and zero_open and start_eq
    if w > 60000 - 1:
        return  # the host build over 240 000 records per channel: run on the device's side only
    bounds = [0] + cuts + [n_ms]
    ts = 0.001 * np.arange(n_ms)
    for i, run in enumerate(runs):
        rec = records(1000 * w + i, 4, n_ms, run)
        got = emulate(rec, ts, w, bounds)
        for c, k in enumerate(run):
            if k is None:
                continue
            a, s, j, off, r, emitted = stop_edge(k, w, cuts)
            ci = bounds.index(a)
            assert len(got[c][ci]) == emitted, (w, k)
            win = np.concatenate(got[c])
            assert win[-1]["first_ms"] + win[-1]["n_ms"] == k and all(len(x) == 0 for x in got[c][ci + 1:])


@pytest.mark.parametrize("w", (20, 27, 1000))
def test_host_build_equals_oracle_on_the_plans(w):
    """The host build, one call and the carry sizes' calls, against the float64 oracle over the stop runs' records."""
    cuts, n_ms, runs = stop_runs(w)
    ts = 0.001 * np.arange(n_ms)
    rec = records(1000 * w, 4, n_ms, runs[0])
    floor = ss.SignalEmulator(w, N).floor
    for c in range(4):
        want = ss.oracle_windows(rec[c], ts, w, floor)
        ss.assert_windows_match(ss.SignalEmulator(w, N).run(rec[c], ts), want, (w, c))
    sizes = carry_sizes(w)
    total = sum(sizes)
    rec = records(7 * w, 1, total, [None])
    ts = 0.001 * np.arange(total)
    bounds = list(np.cumsum([0] + sizes))
    split = np.concatenate(emulate(rec, ts, w, bounds)[0])
    one = ss.SignalEmulator(w, N).run(rec[0], ts)
    assert ss.without_ms_index(split) == ss.without_ms_index(one)
    ss.assert_windows_match(one, ss.oracle_windows(rec[0], ts, w, floor), w)
