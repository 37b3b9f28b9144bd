"""k_signal_windows (signal.cu) at every batch, carry, stop, grid and output edge, on seeded synthetic tracking records
through records_device_ptr, 4 channels per call.  The plans are tests/test_signal_edges_cpu.py's, which shows on the
CPU that each reaches its edge: W = 20, 21, 27, 1000, 1024 and 60 000; calls of 1 to 9, W - 1, W and W + 1 ms that
carry every open.n into a call (every one for W <= 27, else 0 to 8 and W - 8 to W - 1), so window 0's length takes
every value mod 8; a call of more than 128 windows (the second blockIdx.y); calls crossing a 60 000-ms window; stops at
offsets 0 to 8 of a window's first batch, at start == stop of a window j > 0, at end - 1, at end, at a call's last ms
and at ms 0 of a call with an open window, and nothing from a stopped channel afterwards; max_windows equal to the
emitted count, and one below.  Every call's windows against the host build of signal_core.cuh (exact, C/N0 within
1e-12 relative); one call and the split byte-identical apart from ms_index; a subset against the float64 oracle."""
import numpy as np
import pytest

import signal_support as ss
from gpu_support import make_engine
from test_signal_edges_cpu import W_SIZES, carry_sizes, emulate, records, stop_edge, stop_runs

pytestmark = pytest.mark.gpu
N, FS = 2046, 2046000


@pytest.fixture(scope="module")
def engine(native_lib):
    e = make_engine(FS, N)
    yield e
    e.close()


def _device(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def _run(engine, rec, ts, w, bounds, max_windows=None):
    """The records in calls [bounds[i], bounds[i + 1]) on one tracker: per channel the windows of each call."""
    import torch

    from gypsum_b200 import _native

    n_ch = rec.shape[0]
    trk = _native.Tracker(engine, list(range(n_ch)), [0.0] * n_ch, [0.0] * n_ch, [0] * n_ch)
    got = [[] for _ in range(n_ch)]
    for a, b in zip(bounds[:-1], bounds[1:]):
        d = _device(rec[:, a:b])
        out = trk.signal_windows(b - a, ts[a:b], w, records_device_ptr=d.data_ptr(), max_windows=max_windows)
        torch.cuda.synchronize()
        for c in range(n_ch):
            got[c].append(out[c])
    trk.close()
    return got


def _check(got, want, what):
    for c, (g, w) in enumerate(zip(got, want)):
        for i, (gi, wi) in enumerate(zip(g, w)):
            ss.assert_windows_match(gi, wi, (what, c, i))


@pytest.mark.parametrize("w", W_SIZES)
def test_carried_window_and_call_sizes(engine, w):
    """The carry sizes' calls: every call == the host build, the split == one call byte for byte apart from
    ms_index, and window 0 of every call ends where r = W - open.n says."""
    sizes = carry_sizes(w)
    total = sum(sizes)
    bounds = [int(b) for b in np.cumsum([0] + sizes)]
    rec = records(11 * w, 4, total, [None] * 4)
    ts = 0.001 * np.arange(total) + 100.0
    got = _run(engine, rec, ts, w, bounds)
    _check(got, emulate(rec, ts, w, bounds), w)
    one = _run(engine, rec, ts, w, [0, total])
    for c in range(4):
        split = np.concatenate(got[c])
        assert len(split) == total // w and ss.without_ms_index(split) == ss.without_ms_index(one[c][0]), (w, c)
    for a, out in zip(bounds[:-1], got[0]):
        r = w - a % w
        if len(out):
            assert out[0]["ms_index"] == r - 1 and out[0]["first_ms"] == a + r - w  # window 0 closes after r records
    most = max(len(o) for o in got[0])
    print(f"W {w}: {len(sizes)} calls, {total} ms, at most {most} windows in one call")
    if w <= 27:
        assert most > 128


@pytest.mark.parametrize("w", W_SIZES)
def test_stops(engine, w):
    """Every stop placement: the call holding it emits stop_edge's count, the last window ends at the stop, nothing
    follows (a further call included); the same records in one call give the same windows; every call == the host
    build."""
    cuts, n_ms, runs = stop_runs(w)
    bounds = [0] + cuts + [n_ms]
    ts = 0.001 * np.arange(n_ms + 2 * w + 3)
    for i, run in enumerate(runs):
        rec = records(1000 * w + i, 4, n_ms + 2 * w + 3, run)
        b = bounds + [n_ms + 2 * w + 3]  # a further call of 2 W + 3 ms
        got = _run(engine, rec, ts, w, b)
        _check(got, emulate(rec, ts, w, b), (w, run))
        one = _run(engine, rec, ts, w, [0, len(ts)])
        for c, k in enumerate(run):
            assert ss.without_ms_index(np.concatenate(got[c])) == ss.without_ms_index(one[c][0]), (w, k)
            if k is None:
                continue
            a, s, j, off, r, emitted = stop_edge(k, w, cuts)
            ci = b.index(a)
            assert len(got[c][ci]) == emitted, (w, k, s, j, off)
            win = np.concatenate(got[c])
            assert win[-1]["first_ms"] + win[-1]["n_ms"] == k and all(len(x) == 0 for x in got[c][ci + 1:]), (w, k)
        if i == 0 and w in (20, 27, 1000):  # the float64 oracle over one call
            floor = ss.SignalEmulator(w, N).floor
            for c in range(4):
                ss.assert_windows_match(one[c][0], ss.oracle_windows(rec[c], ts, w, floor), (w, "oracle", c))
    print(f"W {w}: {sum(k is not None for r in runs for k in r)} stops in {len(runs)} runs")


@pytest.mark.parametrize("w", (20, 1024))
def test_output_limit(engine, w):
    """max_windows equal to the most windows a channel emits gives the same windows; one below raises."""
    n_ms = 5 * w + 3
    rec = records(3 * w, 4, n_ms, [None, 2 * w, 3 * w + 1, None])
    ts = 0.001 * np.arange(n_ms)
    full = _run(engine, rec, ts, w, [0, n_ms])
    most = max(len(o[0]) for o in full)
    exact = _run(engine, rec, ts, w, [0, n_ms], max_windows=most)
    for c in range(4):
        assert exact[c][0].tobytes() == full[c][0].tobytes()
    with pytest.raises(RuntimeError):
        _run(engine, rec, ts, w, [0, n_ms], max_windows=most - 1)
