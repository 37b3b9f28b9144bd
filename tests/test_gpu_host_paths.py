"""The host-to-host paths against the float64 oracle at every branch (shapes and rules in host_paths_support): the
graph-replayed gb200_acquire_grid_host (eager, captured, replayed, eager_src, direct and to-caller records, the plain path),
what may change between a capture and a replay, the pipelined grid stream (every slot reused with its staging flipped,
interleaved calls, batches over the scratch budget and in L2 windows, closing with batches in flight, opening without an
IQ binding) and the device ring (wrapping and full-capacity appends from pageable and pinned sources, every window).

Every record goes through acq_support.check_grid against vector_grid on that call's own samples; where a synchronous path
exists the records must also equal upload_iq + acquire_grid byte for byte.  A pinned source is never rewritten before a
call that synchronises (include/gypsum_b200.h)."""
import numpy as np
import pytest

from acq_support import check_cells, check_grid, check_search, oracle_searches, rate, vector_cells, vector_grid
from gpu_support import EngineCache, all_chips, make_engine, run_child
from host_paths_support import (BUDGET_D, BUDGET_MB, CO, HOST_CASES, NC, RING_APPENDS, RING_CAPACITY, STREAM_CASES,
                                host_branch, records_to_caller, stream_pinning)
from oracle import gypsum_oracle as o

pytestmark = pytest.mark.gpu
PRNS = [24, 0, 6, 31, 13, 2, 19, 9]


@pytest.fixture(scope="module")
def engines(native_lib):
    cache = EngineCache()
    yield cache
    cache.close()


def native_kind(kind):
    from gypsum_b200 import _native

    return _native.COHERENT if kind == CO else _native.NON_COHERENT


def samples(seed, s, n_ms):
    """n_ms milliseconds of unit noise with SV 25 at 1500 Hz and SV 1 at -2500 Hz, code phases that move with the seed."""
    n, fs = rate(s)
    return o.synth_iq(seed, n, n_ms, fs, [(25, 1500.0, (97 * seed) % n, 0.3, 0.3), (1, -2500.0, (n - 1 - seed) % n, 1.1, 0.3)])


def axes(p, d):
    """(p replica rows, d Doppler bins): rows from PRNS, or all 32 in a shuffled order past eight."""
    rows = PRNS[:p] if p <= len(PRNS) else [(7 * i) % 32 for i in range(p)]
    return np.array(rows, np.int32), np.linspace(-5000.0, 5000.0, d)


def pinned_iq(x):
    """(pinned tensor, complex64 view of it) holding x."""
    import torch

    t = torch.from_numpy(np.ascontiguousarray(x, np.complex64).view(np.float32).copy()).pin_memory()
    return t, t.numpy().view(np.complex64)


def records(shape, pinned):
    """(keep-alive, RECORD_DTYPE array of shape), in pinned memory or not, every byte 0xFF."""
    import torch

    from gypsum_b200 import _native

    if pinned:
        t = torch.empty(int(np.prod(shape)) * 32, dtype=torch.uint8).pin_memory()
        out = t.numpy().view(_native.RECORD_DTYPE).reshape(shape)
    else:
        t, out = None, np.empty(shape, _native.RECORD_DTYPE)
    fill(out)
    return t, out


def fill(out):
    out.reshape(-1).view(np.uint8).fill(0xFF)


def check_blocks(rec, x, s, m, prn, dop, kind, what, svs=None):
    """Every block of a grid's records against vector_grid on that block's samples."""
    n, fs = rate(s)
    svs = [int(p) + 1 for p in prn] if svs is None else svs
    ok = o.COHERENT if kind == CO else o.NON_COHERENT
    for b in range(rec.shape[0]):
        xb = x[b * m * n:(b + 1) * m * n]
        check_grid(rec[b], xb, fs, n, svs, dop, (what, b), ok, ref=vector_grid(xb, fs, n, svs, dop, ok)[:4])


def check_host_call(eng, src, x, s, nb, m, prn, dop, kind, out, what, svs=None):
    """One acquire_grid_host call: its records land in out, match the oracle, and equal acquire_grid of the same shape
    on the engine's binding afterwards -- which holds that call's samples."""
    fill(out)
    got = eng.acquire_grid_host(src, nb, m, prn, dop, native_kind(kind), out=out)
    assert got is out, what
    check_blocks(out, x, s, m, prn, dop, kind, what, svs)
    assert eng.acquire_grid(nb, m, prn, dop, native_kind(kind)).tobytes() == out.tobytes(), what
    eng.upload_iq(x)
    assert eng.acquire_grid(nb, m, prn, dop, native_kind(kind)).tobytes() == out.tobytes(), what


# ---- 1. the host call's branch matrix --------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", HOST_CASES, ids=[c[0] for c in HOST_CASES])
def test_host_call_branches(engines, case):
    """Four calls of the shape -- eager, captured, replayed, and replayed again on new samples (a pinned input rewritten in
    place after the previous call returned) -- or four eager_src calls; records to a pinned or pageable buffer, directly
    or copied."""
    name, s, nb, m, kind, p, d, pin_in, pin_out = case
    n, _ = rate(s)
    eng = engines(n)
    prn, dop = axes(p, d)
    keep_out, out = records((nb, p, d), pin_out)
    keep_in, buf = pinned_iq(np.zeros(nb * m * n, np.complex64)) if pin_in else (None, None)
    for call in range(4):
        x = samples(10 * call + s, s, nb * m)
        if pin_in:
            buf[:] = x
        check_host_call(eng, buf if pin_in else x, x, s, nb, m, prn, dop, kind, out,
                        (name, call, host_branch(s, nb, m, d, pin_in, call), records_to_caller(nb, p, d, pin_out)))


def test_alternating_pinned_outs(engines):
    """One shape, two pinned record buffers passed in turn: each call's records land in the buffer it passed (the kernel
    stores them there directly) and the other buffer keeps what it held."""
    s, nb, m, p, d = 2, 1, 1, 3, 5
    assert records_to_caller(nb, p, d, True)
    eng = engines(rate(s)[0])
    prn, dop = axes(p, d)
    bufs = [records((nb, p, d), True) for _ in range(2)]
    for call in range(6):
        out, other = bufs[call % 2][1], bufs[1 - call % 2][1]
        before = other.tobytes()
        x = samples(50 + call, s, nb * m)
        check_host_call(eng, x, x, s, nb, m, prn, dop, NC, out, ("alternate", call))
        assert other.tobytes() == before, call


# ---- 2. what may change between a capture and a replay ---------------------------------------------------------------------
CHANGES = ["doppler_in_place", "prn_in_place", "d_grow_shrink", "replicas_permuted", "replicas_larger", "cells_fused",
           "cells_split", "detect", "weak_grid", "larger_grid", "grid_stream", "kernel_timing", "set_stream"]


@pytest.mark.parametrize("change", CHANGES)
def test_change_between_capture_and_replay(native_lib, change):
    """A shape eager, captured and replayed (S = 2, two blocks of 2 ms, records to a pageable buffer through the address
    cache), then one change, then three more host calls on new samples, each against the oracle with the axes and
    replicas as they are now."""
    import torch

    from gypsum_b200 import _native

    s, nb, m, p, d = 2, 2, 2, 3, 5
    n, fs = rate(s)
    eng = make_engine(fs, n)
    try:
        prn, dop = axes(p, d)
        _, out = records((nb, p, d), False)
        svs = None
        seed = iter(range(200, 300))
        for call in range(3):
            x = samples(next(seed), s, nb * m)
            check_host_call(eng, x, x, s, nb, m, prn, dop, NC, out, (change, "before", call))
        bound = x  # the engine's binding holds the last call's samples
        if change == "doppler_in_place":
            dop += 250.0  # the same array object: the address cache hands C the same pointer with new values
        elif change == "prn_in_place":
            prn[1] = 17
        elif change == "d_grow_shrink":
            dop2 = np.append(dop, 3125.0)
            _, out2 = records((nb, p, d + 1), False)
            x = samples(next(seed), s, nb * m)
            check_host_call(eng, x, x, s, nb, m, prn, dop2, NC, out2, (change, "grown"))
        elif change in ("replicas_permuted", "replicas_larger"):
            perm = np.random.default_rng(3).permutation(32) if change == "replicas_permuted" else np.arange(32)
            chips = all_chips()[perm]
            if change == "replicas_larger":
                chips = np.concatenate([chips, all_chips()[:8]])
            eng.set_replicas(chips)
            svs = [int(perm[i]) + 1 for i in prn]
        elif change in ("cells_fused", "cells_split"):
            cp, cd = (np.array([3, 24, 7, 0]), np.array([1500.0, 1500.0, -2500.0, 333.0])) if change == "cells_fused" \
                else (np.array([24, 0]), np.array([1500.0, -2500.0]))
            eng.set_fused(change == "cells_fused")
            try:
                got = eng.acquire_cells(cp, cd, m)
            finally:
                eng.set_fused(None)
            ref = vector_cells(bound[:m * n], fs, n, [int(c) + 1 for c in cp], cd)
            check_cells(got, ref, bound[:m * n], fs, n, [int(c) + 1 for c in cp], cd, change)
        elif change == "detect":
            got = eng.detect([24, 0], m)
            for (ref, amb), g, sv in zip(oracle_searches([25, 1], bound[:m * n], fs, n), got, [25, 1]):
                check_search((g["doppler"], g["code_phase"], g["strength"], float(np.angle(complex(g["probe_re"], g["probe_im"])))),
                             sv, (ref.doppler, ref.code_phase, ref.strength, ref.carrier_phase), amb, bound[:m * n], fs, n,
                             (change, sv))
        elif change == "weak_grid":
            # B * D = 10 folded Doppler slots, other values than the grid's, in the grid's axis buffers
            rec = eng.acquire_grid_weak(1, 3, 2, 2, prn, dop + 125.0)
            assert rec.shape == (1, p, 2, d)
        elif change == "larger_grid":
            y = samples(next(seed), s, 4 * m)
            eng.upload_iq(y)
            big_prn, big_dop = axes(6, 41)
            rec = eng.acquire_grid(4, m, big_prn, big_dop)
            check_blocks(rec, y, s, m, big_prn, big_dop, NC, change)
        elif change == "grid_stream":
            sp, sd = axes(4, 7)
            y = samples(next(seed), s, 1)
            gs = _native.GridStream(eng, 1, 1, sp, sd, _native.NON_COHERENT, depth=2)
            gs.submit(y)
            check_blocks(gs.collect(), y, s, 1, sp, sd, NC, change)
            gs.close()
        elif change == "kernel_timing":
            eng.enable_kernel_timing(True)
            assert host_branch(s, nb, m, d, False, 3, timing=True) == "plain"
            x = samples(next(seed), s, nb * m)
            check_host_call(eng, x, x, s, nb, m, prn, dop, NC, out, (change, "timed"))
            assert eng.kernel_timing(1)[1] >= 1
            eng.enable_kernel_timing(False)
        elif change == "set_stream":
            torch_stream = torch.cuda.Stream()
            eng.set_stream(torch_stream.cuda_stream)
            for call in range(3):
                x = samples(next(seed), s, nb * m)
                check_host_call(eng, x, x, s, nb, m, prn, dop, NC, out, (change, "torch stream", call))
            eng.set_stream(0)
        for call in range(3):
            x = samples(next(seed), s, nb * m)
            check_host_call(eng, x, x, s, nb, m, prn, dop, NC, out, (change, "after", call), svs)
    finally:
        eng.close()


# ---- 3. the plain path under a 1 MB budget (child process) ------------------------------------------------------------------
_BUDGET_CHILD = r"""
import os, sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
os.environ["GB200_SPEC_BUDGET_MB"] = sys.argv[2]
from gpu_support import make_engine
from test_gpu_host_paths import samples, axes
from gypsum_b200 import _native
n = 2046
e = make_engine(1000 * n, n)
res = {}
for d in (int(v) for v in sys.argv[3].split(",")):
    prn, dop = axes(3, d)
    for call in range(3):
        x = samples(300 + 10 * d + call, 2, 1)
        rec = e.acquire_grid_host(x, 1, 1, prn, dop, _native.NON_COHERENT)
        assert e.acquire_grid(1, 1, prn, dop, _native.NON_COHERENT).tobytes() == rec.tobytes()
        e.upload_iq(x)
        assert e.acquire_grid(1, 1, prn, dop, _native.NON_COHERENT).tobytes() == rec.tobytes()
        res[f"host_{d}_{call}"] = rec
# a stream whose every submit runs several scratch batches (13 blocks of 5 bins: 6, 6 and 1 under 1 MB)
prn, dop = axes(3, 5)
gs = _native.GridStream(e, 13, 1, prn, dop, _native.NON_COHERENT, depth=2)
for k in range(3):
    gs.submit(samples(400 + k, 2, 13))
    if gs.in_flight == 2:
        res[f"stream_{k - 1}"] = gs.collect().copy()
res["stream_2"] = gs.collect().copy()
gs.close()
for k in range(3):
    e.upload_iq(samples(400 + k, 2, 13))
    assert e.acquire_grid(13, 1, prn, dop, _native.NON_COHERENT).tobytes() == res[f"stream_{k}"].tobytes()
np.savez(sys.argv[4], **res)
e.close()
print("budget ok")
"""


def test_budget_fallback(native_lib, tmp_path):
    """GB200_SPEC_BUDGET_MB = 1, S = 2, M = 1: D = 32 fills the budget exactly (graph path), D = 33 is one bin past it
    (plain path); three host calls each, against the oracle and the synchronous path.  A grid stream of 13 blocks then
    runs three scratch batches per submit."""
    assert [host_branch(2, 1, 1, d, False, 2, BUDGET_MB) for d in BUDGET_D] == ["replay", "plain"]
    run_child(_BUDGET_CHILD, BUDGET_MB, ",".join(map(str, BUDGET_D)), tmp_path / "rec.npz", ok="budget ok")
    z = np.load(tmp_path / "rec.npz")
    for d in BUDGET_D:
        prn, dop = axes(3, d)
        for call in range(3):
            check_blocks(z[f"host_{d}_{call}"], samples(300 + 10 * d + call, 2, 1), 2, 1, prn, dop, NC, ("budget", d, call))
    prn, dop = axes(3, 5)
    for k in range(3):
        check_blocks(z[f"stream_{k}"], samples(400 + k, 2, 13), 2, 1, prn, dop, NC, ("budget stream", k))


# ---- 4. the grid stream -----------------------------------------------------------------------------------------------------
def run_stream(eng, case, seed):
    """stream_batches, then every batch against upload_iq + acquire_grid byte for byte."""
    xs, got = stream_batches(eng, case, seed)
    depth, s, nb, m, kind, p, d = case
    prn, dop = axes(p, d)
    for k, x in enumerate(xs):
        eng.upload_iq(x)
        assert eng.acquire_grid(nb, m, prn, dop, native_kind(kind)).tobytes() == got[k].tobytes(), (case, k)


def stream_batches(eng, case, seed):
    """2 * depth + 1 batches through a stream of the case's shape, inputs and outputs pinned per stream_pinning, the stream
    closed; each batch checked against the oracle.  Returns (samples, records) per batch."""
    from gypsum_b200 import _native

    depth, s, nb, m, kind, p, d = case
    prn, dop = axes(p, d)
    pins = stream_pinning(depth)
    xs = [samples(seed + k, s, nb * m) for k in range(len(pins))]
    keep, outs, got = [], [], []
    gs = _native.GridStream(eng, nb, m, prn, dop, native_kind(kind), depth=depth)
    for k, (pi, po) in enumerate(pins):
        if gs.in_flight == depth:
            got.append(gs.collect())
        t_in, src = pinned_iq(xs[k]) if pi else (None, xs[k])
        t_out, out = records((nb, p, d), po)
        keep += [t_in, t_out]
        outs.append(out)
        gs.submit(src, out)
    while gs.in_flight:
        got.append(gs.collect())
    gs.close()
    for k, x in enumerate(xs):
        assert got[k] is outs[k], k
        check_blocks(got[k], x, s, m, prn, dop, kind, (case, k, pins[k]))
    return xs, got


@pytest.mark.parametrize("case", STREAM_CASES, ids=[f"d{c[0]}_s{c[1]}_{c[4]}_m{c[3]}" for c in STREAM_CASES])
def test_grid_stream_slots(engines, case):
    run_stream(engines(rate(case[1])[0]), case, 500)


def test_grid_stream_interleaved_calls(engines):
    """Between each submit and its collect, one of: acquire_grid on uploaded samples, acquire_cells, detect,
    acquire_grid_host.  Every interleaved result and every collected batch against the oracle."""
    from gypsum_b200 import _native

    s, nb, m, p, d, depth = 2, 2, 1, 3, 5, 3
    n, fs = rate(s)
    eng = engines(n)
    prn, dop = axes(p, d)
    gs = _native.GridStream(eng, nb, m, prn, dop, _native.NON_COHERENT, depth=depth)
    xs = [samples(600 + k, s, nb * m) for k in range(8)]
    got = []
    for k, x in enumerate(xs):
        if gs.in_flight == depth:
            got.append(gs.collect())
        gs.submit(x)
        y = samples(700 + k, s, 3)
        what = ("interleaved", k)
        if k % 4 == 0:
            eng.upload_iq(y)
            gp, gd = axes(4, 7)
            check_blocks(eng.acquire_grid(1, 3, gp, gd), y, s, 3, gp, gd, NC, what)
        elif k % 4 == 1:
            eng.upload_iq(y)
            cp, cd = np.array([24, 0, 5, 24]), np.array([1500.0, -2500.0, 750.0, 1000.0])
            svs = [int(c) + 1 for c in cp]
            check_cells(eng.acquire_cells(cp, cd, 3), vector_cells(y, fs, n, svs, cd), y, fs, n, svs, cd, what)
        elif k % 4 == 2:
            eng.upload_iq(y)
            g = eng.detect([24], 3)[0]
            (ref, amb), = oracle_searches([25], y, fs, n)
            check_search((g["doppler"], g["code_phase"], g["strength"], float(np.angle(complex(g["probe_re"], g["probe_im"])))),
                         25, (ref.doppler, ref.code_phase, ref.strength, ref.carrier_phase), amb, y, fs, n, what)
        else:
            hp, hd = axes(2, 4)
            _, out = records((1, 2, 4), False)
            check_host_call(eng, y, y, s, 1, 3, hp, hd, NC, out, what)
    while gs.in_flight:
        got.append(gs.collect())
    gs.close()
    for k, x in enumerate(xs):
        check_blocks(got[k], x, s, m, prn, dop, NC, ("stream", k))


_WINDOW_CHILD = r"""
import os, sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
os.environ.update(GB200_L2_WINDOW_MB="1", GB200_L2_WINDOW_MIN_GROUPS="0")
from gpu_support import make_engine
from test_gpu_host_paths import axes, pinned_iq, records, samples
from gypsum_b200 import _native
n = 2046
e = make_engine(1000 * n, n)
prn, dop = axes(5, 41)
gs = _native.GridStream(e, 2, 1, prn, dop, _native.NON_COHERENT, depth=2)
keep, res = [], {}
for k in range(4):
    t_in, src = pinned_iq(samples(800 + k, 2, 2)) if k % 2 else (None, samples(800 + k, 2, 2))
    t_out, out = records((2, 5, 41), k % 3 == 0)
    keep += [t_in, t_out]
    if gs.in_flight == 2:
        res[f"b{k - 2}"] = gs.collect().copy()
    gs.submit(src, out)
res["b2"] = gs.collect().copy()
res["b3"] = gs.collect().copy()
gs.close()
for k in range(4):
    e.upload_iq(samples(800 + k, 2, 2))
    assert e.acquire_grid(2, 1, prn, dop, _native.NON_COHERENT).tobytes() == res[f"b{k}"].tobytes()
np.savez(sys.argv[2], **res)
e.close()
print("windows ok")
"""


def test_grid_stream_l2_windows(native_lib, tmp_path):
    """GB200_L2_WINDOW_MB = 1 in a child process: each 2-block batch of 41 bins (2.7 MB of spectra) is walked in L2
    windows; every batch against the oracle and the synchronous path."""
    run_child(_WINDOW_CHILD, tmp_path / "rec.npz", ok="windows ok")
    z = np.load(tmp_path / "rec.npz")
    prn, dop = axes(5, 41)
    for k in range(4):
        check_blocks(z[f"b{k}"], samples(800 + k, 2, 2), 2, 1, prn, dop, NC, ("windows", k))


def test_grid_stream_close_in_flight(engines):
    """Closing a stream with every slot in flight waits for the batches: the records sent to pinned buffers are there.
    The engine then works as before, and another stream opens at once, with no IQ bound."""
    from gypsum_b200 import _native

    s, nb, m, p, d, depth = 5, 1, 2, 3, 4, 3
    n, fs = rate(s)
    eng = engines(n)
    prn, dop = axes(p, d)
    eng.upload_iq(samples(899, s, 1))
    gs = _native.GridStream(eng, nb, m, prn, dop, _native.COHERENT, depth=depth)
    xs = [samples(900 + k, s, nb * m) for k in range(depth)]
    outs = [records((nb, p, d), k != 1) for k in range(depth)]
    for x, (_, out) in zip(xs, outs):
        gs.submit(x, out)
    gs.close()
    for k in (0, 2):
        check_blocks(outs[k][1], xs[k], s, m, prn, dop, CO, ("closed", k))
    with pytest.raises(RuntimeError, match="no IQ loaded"):
        eng.acquire_grid(nb, m, prn, dop, _native.COHERENT)
    stream_batches(eng, (2, s, nb, m, CO, p, d), 950)
    y = samples(990, s, 2)
    eng.upload_iq(y)
    check_blocks(eng.acquire_grid(1, 2, prn, dop), y, s, 2, prn, dop, NC, "after close")


def test_grid_stream_opens_on_fresh_engine(native_lib):
    """A stream brings its own IQ: it opens on an engine that has never had any bound."""
    n, fs = rate(1)
    eng = make_engine(fs, n)
    try:
        run_stream(eng, (2, 1, 2, 1, NC, 3, 4), 1000)
    finally:
        eng.close()


def test_grid_stream_opens_after_another_closes(engines):
    """Closing a stream takes its slot buffers, and with them the engine's IQ binding; a second stream opens right after."""
    from gypsum_b200 import _native

    eng = engines(rate(2)[0])
    eng.upload_iq(samples(1100, 2, 2))
    stream_batches(eng, (1, 2, 1, 1, NC, 3, 4), 1110)
    with pytest.raises(RuntimeError, match="no IQ loaded"):
        eng.acquire_grid(1, 1, [0], [0.0], _native.NON_COHERENT)
    run_stream(eng, (3, 2, 2, 2, CO, 2, 3), 1120)


# ---- 5. the device ring -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", [2, 5])
def test_ring_appends_and_windows(engines, s):
    """Capacity 7, appends of 1, 7, 3, 6, 3, 7 and 1 ms (full-capacity appends at slots 1 and 6, two of them wrapping),
    alternately from pageable and pinned memory.  After each, every window bind_newest(k) can give: the grid on it equals
    the upload path byte for byte, and the full window is checked against the oracle.  The refusals leave the next grid
    as it was."""
    from gypsum_b200 import _native

    n, fs = rate(s)
    eng = engines(n)
    prn, dop = axes(3, 5)
    ring = _native.Ring(eng, RING_CAPACITY)
    try:
        with pytest.raises(ValueError):
            ring.bind_newest(1)  # nothing appended yet
        stream = samples(1200 + s, s, sum(RING_APPENDS))
        appended, keep = 0, []
        for i, n_ms in enumerate(RING_APPENDS):
            chunk = stream[appended * n:(appended + n_ms) * n]
            if i % 2:
                t, v = pinned_iq(chunk)
                keep.append(t)
                ring.append(v)
            else:
                ring.append(chunk.copy())
            appended += n_ms
            assert ring.appended_ms == appended
            top = min(appended, RING_CAPACITY)
            for k in range(1, top + 1):
                ring.bind_newest(k)
                got = eng.acquire_grid(k, 1, prn, dop)
                coh = eng.acquire_grid(1, k, prn, dop, _native.COHERENT) if k == top else None
                win = stream[(appended - k) * n:appended * n]
                eng.upload_iq(win)
                assert eng.acquire_grid(k, 1, prn, dop).tobytes() == got.tobytes(), (s, i, k)
                if k == top:
                    assert eng.acquire_grid(1, k, prn, dop, _native.COHERENT).tobytes() == coh.tobytes(), (s, i, k)
                    check_blocks(got, win, s, 1, prn, dop, NC, ("ring", s, i, k))
                    check_blocks(coh, win, s, k, prn, dop, CO, ("ring coherent", s, i, k))
        ring.bind_newest(RING_CAPACITY)
        want = eng.acquire_grid(RING_CAPACITY, 1, prn, dop)
        with pytest.raises(ValueError):
            ring.append(samples(1300, s, RING_CAPACITY + 1))  # more than the ring holds
        with pytest.raises(ValueError):
            ring.bind_newest(RING_CAPACITY + 1)
        assert ring.appended_ms == appended
        assert eng.acquire_grid(RING_CAPACITY, 1, prn, dop).tobytes() == want.tobytes()
    finally:
        ring.close()
    fresh = _native.Ring(eng, RING_CAPACITY)
    try:
        fresh.append(stream[:n])
        fresh.bind_newest(1)
        want = eng.acquire_grid(1, 1, prn, dop)
        with pytest.raises(ValueError):
            fresh.bind_newest(2)  # past what was appended
        assert eng.acquire_grid(1, 1, prn, dop).tobytes() == want.tobytes()
        check_blocks(want, stream[:n], s, 1, prn, dop, NC, ("fresh ring", s))
    finally:
        fresh.close()
