"""The streams tests/test_gpu_nav_edges.py feeds the device's preamble scan, shown to reach the scan states they are
built for: the host build of the decoder's state machine (tests/emu/nav_emu.cu, the scalar scan) traces, bit by bit,
the search nav_push chose and the queue it saw, and equals the oracle decoder on every stream, events and final state.
The trace also holds the decoder to the fact the device scan's grid rests on: a full scan only ever sees 600 bits."""
import ctypes as C
import time

import numpy as np
import pytest

import nav_support as ns
from hostbuild import host_library
from oracle import nav_oracle as nav

NO_SCAN, FULL_SCAN, SKIP = 0, 1, 2  # nav_core.cuh NavPush
GRIDS = ["candidate_grid", "word_offset_grid", "wrap_grid", "decoy_grid", "incremental_grid", "raise_streams"]


@pytest.fixture(scope="module")
def nav_emu():
    lib = host_library("nav_emu")
    lib.nav_emu_trace.restype = C.c_int
    return lib


@pytest.fixture(scope="module")
def builder():
    return ns.StreamBuilder()


@pytest.fixture(scope="module")
def oracle():
    return ns.OracleRuns()


def emu_trace(lib, s: ns.Stream):
    """The host build over the whole stream: rows and words (as the oracle's), final state, trace [n, 4]."""
    from gypsum_b200._native import SUBFRAME_DTYPE, subframe_event_capacity

    n = s.bits.size
    st = (C.c_char * lib.nav_emu_state_size())()
    lib.nav_emu_init(st)
    bits = np.ascontiguousarray(s.bits, dtype=np.int32)
    t0, t1 = s.times
    cap = subframe_event_capacity(n)
    ev = np.zeros(cap, dtype=SUBFRAME_DTYPE)
    trace = np.zeros((n, 4), dtype=np.int32)
    m = lib.nav_emu_trace(st, n, bits.ctypes.data_as(C.c_void_p), t0.ctypes.data_as(C.c_void_p),
                          t1.ctypes.data_as(C.c_void_p), ev.ctypes.data_as(C.c_void_p), cap,
                          trace.ctypes.data_as(C.c_void_p))
    assert m <= cap
    ev = ev[:m]
    rows = np.array([[e["bit_index"], e["kind"], e["subframe_id"], e["tow"], e["phase"], e["polarity"], e["parity_ok"],
                      e["receiver_timestamp"], e["trailing_edge_receiver_timestamp"]] for e in ev],
                    dtype=np.float64).reshape(-1, 9)
    words = np.array([e["words"] for e in ev], dtype=np.int64).reshape(-1, 10)
    summary = np.zeros(6, dtype=np.int64)
    lib.nav_emu_summary(st, summary.ctypes.data_as(C.c_void_p))
    return rows, words, list(summary), trace


def check_stream(lib, oracle, s: ns.Stream):
    rows, words, final, tr = emu_trace(lib, s)
    what = (s.name, s.qhead, s.c, s.pol)
    full = tr[:, 0] == FULL_SCAN
    assert (tr[full, 2] == ns.WINDOW).all(), what  # a larger full scan would need the device grid widened
    for start, _, _ in s.cycles:  # every cycle's pair comes from a full scan at the head the plan put it
        k = start + ns.WINDOW - 1
        assert list(tr[k, :3]) == [FULL_SCAN, start % ns.CAP, ns.WINDOW], (what, start)
    k = s.decide
    if s.c <= ns.LAST_FULL:
        assert list(tr[k, :3]) == [FULL_SCAN, s.qhead, ns.WINDOW], what
    else:  # the full scan at 600 found nothing; the append that completes the pair finds it
        first = k - (s.c + ns.SUB + 8) + ns.WINDOW
        assert list(tr[first, :3]) == [FULL_SCAN, s.qhead, ns.WINDOW] and tr[first, 3] == -1, what
        assert list(tr[k, :3]) == [NO_SCAN, s.qhead, s.c + ns.SUB + 8], what
    want_rows, want_words, want_final = oracle(s)
    assert np.array_equal(rows, want_rows) and np.array_equal(words, want_words), what
    assert final == want_final, what
    if s.name == "raise":
        assert want_rows[-1, 0] == k and want_rows[-1, 1] == nav.KIND_RAISED, what
    else:
        assert ns.first_phase(want_rows, k) == (k, s.c, s.pol), what
    return tr


@pytest.mark.parametrize("grid", GRIDS)
def test_streams_reach_their_scan_states(nav_emu, builder, oracle, grid):
    t0 = time.time()
    streams = getattr(ns, grid)(builder)
    states = set()
    for s in streams:
        check_stream(nav_emu, oracle, s)
        states.add((s.qhead, s.c, s.pol))
    if grid == "candidate_grid":
        assert states == {(q, c, p) for q in ns.QHEADS for c in range(ns.LAST_FULL + 2) for p in (1, -1)}
    if grid == "word_offset_grid":
        assert {q % 32 for q, _, _ in states} == set(range(32))
    if grid == "wrap_grid":  # the first preamble or the partner straddles the ring's end
        assert any(0 < ns.CAP - q - c < 8 for q, c, _ in states) and any(0 < ns.CAP - q - c - ns.SUB < 8 for q, c, _ in states)
    print(f"{grid}: {len(streams)} streams, {len(states)} scan states, {time.time() - t0:.1f} s")


def test_cycle_plan_reaches_every_ring_head():
    for q in range(ns.CAP):
        c1 = ns.cycle_plan(q)
        assert all(1 <= c <= ns.LAST_FULL for c in c1)
        assert (sum(c1) + ns.SUB * max(len(c1) - 1, 0) + ns.WINDOW * (len(c1) > 0)) % ns.CAP == q
