"""The subframe decoder's warp-parallel preamble scan (warp_first_pair in nav.cu) at every candidate, ring and call edge,
and the decoder kernel at its channel edges, against the oracle decoder bit for bit: rows, words and final state.

The scan runs on the device only (the host build scans serially), so these streams are built to reach chosen scan
states (tests/nav_support.py; tests/test_nav_edges_cpu.py shows each one gets there): every pair start 0..292 at ring
heads 0, 1, 31 and 32, upright and complemented; every head modulo 32 at the pair starts on both sides of a 32-bit chunk
edge; windows across the end of the 4096-bit ring; decoys the scan must reject or rank below the planted pair; pairs
first completed by an append, up to the last bit before the queue is full.  The streams go to the device as bit events
through Tracker.decode_subframes, one stream per channel, at most 1000 channels per tracker."""
import time

import numpy as np
import pytest

import nav_support as ns
from gpu_support import make_engine
from oracle import nav_oracle as nav

pytestmark = pytest.mark.gpu
N, FS = 2046, 2046000
MAX_CHANNELS = 1000
PLACEMENTS = (0, 1, 30, 31, 32, 33, "last", "alone")


@pytest.fixture(scope="module")
def engine(native_lib):
    e = make_engine(FS, N)
    yield e
    e.close()


@pytest.fixture(scope="module")
def builder():
    return ns.StreamBuilder()


@pytest.fixture(scope="module")
def oracle():
    return ns.OracleRuns()


def decode_on_device(engine, chans, stride_pad=0):
    """chans: (stream, cuts) per channel.  Call i hands channel c the i-th piece of its stream cut at its cuts (none
    once they run out) in a [n_channels][stride] device array, stride the longest piece + stride_pad.  Returns the
    rows and words per channel (bit indices within the stream) and the tracker, still open."""
    import torch

    from gypsum_b200 import _native

    n_ch = len(chans)
    pieces = [list(zip([0, *cuts], [*cuts, s.bits.size])) for s, cuts in chans]
    times = [s.times for s, _ in chans]
    trk = _native.Tracker(engine, [c % 32 for c in range(n_ch)], [0.0] * n_ch, [0.0] * n_ch, [0] * n_ch)
    rows = [[] for _ in range(n_ch)]
    words = [[] for _ in range(n_ch)]
    for i in range(max(len(p) for p in pieces)):
        spans = [p[i] if i < len(p) else (0, 0) for p in pieces]
        counts = np.array([b - a for a, b in spans], dtype=np.int32)
        stride = max(1, int(counts.max())) + stride_pad
        host = np.zeros((n_ch, stride), dtype=_native.BIT_DTYPE)
        for c, ((s, _), (a, b), (t0, t1)) in enumerate(zip(chans, spans, times)):
            host["bit_value"][c, :b - a] = s.bits[a:b]
            host["receiver_timestamp"][c, :b - a] = t0[a:b]
            host["trailing_edge_receiver_timestamp"][c, :b - a] = t1[a:b]
        dev = torch.from_numpy(host.view(np.uint8).reshape(n_ch, -1)).cuda()
        ev = trk.decode_subframes(dev.data_ptr(), counts, stride)
        for c, (a, _) in enumerate(spans):
            e = ev[c]
            rows[c].append(np.stack([a + e["bit_index"], e["kind"], e["subframe_id"], e["tow"], e["phase"], e["polarity"],
                                     e["parity_ok"], e["receiver_timestamp"], e["trailing_edge_receiver_timestamp"]],
                                    axis=1).astype(np.float64).reshape(-1, 9))
            words[c].append(e["words"].astype(np.int64).reshape(-1, 10))
    return [np.concatenate(r) for r in rows], [np.concatenate(w) for w in words], trk


def _state_list(st):
    return [-1 if st["determined_subframe_phase"] is None else st["determined_subframe_phase"], st["emitted_subframe_count"],
            st["polarity"], st["queued_bit_count"], st["stopped"], st["processed_bit_count"]]


def check_on_device(engine, oracle, chans, what, stride_pad=0):
    """chans through the device, at most MAX_CHANNELS per tracker, each channel against the oracle."""
    for g in range(0, len(chans), MAX_CHANNELS):
        group = chans[g:g + MAX_CHANNELS]
        rows, words, trk = decode_on_device(engine, group, stride_pad)
        for c, (s, cuts) in enumerate(group):
            want_rows, want_words, want_final = oracle(s)
            tag = (what, s.name, s.qhead, s.c, s.pol, cuts[:4])
            assert np.array_equal(rows[c], want_rows), (tag, rows[c][-3:, :7], want_rows[-3:, :7])
            assert np.array_equal(words[c], want_words), tag
            assert _state_list(trk.subframe_state(c)) == want_final, tag
        trk.close()


def _in_calls(streams, size=1000):
    """Each stream in calls of `size` bits, the first call shorter by the channel's number modulo 61, so that the
    deciding bits fall on many lanes."""
    return [(s, list(range(size - c % 61, s.bits.size, size))) for c, s in enumerate(streams)]


def _run_grid(engine, builder, oracle, grid):
    t0 = time.time()
    streams = getattr(ns, grid)(builder)
    check_on_device(engine, oracle, _in_calls(streams), grid)
    print(f"{grid}: {len(streams)} streams, {time.time() - t0:.1f} s")


def test_every_candidate(engine, builder, oracle):
    """Pair starts 0..292 (full scan) and 293 (the append on bit 601) at ring heads 0, 1, 31, 32, both polarities."""
    _run_grid(engine, builder, oracle, "candidate_grid")


def test_every_word_offset(engine, builder, oracle):
    _run_grid(engine, builder, oracle, "word_offset_grid")


def test_ring_wrap(engine, builder, oracle):
    _run_grid(engine, builder, oracle, "wrap_grid")


def test_decoys(engine, builder, oracle):
    """Lone preambles, partners at +299 / +301, a partner or first preamble with one UNKNOWN bit at each position, a
    partner of the other polarity, an inverted pair before the upright one, two upright pairs in one 32-bit chunk."""
    _run_grid(engine, builder, oracle, "decoy_grid")


def test_incremental_finds_and_raises(engine, builder, oracle):
    """Pairs completed by an append at 601 .. 4096 queued bits (CannotDetermine from 3600 on, the last bit before the
    queue is full, a pair at a multiple of 300), and subframe 5 raises behind both kinds of search."""
    _run_grid(engine, builder, oracle, "incremental_grid")
    _run_grid(engine, builder, oracle, "raise_streams")


def _call_edge_streams(builder):
    return [builder.build(0, 100, 1, name="edge"), builder.build(31, 292, -1, name="edge"),
            builder.build(32, 0, 1, name="edge"), builder.build(1, 325, -1, name="edge", tail=30),
            builder.build(4000, 17, 1, name="edge", tail=40)] + ns.raise_streams(builder)


def _placed_cuts(s, p):
    """Cuts that put every deciding bit of s at in-call index p, at the end of its call ("last") or alone in a
    one-bit call ("alone")."""
    cuts = set()
    for d in ns.deciding_bits(s):
        if p == "last":
            cuts.add(d + 1)
        elif p == "alone":
            cuts |= {d, d + 1}
        else:
            cuts.add(d - p)
    return sorted(c for c in cuts if 0 < c < s.bits.size)


def test_call_edges(engine, builder, oracle):
    """The 600th bit of every full scan, the bit that completes a pair and the bit of a subframe 5 raise, each at
    in-call index 0, 1, 30, 31, 32, 33, at the last index and alone in a one-bit call; one channel per placement and
    stream, so the calls carry different counts, zero once a channel's pieces run out."""
    chans = []
    for s in _call_edge_streams(builder):
        for p in PLACEMENTS:
            cuts = _placed_cuts(s, p)
            for d in ns.deciding_bits(s):
                start = max([0] + [c for c in cuts if c <= d])
                end = min([s.bits.size] + [c for c in cuts if c > d])
                assert {"last": end - 1 == d, "alone": start == d and end == d + 1}.get(p, d - start == p)
            chans.append((s, cuts))
    check_on_device(engine, oracle, chans, "call edges")


@pytest.mark.parametrize("n_ch", range(1, 10))
def test_channel_counts(engine, builder, oracle, n_ch):
    """1..9 channels (blocks of four decoder warps, the last one partial), each its own stream in calls of its own
    size, so counts differ within a call and drop to zero, with a stride larger than the longest count."""
    pool = _call_edge_streams(builder)
    chans = []
    for c in range(n_ch):
        s = pool[(c + n_ch) % len(pool)]
        size = 97 + 131 * c
        chans.append((s, list(range(size, s.bits.size, size))))
    check_on_device(engine, oracle, chans, ("channels", n_ch), stride_pad=7)
