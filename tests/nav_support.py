"""Bit streams that drive the subframe decoder (nav_core.cuh, nav.cu) into chosen preamble-scan states, and one oracle
run per stream that shares the work of streams with a common prefix.

A full preamble scan only ever runs with 600 bits queued (the first search after the queue's front moved), so what
the device's warp scan sees is fixed by two numbers: the ring position of the queue's head (`qhead`) and the position
`c` of the first preamble pair in the 600 queued bits.  A stream reaches a chosen `qhead` through cycles that each
plant a preamble pair at `c1` of a 600-bit window, which the decoder finds in its full scan:
- a reset cycle's first subframe holds an UNKNOWN bit, so the decoder resets on it, having popped c1 + 300 bits, and
  keeps the 300 - c1 bits from the partner preamble on: the next window starts with that preamble;
- the last cycle's first subframe is an intact LNAV subframe, which the decoder emits; the second, from the partner
  on, holds an UNKNOWN bit, and the reset on it, c1 + 600 bits into the window, leaves the queue empty.  So the target
  window may hold anything from its first bit on (a pair at 1..7 could not follow a partner preamble).
Everything not planted is noise with no run of three equal bits, which holds neither preamble (the upright one
contains 000, the inverted one 111); every window is checked against a model of the search before a stream is
returned."""
from __future__ import annotations

import copy
import zlib
from dataclasses import dataclass, field

import numpy as np

from oracle import nav_oracle as nav

SUB = nav.SUBFRAME
CAP = nav.QUEUE_CAPACITY
WINDOW = 2 * SUB  # bits queued at every full scan
LAST_FULL = WINDOW - 8 - SUB  # 292: the last pair start a full scan can find
PRE = {1: np.array(nav.PREAMBLE, dtype=np.int8), -1: 1 - np.array(nav.PREAMBLE, dtype=np.int8)}


@dataclass
class Stream:
    """One channel's bits.  bits[:split] are shared by every stream with the same key; `decide` is the index of the
    bit whose search finds the target pair, `qhead` the ring position of the queue then."""
    bits: np.ndarray
    key: tuple
    split: int
    qhead: int
    c: int
    pol: int
    decide: int
    name: str = ""
    cycles: list = field(default_factory=list)  # (first bit of the window, c1, polarity) of each cycle

    @property
    def times(self):
        return nav.bit_times(self.bits.size)


def cycle_plan(qhead: int):
    """c1 of each cycle, the reset cycles' first: the reset cycles pop c1 + 300 bits each and the last one c1 + 600,
    c1 in [1, 292], which adds up to qhead modulo the ring."""
    if qhead == 0:
        return []
    q = qhead
    while True:
        for k in range(q // (SUB + 1) + 1):  # k reset cycles
            if (SUB + 1) * k + WINDOW + 1 <= q <= (SUB + LAST_FULL) * k + WINDOW + LAST_FULL:
                base, rem = divmod(q - SUB * k - WINDOW, k + 1)
                return [base + (1 if i < rem else 0) for i in range(k + 1)]
        q += CAP


def decision(window: np.ndarray):
    """The decoder's search over a queue that starts at window[0] and grows one bit at a time: (queued bits when a
    pair is found, pair start, polarity), or None.  The upright preamble is searched first at every length."""
    n = window.size
    if n < WINDOW:
        return None
    hits = {}
    for pol in (1, -1):
        v = np.lib.stride_tricks.sliding_window_view(window, 8)
        h = np.all(v == PRE[pol], axis=1)
        hits[pol] = np.flatnonzero(h[:-SUB] & h[SUB:]) if h.size > SUB else np.zeros(0, dtype=np.int64)
    ends = [int(p[0]) + SUB + 8 for p in hits.values() if p.size]
    if not ends:
        return None
    at = max(WINDOW, min(ends))
    for pol in (1, -1):
        p = hits[pol][hits[pol] + SUB + 8 <= at]
        if p.size:
            return at, int(p[0]), pol
    return None


def _fill(val, fixed, rng, a, b):
    """Noise into the free positions of [a, b): no run of three equal bits with what is left of it or planted right of
    it, where a choice can avoid one."""
    r = rng.integers(0, 2, b - a).tolist()
    v, f = val.tolist(), fixed.tolist()
    n = len(v)
    for i in range(a, b):
        if f[i]:
            continue
        bad = set()
        if i >= 2 and v[i - 1] == v[i - 2] >= 0:
            bad.add(v[i - 1])
        if i + 2 < n and f[i + 1] and f[i + 2] and v[i + 1] == v[i + 2] >= 0:
            bad.add(v[i + 1])
        if i >= 1 and i + 1 < n and f[i + 1] and v[i - 1] == v[i + 1] >= 0:
            bad.add(v[i - 1])
        x = r[i - a]
        v[i] = x ^ 1 if x in bad and len(bad) == 1 else x
    val[a:b] = v[a:b]


def _plant(val, fixed, at, bits):
    bits = np.asarray(bits, dtype=np.int8)
    if at < 0 or at + bits.size > val.size:
        return
    val[at:at + bits.size] = bits
    fixed[at:at + bits.size] = True


class StreamBuilder:
    """Streams for (qhead, c, polarity, content, decoys); the cycles that reach a (qhead, polarity) are built once."""

    def __init__(self, seed: int = 0):
        self.seed = seed
        self._prefix = {}

    def _layout(self, qhead, pol):
        c1s = cycle_plan(qhead)
        k = len(c1s)
        pols = [pol if (k - 1 - i) % 2 == 0 else -pol for i in range(k)]
        starts = [0]
        for i, c1 in enumerate(c1s):
            starts.append(starts[-1] + c1 + (WINDOW if i == k - 1 else SUB))
        split = starts[k - 2] + WINDOW if k >= 2 else 0
        return c1s, pols, starts, split

    def _cycles(self, qhead, pol):
        """(plan, plants, prefix bits) of the cycles that reach qhead, the prefix's windows checked."""
        key = (qhead, pol)
        if key not in self._prefix:
            c1s, pols, starts, split = plan = self._layout(qhead, pol)
            plants = []
            for i, (s, c1, p) in enumerate(zip(starts, c1s, pols)):
                if i < len(c1s) - 1:
                    plants += [(s + c1, PRE[p]), (s + c1 + 150, [-1])]
                else:
                    # the subframe must not complete a pair with the preamble the reset before it left at the window's
                    # start
                    for a in range(100):
                        sf = np.asarray(nav.lnav_subframe(2, 1234, np.random.default_rng((self.seed, 3, s, p + 1, a))), np.int8)
                        sf = sf if p > 0 else 1 - sf
                        if i == 0 or not np.array_equal(sf[SUB - c1:SUB - c1 + 8], PRE[pols[i - 1]]):
                            break
                    plants += [(s + c1, sf), (s + c1 + WINDOW - 150, [-1])]
                plants.append((s + c1 + SUB, PRE[p]))
            n = starts[-1] + WINDOW
            val = np.zeros(n, dtype=np.int8)
            fixed = np.zeros(n, dtype=bool)
            for at, bits in plants:
                _plant(val, fixed, at, bits)
            _fill(val, fixed, np.random.default_rng((self.seed, 1, qhead, pol + 1)), 0, split)
            for s, c1, p in list(zip(starts, c1s, pols))[:-1]:
                assert decision(val[s:s + WINDOW]) == (WINDOW, c1, p), (qhead, pol, s)
            self._prefix[key] = (plan, plants, val[:split].copy())
        return self._prefix[key]

    def build(self, qhead: int, c: int, pol: int = 1, content: str = "lnav", decoys=(), tail: int = 0,
              name: str = "", share: int = 0, attempt: int = 0) -> Stream:
        """content: "lnav" an LNAV subframe (subframe 1, upright or complemented) from the target pair on, "raise" a
        subframe 5 whose data id makes the reference raise, "bare" only the two preambles.  decoys: (offset in the
        target window, bits) planted after the target.  tail: noise bits after the deciding one.  share: the first `share`
        bits of the target window are the same in every stream of this name, qhead and polarity (c > share + 1), so
        that the oracle runs them once."""
        qhead %= CAP
        (c1s, pols, starts, split), plants, prefix = self._cycles(qhead, pol)
        s_t = starts[-1]
        decide_len = max(WINDOW, c + SUB + 8)
        n = s_t + decide_len + tail
        val = np.zeros(n, dtype=np.int8)
        fixed = np.zeros(n, dtype=bool)
        val[:split] = prefix
        fixed[:split] = True
        for at, bits in plants:
            _plant(val, fixed, at, bits)
        rng = np.random.default_rng((self.seed, 2, qhead, pol + 1, 0 if share else c, attempt, zlib.crc32(name.encode())))
        if content == "bare":
            _plant(val, fixed, s_t + c, PRE[pol])
        else:
            sf = nav.lnav_subframe(5 if content == "raise" else 1, 4321, rng, data_id=2)
            sf = np.asarray(sf, dtype=np.int8)
            _plant(val, fixed, s_t + c, sf if pol > 0 else 1 - sf)
        _plant(val, fixed, s_t + c + SUB, PRE[pol])
        for off, bits in decoys:
            _plant(val, fixed, s_t + off, bits)
        _fill(val, fixed, rng, split, n)
        ok = not c1s or decision(val[starts[-2]:starts[-2] + WINDOW]) == (WINDOW, c1s[-1], pols[-1])
        ok = ok and decision(val[s_t:s_t + decide_len]) == (decide_len, c, pol)
        if not ok:
            if attempt >= 20:
                raise RuntimeError(f"no stream for qhead {qhead}, c {c}, polarity {pol}, {name}")
            return self.build(qhead, c, pol, content, decoys, tail, name, share, attempt + 1)
        key = (qhead, pol)
        if share:
            assert c > share + 1
            key, split = (qhead, pol, name, attempt), s_t + share
        return Stream(val, key, split, qhead, c, pol, s_t + decide_len - 1, name, list(zip(starts, c1s, pols)))


# ---- one oracle run per stream, the prefix shared


class OracleRuns:
    """nav_oracle.NavDecoderOracle over streams: (rows, words, final state), bit indices global.  The decoder state
    after a prefix is kept per key and copied for every stream that starts with it."""

    def __init__(self):
        self._after = {}

    def _push(self, dec, s, a, b, out):
        t0, t1 = s.times
        for k in range(a, b):
            out += dec.push(int(s.bits[k]), float(t0[k]), float(t1[k]), k)

    def __call__(self, s: Stream):
        if s.key not in self._after:
            dec, ev = nav.NavDecoderOracle(), []
            self._push(dec, s, 0, s.split, ev)
            self._after[s.key] = (s.bits[:s.split].copy(), dec, ev)
        prefix, dec, ev = self._after[s.key]
        assert np.array_equal(prefix, s.bits[:s.split])
        dec, ev = copy.deepcopy(dec), list(ev)
        self._push(dec, s, s.split, s.bits.size, ev)
        rows, words = nav.events_to_arrays(ev)
        return rows, words, dec.state()


def first_phase(rows, at: int):
    """(bit index, phase, polarity) of the first phase event at or after bit `at`, or of the raise that took it along
    (a subframe 5 drained by the same bit)."""
    ph = rows[np.isin(rows[:, 1], (nav.KIND_PHASE, nav.KIND_RAISED)) & (rows[:, 0] >= at)]
    return (int(ph[0, 0]), int(ph[0, 4]), int(ph[0, 5])) if len(ph) else None


# ---- decoys, as (offset in the target window, bits)


def unknown_at(pol, k):
    b = PRE[pol].copy()
    b[k] = -1
    return b


# ---- the grids the CPU and GPU tests share

QHEADS = (0, 1, 31, 32)
WORD_C = (0, 1, 19, 20, 31, 32, 287, 288, 291, 292)
INCREMENTAL_QLEN = (601, 602, 631, 632, 633, 900, 908, 3599, 3600, 3601, 3608, 4095, 4096)


def candidate_grid(b: StreamBuilder):
    """Every pair start 0..292 a full scan can find, and 293 (found by the append after it), at ring heads 0, 1, 31
    and 32, upright and complemented."""
    return [b.build(q, c, pol, name="cand") for q in QHEADS for pol in (1, -1) for c in range(LAST_FULL + 2)]


def word_offset_grid(b: StreamBuilder):
    """Every ring head modulo 32, at pair starts on both sides of each 32-bit chunk edge and the last one."""
    return [b.build(32 * (10 + o % 8) + o, c, pol, name="word") for o in range(32) for c in WORD_C for pol in (1, -1)]


def wrap_grid(b: StreamBuilder):
    """Windows that cross the end of the ring (the wrap `w` bits into the window) at every 32-bit chunk of the window:
    the first preamble straddles it, the partner straddles it, or the wrap falls inside the first subframe."""
    out = []
    for w in sorted({32 * k + o for k in range(19) for o in (0, 1, 31)} - {0}):
        if w >= WINDOW:
            continue
        for c in sorted({w - 4, w - 7, w - SUB - 4, w - SUB - 1, w - 150}):
            if 0 <= c <= LAST_FULL:
                for pol in (1, -1):
                    out.append(b.build(CAP - w, c, pol, name=f"wrap{w}"))
    return out


def decoy_grid(b: StreamBuilder):
    """Candidates the scan must reject or rank below the planted pair, at ring heads inside a word, at a word edge and
    across the wrap."""
    out = []
    for q in (0, 333, 3700):
        for pol in (1, -1):
            c, d = 200, 60
            cases = {
                "lone": [(d, PRE[pol])],
                "lone_other": [(d, PRE[-pol])],
                "lone_after": [(c + 40, PRE[pol]), (c + 23, PRE[-pol])],
                "gap299": [(d, PRE[pol]), (d + SUB - 1, PRE[pol])],
                "gap301": [(d, PRE[pol]), (d + SUB + 1, PRE[pol])],
                "partner_other": [(d, PRE[pol]), (d + SUB, PRE[-pol])],
            }
            for k in range(8):
                cases[f"partner_unknown{k}"] = [(d, PRE[pol]), (d + SUB, unknown_at(pol, k))]
                cases[f"first_unknown{k}"] = [(d, unknown_at(pol, k)), (d + SUB, PRE[pol])]
            for name, decoys in cases.items():
                out.append(b.build(q, c, pol, "bare", decoys, name=name))
        # an inverted pair before the upright one: the upright pair wins
        for d in (8, 60, 199):
            out.append(b.build(q, 207, 1, "bare", [(d, PRE[-1]), (d + SUB, PRE[-1])], name=f"inverted_first{d}"))
        # two upright pairs in one 32-bit chunk of the scan: the first wins
        for c in (0, 5, 64, 100, 227, 266):
            for d2 in sorted({8, 31 - c % 32}):
                if c + d2 <= LAST_FULL:
                    out.append(b.build(q, c, 1, "bare", [(c + d2, PRE[1]), (c + d2 + SUB, PRE[1])], name=f"two{d2}"))
    return out


def incremental_grid(b: StreamBuilder):
    """Pairs the append after a search without one completes, at the queue lengths around 600, the chunk edges of
    the first scan, 3600 (where CannotDetermine starts) and 4096 (the last bit before the queue is full), and at pair
    starts that are multiples of 300 (nothing popped before the drain)."""
    return [b.build(0 if pol > 0 else 3001, n - SUB - 8, pol, name="incr" if n < 1000 else "incr_long", tail=5,
                    share=0 if n < 1000 else min(INCREMENTAL_QLEN[7:]) - SUB - 10)
            for n in INCREMENTAL_QLEN for pol in (1, -1)]


def raise_streams(b: StreamBuilder):
    """A subframe 5 that makes the reference raise, right behind the full scan and behind an append."""
    return [b.build(q, c, pol, "raise", name="raise", tail=40) for q, c, pol in ((0, 100, 1), (32, 292, -1), (31, 300, 1),
                                                                               (4000, 3, -1))]


def deciding_bits(s: Stream):
    """The bits whose search finds a pair: each reset cycle's 600th and the target's."""
    return [st + WINDOW - 1 for st, _, _ in s.cycles] + [s.decide]
