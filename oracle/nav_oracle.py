"""CPU oracle for navigation-message subframe decoding (gypsum/navigation_message_decoder.py with the parts of
gypsum/navigation_message_parser.py it relies on), and a generator of LNAV data and of tracking IQ that carries it.
TEST INFRASTRUCTURE -- see oracle/__init__.py.  Pinned against the live reference decoder through
tests/golden/nav_decoder.npz (tools/make_golden_subframes.py)."""
from __future__ import annotations

import math

import numpy as np

from oracle.gypsum_oracle import replica

SUBFRAME = 300
PREAMBLE = (1, 0, 0, 0, 1, 0, 1, 1)
# IS-GPS-200 Table 20-XIV: for parity bits D25..D30, the previous word's bit that enters (29 = D29*, 30 = D30*) and the
# source data bits d1..d24.
PARITY_EQUATIONS = (
    (29, (1, 2, 3, 5, 6, 10, 11, 12, 13, 14, 17, 18, 20, 23)),
    (30, (2, 3, 4, 6, 7, 11, 12, 13, 14, 15, 18, 19, 21, 24)),
    (29, (1, 3, 4, 5, 7, 8, 12, 13, 14, 15, 16, 19, 20, 22)),
    (30, (2, 4, 5, 6, 8, 9, 13, 14, 15, 16, 17, 20, 21, 23)),
    (30, (1, 3, 5, 6, 7, 9, 10, 14, 15, 16, 17, 18, 21, 22, 24)),
    (29, (3, 5, 6, 8, 9, 10, 11, 13, 15, 19, 22, 23, 24)),
)
KIND_SUBFRAME, KIND_PHASE, KIND_CANNOT, KIND_RAISED = 0, 1, 2, 3
QUEUE_CAPACITY = 4096  # the device decoder's queue (gypsum_b200/csrc/nav_core.cuh)


def parity_bits(source: list[int], d29: int, d30: int) -> list[int]:
    """D25..D30 of a word whose source data bits are `source` (d1..d24), after a word ending in D29*, D30*."""
    out = []
    for prev, taps in PARITY_EQUATIONS:
        acc = d29 if prev == 29 else d30
        for i in taps:
            acc ^= source[i - 1]
        out.append(acc)
    return out


def word_value(bits30) -> int:
    v = 0
    for b in bits30:
        v = (v << 1) | int(b)
    return v


# ---------------------------------------------------------------------------------------------------------------------
# decoder
# ---------------------------------------------------------------------------------------------------------------------
class NavDecoderOracle:
    """One channel's decoder.  `push(bit, t0, t1, index)` takes one bit event (1 / 0 / -1 = unknown) and returns the
    events it produced as tuples (index, kind, subframe_id, tow, phase, polarity, parity_ok, t0, t1, words)."""

    def __init__(self, capacity: int | None = QUEUE_CAPACITY):
        self.capacity = capacity
        self.bits: list[int] = []
        self.t0: list[float] = []
        self.t1: list[float] = []
        self.phase = None
        self.polarity = 0  # +1 upright, -1 inverted, 0 undetermined
        self.emitted = 0
        self.processed = 0
        self.stopped = 0  # 1 the reference raised, 2 the queue was full

    def state(self) -> list[int]:
        """[phase (-1 = None), emitted subframes, polarity, queued bits, stopped, bits taken]."""
        return [-1 if self.phase is None else self.phase, self.emitted, self.polarity, len(self.bits), self.stopped,
                self.processed]

    def _first_pair(self, pattern) -> int | None:
        n = len(self.bits)
        if n < 8:
            return None
        windows = np.lib.stride_tricks.sliding_window_view(np.asarray(self.bits, dtype=np.int8), 8)
        hit = np.all(windows == np.asarray(pattern, dtype=np.int8), axis=1)  # an unknown bit (-1) never matches
        both = hit[:-SUBFRAME] & hit[SUBFRAME:] if hit.size > SUBFRAME else np.zeros(0, dtype=bool)
        idx = np.flatnonzero(both)
        return int(idx[0]) if idx.size else None

    def _search(self, index):
        if len(self.bits) < 2 * SUBFRAME:
            return []
        for pattern, pol in ((PREAMBLE, 1), (tuple(1 - b for b in PREAMBLE), -1)):
            c = self._first_pair(pattern)
            if c is not None:
                self.phase, self.polarity = c, pol
                drop = c % SUBFRAME  # only the partial first subframe goes
                del self.bits[:drop], self.t0[:drop], self.t1[:drop]
                return [(index, KIND_PHASE, 0, 0, c, pol, 0, 0.0, 0.0, (0,) * 10)]
        if len(self.bits) >= 12 * SUBFRAME:
            return [(index, KIND_CANNOT, 0, 0, -1, 0, 0, 0.0, 0.0, (0,) * 10)]
        return []

    def _take_subframe(self, index):
        """(result, event): result 0 = nothing, 1 = a subframe, 2 = the reference raises."""
        block, a, b = self.bits[:SUBFRAME], self.t0[0], self.t1[SUBFRAME - 1]
        del self.bits[:SUBFRAME], self.t0[:SUBFRAME], self.t1[:SUBFRAME]
        if any(v < 0 for v in block):
            self.phase, self.polarity = None, 0
            return 0, None
        if self.polarity < 0:
            block = [1 - v for v in block]
        words = [block[30 * k: 30 * k + 30] for k in range(10)]
        d29 = d30 = 0
        data, ok = [], 0
        for k, w in enumerate(words):
            source = [v ^ d30 for v in w[:24]]
            if parity_bits(source, d29, d30) == list(w[24:]):
                ok |= 1 << k
            data.append(source)
            d29, d30 = w[28], w[29]
        if tuple(data[0][:8]) != PREAMBLE:
            self.phase, self.polarity = None, 0
            return 0, None
        sf_id = word_value(data[1][19:22])
        if not 1 <= sf_id <= 5:
            self.phase, self.polarity = None, 0
            return 0, None
        tow = word_value(data[1][:17])
        ev = (index, KIND_SUBFRAME, sf_id, tow, -1 if self.phase is None else self.phase, self.polarity, ok, a, b,
              tuple(word_value(w) for w in words))
        if sf_id == 5 and data[2][:2] != [0, 1]:
            return 2, ev
        return 1, ev

    def push(self, bit: int, t0: float, t1: float, index: int) -> list:
        if self.stopped:
            return []
        if self.capacity is not None and len(self.bits) == self.capacity:
            self.stopped = 2
            return []
        self.bits.append(int(bit))
        self.t0.append(float(t0))
        self.t1.append(float(t1))
        self.processed += 1
        events = self._search(index) if self.phase is None else []
        if self.phase is not None:
            # every whole subframe is parsed, even after a reset on the way (then with no polarity flip)
            while len(self.bits) >= SUBFRAME:
                r, ev = self._take_subframe(index)
                if r == 1:
                    self.emitted += 1
                    events.append(ev)
                elif r == 2:
                    self.stopped = 1
                    return [(ev[0], KIND_RAISED, *ev[2:])]  # the exception carries nothing else this bit produced
        return events


def decode(bits, t0, t1, capacity: int | None = QUEUE_CAPACITY):
    """A whole stream through one decoder: (event tuples, final state)."""
    dec = NavDecoderOracle(capacity)
    out = []
    for k, (b, a, c) in enumerate(zip(bits, t0, t1)):
        out += dec.push(int(b), float(a), float(c), k)
    return out, dec.state()


def events_to_arrays(events):
    """Event tuples -> (rows float64 [n, 9]: index, kind, id, tow, phase, polarity, parity_ok, t0, t1; words int64 [n, 10])."""
    rows = np.array([e[:9] for e in events], dtype=np.float64).reshape(-1, 9)
    words = np.array([e[9] for e in events], dtype=np.int64).reshape(-1, 10)
    return rows, words


# ---------------------------------------------------------------------------------------------------------------------
# LNAV generator
# ---------------------------------------------------------------------------------------------------------------------
def encode_word(source: list[int], d29: int, d30: int) -> list[int]:
    """The 30 transmitted bits of a word: data complemented by the previous word's D30, then D25..D30."""
    return [v ^ d30 for v in source] + parity_bits(source, d29, d30)


def _int_bits(v: int, n: int) -> list[int]:
    return [(v >> (n - 1 - i)) & 1 for i in range(n)]


def lnav_subframe(sf_id: int, tow_count: int, rng: np.random.Generator, data_id: int = 1, prev=(0, 0)) -> list[int]:
    """300 transmitted bits of one subframe: TLM with the preamble, HOW with the TOW count (of the next subframe's start)
    and the subframe id, random data words (word 3 of subframes 4 and 5 starts with the 2-bit data id), and parity
    throughout.  Words 2 and 10 end in D29 = D30 = 0 through their two solved bits, so the next word starts from 00."""
    d29, d30 = prev
    out = []
    for k in range(10):
        src = [int(v) for v in rng.integers(0, 2, 24)]
        if k == 0:
            src[:8] = PREAMBLE
        elif k == 1:
            src[:17] = _int_bits(tow_count, 17)
            src[19:22] = _int_bits(sf_id, 3)
        elif k == 2 and sf_id in (4, 5):
            src[:2] = _int_bits(data_id, 2)
        if k in (1, 9):
            for t in range(4):
                src[22:24] = _int_bits(t, 2)
                w = encode_word(src, d29, d30)
                if w[28] == 0 and w[29] == 0:
                    break
        w = encode_word(src, d29, d30)
        out += w
        d29, d30 = w[28], w[29]
    return out


def lnav_frames(seed: int, n_subframes: int, first_id: int = 1, tow0: int = 1000, sf5_data_id=lambda k: 1) -> list[list[int]]:
    """n_subframes consecutive subframes (ids cycling 1..5 from first_id, TOW count tow0, tow0 + 1, ...); sf5_data_id(k)
    chooses the data id of subframe k when it is a subframe 5."""
    rng = np.random.default_rng(seed)
    out, prev = [], (0, 0)
    for k in range(n_subframes):
        sf_id = (first_id - 1 + k) % 5 + 1
        bits = lnav_subframe(sf_id, tow0 + k, rng, data_id=sf5_data_id(k) if sf_id == 5 else 1, prev=prev)
        out.append(bits)
        prev = (bits[-2], bits[-1])
    return out


def check_parity(bits300) -> int:
    """parity_ok mask of a subframe from the IS-GPS-200 equations, written out bit by bit."""
    ok, d29, d30 = 0, 0, 0
    for k in range(10):
        w = bits300[30 * k: 30 * k + 30]
        d = [w[i] ^ d30 for i in range(24)]
        want = [
            d29 ^ d[0] ^ d[1] ^ d[2] ^ d[4] ^ d[5] ^ d[9] ^ d[10] ^ d[11] ^ d[12] ^ d[13] ^ d[16] ^ d[17] ^ d[19] ^ d[22],
            d30 ^ d[1] ^ d[2] ^ d[3] ^ d[5] ^ d[6] ^ d[10] ^ d[11] ^ d[12] ^ d[13] ^ d[14] ^ d[17] ^ d[18] ^ d[20] ^ d[23],
            d29 ^ d[0] ^ d[2] ^ d[3] ^ d[4] ^ d[6] ^ d[7] ^ d[11] ^ d[12] ^ d[13] ^ d[14] ^ d[15] ^ d[18] ^ d[19] ^ d[21],
            d30 ^ d[1] ^ d[3] ^ d[4] ^ d[5] ^ d[7] ^ d[8] ^ d[12] ^ d[13] ^ d[14] ^ d[15] ^ d[16] ^ d[19] ^ d[20] ^ d[22],
            d30 ^ d[0] ^ d[2] ^ d[4] ^ d[5] ^ d[6] ^ d[8] ^ d[9] ^ d[13] ^ d[14] ^ d[15] ^ d[16] ^ d[17] ^ d[20] ^ d[21] ^ d[23],
            d29 ^ d[2] ^ d[4] ^ d[5] ^ d[7] ^ d[8] ^ d[9] ^ d[10] ^ d[12] ^ d[14] ^ d[18] ^ d[21] ^ d[22] ^ d[23],
        ]
        if want == list(w[24:]):
            ok |= 1 << k
        d29, d30 = w[28], w[29]
    return ok


def no_preamble_noise(seed: int, n: int) -> np.ndarray:
    """Random bits with no run of three equal bits, so neither the preamble (which holds 000) nor its inverse (111)
    appears anywhere."""
    rng = np.random.default_rng(seed)
    b = rng.integers(0, 2, n).astype(np.int8)
    for i in range(2, n):
        if b[i] == b[i - 1] == b[i - 2]:
            b[i] ^= 1
    return b


def bit_times(n: int, t_first: float = 0.1203, period: float = 0.02):
    t0 = np.round(t_first + np.arange(n) * period, 9)
    return t0, np.round(t0 + period, 9)


def synth_lnav_iq(seed: int, n: int, fs: int, k0: int, n_ms: int, channels, sigma: float = 0.02) -> np.ndarray:
    """Milliseconds [k0, k0 + n_ms) of a recording whose channels (sv, doppler_hz, code_phase, carrier_phase, amplitude,
    bits, first_bit_ms) modulate the given 0/1 bit sequence: bit i spans milliseconds [first_bit_ms + 20 i, +20) as
    +1 (bit 1) / -1 (bit 0); before first_bit_ms the symbol is +1.  Noise sigma per sample, drawn per call from
    (seed, k0), so a long recording can be made a block at a time."""
    rng = np.random.default_rng((seed, k0))
    total = n * n_ms
    x = (rng.standard_normal(total) + 1j * rng.standard_normal(total)) * (sigma / math.sqrt(2.0))
    t = (k0 * n + np.arange(total)) / fs
    ms = k0 + np.arange(n_ms)
    for sv, f, tau_s, phi, amp, bits, first_bit_ms in channels:
        code = np.tile(np.roll(replica(sv, n).real, tau_s), n_ms)
        b = np.asarray(bits, dtype=np.int8)
        i = (ms - first_bit_ms) // 20
        sym = np.where((i >= 0) & (i < b.size), 2.0 * b[np.clip(i, 0, b.size - 1)] - 1.0, 1.0)
        x = x + amp * code * np.repeat(sym, n) * np.exp(1j * (math.tau * f * t + phi))
    return x.astype(np.complex64)
