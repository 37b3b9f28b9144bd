"""CPU oracle for subframe field parsing (gypsum/navigation_message_parser.py:426-673), the world model's per-satellite
orbit state and PRN counting (gypsum/world_model.py:297-328, :707-861, receiver.py:106-137) and the per-millisecond
satellite time and position (world_model.py:379-487, :635-705), in float64 with the reference's order of operations;
and an LNAV encoder that writes given ephemeris and clock values into subframes 1-5 with valid parity.
TEST INFRASTRUCTURE -- see oracle/__init__.py.  Pinned against the live reference through tests/golden/orbit.npz
(tools/make_golden_orbit.py)."""
from __future__ import annotations

import math

import numpy as np

from oracle import nav_oracle as nav

N_PARAMS = 26
(SQRT_A, A, E, I0, OMEGA0, OMEGA, M0, DN, CUC, CUS, CRC, CRS, CIC, CIS, OMEGA_DOT, IDOT, WEEK, TOE, TOW_LAST, RX_HOW,
 PRN_LEADING, AF0, AF1, AF2, TOC, TGD) = range(N_PARAMS)
PI = 3.1415926535898  # world_model.py:39
OBS_TIMING, OBS_COMPLETE, OBS_FIX_GATE, OBS_COUNTING, OBS_FROZEN = 1, 2, 4, 8, 16


# ---------------------------------------------------------------------------------------------------------------------
# parsing
# ---------------------------------------------------------------------------------------------------------------------
def data_words(words) -> list[list[int]]:
    """The 24 data bits of each word after preprocess_next_word: complemented by the previous word's D30 (word 1: 0)."""
    out, d30 = [], 0
    for w in words:
        bits = [(int(w) >> (29 - i)) & 1 for i in range(30)]
        out.append([(b + d30) % 2 for b in bits[:24]])
        d30 = bits[29]
    return out


def _value(bits) -> int:
    return int("".join(str(b) for b in bits), 2)


def _num(bits, exp: int, twos: bool) -> float:
    v = _value(bits)
    if twos and bits[0] == 1:
        v -= 1 << len(bits)
    return float(v * (2 ** exp))


def parse(words) -> dict:
    """A subframe's words -> {subframe_id, tow_seconds, ints, bits, widths, values} in gb200_subframe_fields' layout."""
    d = data_words(words)
    flat = [b for w in d[2:] for b in w]  # words 3..10, 24 bits each

    def f(word, first, n):  # data bits [first, first + n) of `word` (1-based)
        k = (word - 3) * 24 + first - 1
        return flat[k:k + n]

    how = d[1]
    sf = _value(how[19:22])
    tow = 0.0
    for i, bit in enumerate(reversed(how[:17])):
        if bit == 1:
            tow += 1.5 * (math.pow(2, i + 2))
    ints, bits, values = [], [], []
    if sf == 1:
        ints = [_value(f(3, 1, 10)), f(4, 1, 1)[0]]
        bits = [f(3, 11, 2), f(3, 13, 4), f(3, 17, 6), f(3, 23, 2) + f(8, 1, 8)]
        values = [_num(f(7, 17, 8), -31, True), _num(f(8, 9, 16), 4, False), _num(f(9, 1, 8), -55, True),
                  _num(f(9, 9, 16), -43, True), _num(f(10, 1, 22), -31, True)]
    elif sf == 2:
        ints = [f(10, 17, 1)[0]]
        bits = [f(3, 1, 8), f(10, 18, 5)]
        values = [_num(f(3, 9, 16), -5, True), _num(f(4, 1, 16), -43, True), _num(f(4, 17, 8) + f(5, 1, 24), -31, True),
                  _num(f(6, 1, 16), -29, True), _num(f(6, 17, 8) + f(7, 1, 24), -33, False), _num(f(8, 1, 16), -29, True),
                  _num(f(8, 17, 8) + f(9, 1, 24), -19, False), _num(f(10, 1, 16), 4, False)]
    elif sf == 3:
        bits = [f(10, 1, 8)]
        values = [_num(f(3, 1, 16), -29, True), _num(f(3, 17, 8) + f(4, 1, 24), -31, True), _num(f(5, 1, 16), -29, True),
                  _num(f(5, 17, 8) + f(6, 1, 24), -31, True), _num(f(7, 1, 16), -5, True),
                  _num(f(7, 17, 8) + f(8, 1, 24), -31, True), _num(f(9, 1, 24), -43, True), _num(f(10, 9, 14), -43, True)]
    elif sf == 4:
        ints = [_value(f(3, 1, 2)), _value(f(3, 3, 6))]
    elif sf == 5:
        bits = [f(3, 1, 2), f(3, 3, 6), f(5, 17, 8)]
        values = [_num(f(3, 9, 16), -21, False), _num(f(4, 1, 8), 12, False), _num(f(4, 9, 16), -19, True),
                  _num(f(5, 1, 16), -38, True), _num(f(6, 1, 24), -11, False), _num(f(7, 1, 24), -23, True),
                  _num(f(8, 1, 24), -23, True), _num(f(9, 1, 24), -23, True), _num(f(10, 1, 8) + f(10, 20, 3), -20, True),
                  _num(f(10, 9, 11), -38, True)]
    pad = lambda xs, n, z: list(xs) + [z] * (n - len(xs))  # noqa: E731
    return {"subframe_id": sf, "tow_seconds": tow, "ints": pad(ints, 2, 0), "bits": pad([_value(b) for b in bits], 4, 0),
            "widths": pad([len(b) for b in bits], 4, 0), "values": pad(values, 10, 0.0)}


# ---------------------------------------------------------------------------------------------------------------------
# the world model's per-satellite state
# ---------------------------------------------------------------------------------------------------------------------
class OrbitOracle:
    """One satellite's entry of GpsWorldModel, with the receiver's per-millisecond order."""

    def __init__(self):
        self.p: list = [None] * N_PARAMS
        self.count = 0
        self.counting = False
        self.frozen = False

    def subframe(self, fields: dict, trailing_edge: float) -> None:  # handle_subframe_emitted
        self.count = 0
        self.counting = True
        p, v, sf = self.p, fields["values"], fields["subframe_id"]
        p[TOW_LAST] = fields["tow_seconds"]
        p[RX_HOW] = p[PRN_LEADING] = trailing_edge
        if sf == 1:
            p[WEEK] = fields["ints"][0] + 2048
            p[AF0], p[AF1], p[AF2], p[TOC], p[TGD] = v[4], v[3], v[2], v[1], v[0]
        elif sf == 2:
            p[M0] = v[2] * PI
            p[E] = v[4]
            p[SQRT_A] = v[6]
            p[A] = math.pow(v[6], 2)
            p[DN] = v[1] * PI
            p[TOE], p[CUC], p[CUS], p[CRS] = v[7], v[3], v[5], v[0]
        elif sf == 3:
            p[I0], p[OMEGA], p[OMEGA0] = v[3] * PI, v[5] * PI, v[1] * PI
            p[CIC], p[CIS] = v[0], v[2]
            p[OMEGA_DOT], p[IDOT] = v[6] * PI, v[7] * PI
            p[CRC] = v[4]

    def lost(self) -> None:  # handle_lost_satellite_lock
        self.counting = False
        self.count = 0
        self.p[TOW_LAST] = None

    def prn_observed(self) -> None:  # handle_prn_observed
        if not self.counting:
            self.counting, self.count = True, 0
        self.count += 1

    # -- observation -----------------------------------------------------------------------------------------------
    def _ecc(self, tk):
        p = self.p
        a = math.pow(p[SQRT_A], 2)
        n = math.sqrt(3.986004418e14) / math.sqrt(math.pow(a, 3)) + p[DN]
        m = p[M0] + (n * tk)
        e = m
        for _ in range(7):
            e = m + (p[E] * math.sin(e))
        return e

    def time_of_week(self):
        p = self.p
        cur = p[TOW_LAST]
        cur += 0.001 * self.count
        dsv = 0
        for _ in range(10):
            t = cur
            tk = cur - p[TOE]
            ek = self._ecc(tk - dsv)
            dtr = -4.442807633e-10 * p[E] * p[SQRT_A] * math.sin(ek)
            dsv = p[AF0] + (p[AF1] * (t - p[TOC])) + (math.pow(p[AF2] * (t - p[TOC]), 2)) + dtr - p[TGD]
        return cur - dsv, dsv

    def position(self, tow):
        p = self.p
        we = 7.2921151467e-5
        tk = tow - p[TOE]
        if tk > 302_400:
            tk -= 604_800
        elif tk < -302_400:
            tk += 604_800
        e = p[E]
        ek = self._ecc(tk)
        vk = math.atan2(math.sqrt(1 - (e * e)) * math.sin(ek), math.cos(ek) - e)
        phi = vk + p[OMEGA]
        duk = (p[CUS] * math.sin(2 * phi)) + (p[CUC] * math.cos(2 * phi))
        drk = (p[CRS] * math.sin(2 * phi)) + (p[CRC] * math.cos(2 * phi))
        dik = (p[CIS] * math.sin(2 * phi)) + (p[CIC] * math.cos(2 * phi))
        uk = phi + duk
        rk = (p[A] * (1 - (e * math.cos(ek)))) + drk
        ik = p[I0] + (p[IDOT] * tk) + dik
        xp, yp = rk * math.cos(uk), rk * math.sin(uk)
        om = p[OMEGA0] + ((p[OMEGA_DOT] - we) * tk) - (we * p[TOE])
        x = (xp * math.cos(om)) - (yp * math.cos(ik) * math.sin(om))
        y = (xp * math.sin(om)) + (yp * math.cos(ik) * math.cos(om))
        z = yp * math.sin(ik)
        return x, y, z

    def observe(self) -> tuple:
        """(tow, dsv, x, y, z, prn_count, flags) at the end of the current millisecond; NaN where not computed."""
        p = self.p
        complete = all(v is not None for v in p)
        timing = self.counting and all(p[k] is not None for k in (TOW_LAST, E, SQRT_A, AF0, AF1, AF2, TOC, TGD))
        flags = ((OBS_COUNTING if self.counting else 0) | (OBS_TIMING if timing else 0) | (OBS_COMPLETE if complete else 0)
                 | (OBS_FIX_GATE if self.counting and self.count <= 6000 else 0) | (OBS_FROZEN if self.frozen else 0))
        tow = dsv = x = y = z = math.nan
        if timing:
            tow, dsv = self.time_of_week()
            if complete:
                x, y, z = self.position(tow)
        return tow, dsv, x, y, z, self.count if self.counting else -1, flags

    def params(self) -> tuple[np.ndarray, int]:
        vals = np.array([0.0 if v is None else float(v) for v in self.p])
        mask = sum(1 << k for k, v in enumerate(self.p) if v is not None)
        return vals, mask


def run_call(sv: OrbitOracle, events, drop_ms: int, n_ms: int, observe=True):
    """One call of one channel: events [(kind, words, trailing_edge, ms)] in millisecond order, the drop millisecond
    (-1 = none).  Returns the parsed fields of the kind-0 events and, with observe, the observation of every ms.

    The events of one millisecond apply in order (DESIGN.md §8b): a raise freezes the channel after the subframes before
    it in its millisecond, so that millisecond is counted only when one of them precedes the raise; what follows the
    raise is ignored.  The reference's decoder never emits both in one millisecond."""
    fields = [(j, ms, parse(w)) for j, (kind, w, _, ms) in enumerate(events) if kind == nav.KIND_SUBFRAME]
    by_ms: dict = {}
    for kind, w, te, ms in events:
        by_ms.setdefault(ms, []).append((kind, w, te))
    obs = []
    tracked = True
    for m in range(n_ms):
        tracked = step(sv, by_ms.get(m, []), m == drop_ms, tracked)
        if observe:
            obs.append(sv.observe())
    return fields, obs


def step(sv: OrbitOracle, evs, dropped_here: bool, tracked: bool) -> bool:
    """One millisecond of run_call: its events [(kind, words, trailing_edge)] in order, whether the channel is dropped
    at it and whether it is still tracked.  Returns whether it is tracked after it."""
    if sv.frozen:
        return tracked
    if dropped_here and tracked:
        sv.lost()
        tracked = False
    r = next((i for i, (k, _, _) in enumerate(evs) if k == nav.KIND_RAISED), len(evs))
    before = [(w, te) for k, w, te in evs[:r] if k == nav.KIND_SUBFRAME]
    if tracked and (r == len(evs) or before):
        sv.prn_observed()
        for w, te in before:
            sv.subframe(parse(w), te)
    if tracked and r < len(evs):
        sv.frozen = True  # the step of millisecond m never returns: nothing after the raise is counted
    return tracked


# ---------------------------------------------------------------------------------------------------------------------
# LNAV encoder
# ---------------------------------------------------------------------------------------------------------------------
# per subframe: (field, word, first bit, width); a split field's parts end in _hi / _lo.  Values are the raw integers
# the satellite transmits (two's complement where the parser reads it so)
LAYOUT = {
    1: [("wn", 3, 1, 10), ("l2_codes", 3, 11, 2), ("ura", 3, 13, 4), ("health", 3, 17, 6), ("iodc_hi", 3, 23, 2),
        ("l2p", 4, 1, 1), ("tgd", 7, 17, 8), ("iodc_lo", 8, 1, 8), ("toc", 8, 9, 16), ("af2", 9, 1, 8),
        ("af1", 9, 9, 16), ("af0", 10, 1, 22)],
    2: [("iode", 3, 1, 8), ("crs", 3, 9, 16), ("dn", 4, 1, 16), ("m0_hi", 4, 17, 8), ("m0_lo", 5, 1, 24),
        ("cuc", 6, 1, 16), ("e_hi", 6, 17, 8), ("e_lo", 7, 1, 24), ("cus", 8, 1, 16), ("sqrta_hi", 8, 17, 8),
        ("sqrta_lo", 9, 1, 24), ("toe", 10, 1, 16), ("fit", 10, 17, 1), ("aodo", 10, 18, 5)],
    3: [("cic", 3, 1, 16), ("omega0_hi", 3, 17, 8), ("omega0_lo", 4, 1, 24), ("cis", 5, 1, 16), ("i0_hi", 5, 17, 8),
        ("i0_lo", 6, 1, 24), ("crc", 7, 1, 16), ("omega_hi", 7, 17, 8), ("omega_lo", 8, 1, 24), ("omegadot", 9, 1, 24),
        ("iode", 10, 1, 8), ("idot", 10, 9, 14)],
    4: [("data_id", 3, 1, 2), ("page_id", 3, 3, 6)],
    5: [("data_id", 3, 1, 2), ("sv_id", 3, 3, 6), ("alm_e", 3, 9, 16), ("toa", 4, 1, 8), ("delta_i", 4, 9, 16),
        ("alm_omegadot", 5, 1, 16), ("alm_health", 5, 17, 8), ("alm_sqrta", 6, 1, 24), ("alm_omega0", 7, 1, 24),
        ("alm_omega", 8, 1, 24), ("alm_m0", 9, 1, 24), ("alm_af0_hi", 10, 1, 8), ("alm_af1", 10, 9, 11),
        ("alm_af0_lo", 10, 20, 3)],
}
SPLIT = {"m0": 24, "e": 24, "sqrta": 24, "omega0": 24, "i0": 24, "omega": 24, "iodc": 8, "alm_af0": 3}


def _raw_fields(sf: int, eph: dict) -> dict:
    """Split fields (m0, e, ...) into their high and low parts, two's complement values into unsigned ones."""
    out = {}
    for name, _, _, width in LAYOUT[sf]:
        base = name[:-3] if name.endswith(("_hi", "_lo")) else name
        v = int(eph.get(base, 0))
        if base in SPLIT:  # the low part is SPLIT[base] bits wide
            lo = SPLIT[base]
            v = (v >> lo) if name.endswith("_hi") else v & ((1 << lo) - 1)
        out[name] = v & ((1 << width) - 1)
    return out


def encode_subframe(sf: int, tow_count: int, eph: dict, prev=(0, 0), rng=None) -> list[int]:
    """300 transmitted bits of subframe `sf` carrying the raw values of `eph` (unlisted fields 0, reserved bits random
    when rng is given), the HOW's TOW count and parity; words 2 and 10 end in D29 = D30 = 0."""
    src = [[0] * 24 for _ in range(10)]
    if rng is not None:
        for k in range(2, 10):
            src[k] = [int(v) for v in rng.integers(0, 2, 24)]
    src[0][:8] = nav.PREAMBLE
    src[1][:17] = [(tow_count >> (16 - i)) & 1 for i in range(17)]
    src[1][17:19] = [0, 0]
    src[1][19:22] = [(sf >> (2 - i)) & 1 for i in range(3)]
    for name, (word, first, width) in ((n, (w, f, wd)) for n, w, f, wd in LAYOUT[sf]):
        v = _raw_fields(sf, eph)[name]
        src[word - 1][first - 1: first - 1 + width] = [(v >> (width - 1 - i)) & 1 for i in range(width)]
    d29, d30 = prev
    out = []
    for k in range(10):
        s = src[k]
        if k in (1, 9):
            for t in range(4):
                s[22:24] = [t >> 1, t & 1]
                w = nav.encode_word(s, d29, d30)
                if w[28] == 0 and w[29] == 0:
                    break
        w = nav.encode_word(s, d29, d30)
        out += w
        d29, d30 = w[28], w[29]
    return out


def words_of(bits300) -> tuple:
    return tuple(nav.word_value(bits300[30 * k: 30 * k + 30]) for k in range(10))


def realistic_ephemeris(rng: np.random.Generator, sv: int) -> dict:
    """Raw ephemeris and clock values in the ranges GPS satellites broadcast."""
    r = lambda lo, hi: int(rng.integers(lo, hi))  # noqa: E731
    toe = r(0, 37800)  # 16 s units
    return {
        "wn": r(0, 1024), "l2_codes": 1, "ura": r(0, 4), "health": 0, "iodc": r(0, 1024), "l2p": 0,
        "tgd": r(-20, 20), "toc": toe, "af2": 0, "af1": r(-500, 500), "af0": r(-400000, 400000),
        "iode": r(0, 256), "crs": r(-3000, 3000), "dn": r(10000, 15000), "m0": r(-2 ** 31, 2 ** 31),
        "cuc": r(-40000, 40000), "e": r(10 ** 6, 1.7 * 10 ** 8), "cus": r(-40000, 40000),
        "sqrta": round(5153.6 * 2 ** 19) + r(-50000, 50000), "toe": toe, "fit": 0, "aodo": r(0, 32),
        "cic": r(-1000, 1000), "omega0": r(-2 ** 31, 2 ** 31), "cis": r(-1000, 1000),
        "i0": round(0.305 * 2 ** 31) + r(-10 ** 7, 10 ** 7), "crc": r(3000, 10000), "omega": r(-2 ** 31, 2 ** 31),
        "omegadot": r(-45000, -30000), "idot": r(-400, 400), "data_id": 1, "page_id": 25, "sv_id": sv,
    }


def ephemeris_subframes(eph: dict, n: int, first_id: int = 1, tow0: int = 1000, seed: int = 0) -> list[list[int]]:
    """n consecutive subframes (ids cycling 1..5 from first_id, TOW counts tow0, tow0 + 1, ...) carrying eph."""
    rng = np.random.default_rng(seed)
    out, prev = [], (0, 0)
    for k in range(n):
        sf = (first_id - 1 + k) % 5 + 1
        bits = encode_subframe(sf, tow0 + k, eph, prev, rng)
        out.append(bits)
        prev = (bits[-2], bits[-1])
    return out


def planted_values(sf: int, eph: dict) -> list[float]:
    """The float fields a parser must return for subframe sf of eph, in gb200_subframe_fields order."""
    s = lambda v, n: v - (1 << n) if v >> (n - 1) & 1 else v  # noqa: E731
    raw = {name: v for name, v in _raw_fields(sf, eph).items()}
    j = lambda a, b, nb: (raw[a] << nb) | raw[b]  # noqa: E731
    if sf == 1:
        return [s(raw["tgd"], 8) * 2.0 ** -31, raw["toc"] * 16.0, s(raw["af2"], 8) * 2.0 ** -55,
                s(raw["af1"], 16) * 2.0 ** -43, s(raw["af0"], 22) * 2.0 ** -31]
    if sf == 2:
        return [s(raw["crs"], 16) * 2.0 ** -5, s(raw["dn"], 16) * 2.0 ** -43, s(j("m0_hi", "m0_lo", 24), 32) * 2.0 ** -31,
                s(raw["cuc"], 16) * 2.0 ** -29, j("e_hi", "e_lo", 24) * 2.0 ** -33, s(raw["cus"], 16) * 2.0 ** -29,
                j("sqrta_hi", "sqrta_lo", 24) * 2.0 ** -19, raw["toe"] * 16.0]
    if sf == 3:
        return [s(raw["cic"], 16) * 2.0 ** -29, s(j("omega0_hi", "omega0_lo", 24), 32) * 2.0 ** -31,
                s(raw["cis"], 16) * 2.0 ** -29, s(j("i0_hi", "i0_lo", 24), 32) * 2.0 ** -31, s(raw["crc"], 16) * 2.0 ** -5,
                s(j("omega_hi", "omega_lo", 24), 32) * 2.0 ** -31, s(raw["omegadot"], 24) * 2.0 ** -43,
                s(raw["idot"], 14) * 2.0 ** -43]
    return []


# ---------------------------------------------------------------------------------------------------------------------
# the recorded timelines (tests/golden/orbit.npz)
# ---------------------------------------------------------------------------------------------------------------------
def golden_calls(z, name: str):
    """[(n_ms, [per channel: ([(kind, words, receiver_timestamp, trailing_edge, ms)], drop_ms)])] of one timeline."""
    ev, words, drop = z[f"{name}_events"], z[f"{name}_words"], z[f"{name}_drop"]
    n_ch = len(z[f"{name}_sv"])
    out = []
    for c, n_ms in enumerate(z[f"{name}_calls"]):
        chans = []
        for ch in range(n_ch):
            sel = np.flatnonzero((ev[:, 0] == c) & (ev[:, 1] == ch))
            chans.append(([(int(ev[i, 3]), tuple(int(w) for w in words[i]), float(ev[i, 4]), float(ev[i, 5]), int(ev[i, 2]))
                           for i in sel], int(drop[c, ch])))
        out.append((int(n_ms), chans))
    return out


def compare_observations(got, want, exact: bool = False) -> tuple[float, float]:
    """got, want: float64 [m, 6] rows of tow, x, y, z, prn count, flags.  Counts and flags must agree exactly, NaNs sit
    in the same places; tow within 1 ulp and ECEF within 1e-4 m (exact: bit for bit).  Returns the largest tow error in
    ulps and the largest ECEF error in metres."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape
    assert np.array_equal(got[:, 4:], want[:, 4:])
    assert np.array_equal(np.isnan(got[:, :4]), np.isnan(want[:, :4]))
    ok = ~np.isnan(want[:, 0])
    if exact:
        assert np.array_equal(got[ok, 0], want[ok, 0])
        pos = ~np.isnan(want[:, 1])
        assert np.array_equal(got[pos, 1:4], want[pos, 1:4])
        return 0.0, 0.0
    ulps = np.abs(got[ok, 0] - want[ok, 0]) / np.spacing(np.abs(want[ok, 0]))
    pos = ~np.isnan(want[:, 1])
    metres = np.abs(got[pos, 1:4] - want[pos, 1:4])
    worst_ulp = float(ulps.max(initial=0.0))
    worst_m = float(metres.max(initial=0.0))
    assert worst_ulp <= 1.0, worst_ulp
    assert worst_m <= 1e-4, worst_m
    return worst_ulp, worst_m
