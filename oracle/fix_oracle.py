"""CPU oracle for the world model's position fix (gypsum/world_model.py:489-633, :749-752; receiver.py:106-137): one
receiver over several channels, millisecond by millisecond in the receiver's order, on top of oracle/orbit_oracle.py.
It calls np.linalg.solve as the reference does, so it equals the reference bit for bit.
TEST INFRASTRUCTURE -- see oracle/__init__.py.  Pinned against the live reference through tests/golden/fix.npz
(tools/make_golden_fix.py)."""
from __future__ import annotations

import math

import numpy as np

from oracle import nav_oracle as nav
from oracle import orbit_oracle as orb

SPEED_OF_LIGHT = 2.99792458e8  # constants.py:35
FIX_NONE, FIX_SOLVED, FIX_RAISED, FIX_STOPPED = 0, 1, 2, 3
FIX_DTYPE = np.dtype([  # the layout of gb200_position_fix
    ("receiver_timestamp", "<f8"), ("slide_in", "<f8"), ("slide_out", "<f8"), ("clock_bias", "<f8"), ("x", "<f8"),
    ("y", "<f8"), ("z", "<f8"), ("pseudorange", "<f8", (4,)), ("status", "<i4"), ("n_ready", "<i4"),
    ("channel", "<i4", (4,))])


def compute_position(rows, receiver_timestamp, slide):
    """_compute_position (:591-633) on rows [(tow, x, y, z)] from the entering slide, as written: returns (slide after,
    clock bias, (x, y, z), round 0's pseudoranges).  Raises np.linalg.LinAlgError where the reference does; the error
    carries the slide at that point in `.slide`."""
    sx = [r[1] for r in rows]
    sy = [r[2] for r in rows]
    sz = [r[3] for r in rows]
    gx = gy = gz = 0  # EcefCoordinates.zero()
    cb = 0
    pr0 = None

    def residuals(ts):
        return np.array([((gx - x) ** 2 + (gy - y) ** 2 + (gz - z) ** 2 - ((SPEED_OF_LIGHT * (t - cb)) ** 2))
                         for x, y, z, t in zip(sx, sy, sz, ts)])

    def jacobian(ts):
        return np.array([[2 * (gx - x), 2 * (gy - y), 2 * (gz - z), 2 * (math.pow(SPEED_OF_LIGHT, 2) * (t - cb))]
                         for x, y, z, t in zip(sx, sy, sz, ts)])

    for _ in range(5):
        ts = [(slide + receiver_timestamp) - r[0] for r in rows]  # get_pseudorange_for_satellite
        if pr0 is None:
            pr0 = ts
        res, jac = residuals(ts), jacobian(ts)
        for _ in range(20):
            try:
                v = np.linalg.solve(jac, -res)
            except np.linalg.LinAlgError as err:
                err.slide = slide
                raise
            gx += v[0]
            gy += v[1]
            gz += v[2]
            cb += v[3]
            res, jac = residuals(ts), jacobian(ts)
        slide -= cb
    return slide, cb, (gx, gy, gz), pr0


class ReceiverOracle:
    """One receiver: a GpsWorldModel entry per channel (one satellite per channel), its clock slide, the order in
    which satellites entered satellite_ids_to_orbital_parameters, and whether its step has raised."""

    def __init__(self, n_channels: int):
        self.sats = [orb.OrbitOracle() for _ in range(n_channels)]
        self.slide = None
        self.order: list[int] = []
        self.stopped = False
        self.rows: dict = {}  # ms of the last call -> the rows [(tow, x, y, z)] of its fix
        self.resets: dict = {}  # ms of the last call -> the slide its subframes set

    def _touch(self, ch: int) -> None:
        if ch not in self.order:
            self.order.append(ch)

    def _ready(self, ch: int) -> bool:
        s = self.sats[ch]
        return all(v is not None for v in s.p) and s.counting and s.count <= 6000

    def call(self, chans, receiver_timestamps, teacher=None, sample=None) -> np.ndarray:
        """chans: per channel (events [(kind, words, trailing_edge, ms)] in ms order, drop ms or -1).  One FIX_DTYPE
        record per millisecond.  teacher: optional records (FIX_DTYPE) whose slide_in replaces the chain's at every
        fixing millisecond, so that each fix starts from the same slide as the record's; with it, `sample` (a set of
        ms) limits the solves to those milliseconds, and elsewhere a fix is only classified and the chain takes the
        teacher's slide_out."""
        n_ms = len(receiver_timestamps)
        by = [{} for _ in chans]
        for ch, (events, _) in enumerate(chans):
            for kind, w, te, m in events:
                by[ch].setdefault(m, []).append((kind, w, te))
        drops = [d for _, d in chans]
        tracked = [True] * len(chans)
        self.rows, self.resets = {}, {}
        out = np.zeros(n_ms, dtype=FIX_DTYPE)
        for m in range(n_ms):
            f = out[m]
            f["receiver_timestamp"] = receiver_timestamps[m]
            for k in ("slide_in", "slide_out", "clock_bias", "x", "y", "z", "pseudorange"):
                f[k] = np.nan
            f["channel"] = -1
            # a decoder raise (event kind 3) of a tracked channel: the step never returns, nothing of m happens
            if not self.stopped and any(tracked[ch] and m != drops[ch] and not self.sats[ch].frozen
                                        and any(k == nav.KIND_RAISED for k, _, _ in by[ch].get(m, ()))
                                        for ch in range(len(chans))):
                self.stopped = True
            if self.stopped:
                f["status"] = FIX_STOPPED
                continue
            for ch, d in enumerate(drops):  # receiver.py:254-255, after every pipeline has run
                if m == d and tracked[ch]:
                    self.sats[ch].lost()
                    self._touch(ch)
                    tracked[ch] = False
            for ch in range(len(chans)):  # :110-115
                if tracked[ch]:
                    self.sats[ch].prn_observed()
            for ch in range(len(chans)):  # :120-124, channel by channel, each in event order
                if tracked[ch]:
                    for kind, w, te in by[ch].get(m, ()):
                        if kind == nav.KIND_SUBFRAME:
                            fields = orb.parse(w)
                            self._touch(ch)
                            self.sats[ch].subframe(fields, te)
                            self.slide = fields["tow_seconds"] - te  # world_model.py:749-752
                            self.resets[m] = self.slide
            ready = [ch for ch in self.order if self._ready(ch)]
            f["n_ready"] = len(ready)
            f["channel"][:min(4, len(ready))] = ready[:4]
            if len(ready) < 4 or self.slide is None:
                f["status"] = FIX_NONE
                continue
            if teacher is not None:
                self.slide = float(teacher[m]["slide_in"])
            f["slide_in"] = self.slide
            if len(ready) > 4:  # np.linalg.solve on a non-square system raises before anything changes
                f["status"] = FIX_RAISED
                f["slide_out"] = self.slide
                self.stopped = True
                continue
            if teacher is not None and sample is not None and m not in sample:
                f["status"] = FIX_SOLVED
                self.slide = float(teacher[m]["slide_out"])
                continue
            rows = []
            for ch in ready:
                tow, _ = self.sats[ch].time_of_week()
                rows.append((tow, *self.sats[ch].position(tow)))
            self.rows[m] = rows
            try:
                slide, cb, pos, pr = compute_position(rows, receiver_timestamps[m], self.slide)
            except np.linalg.LinAlgError as err:
                f["status"] = FIX_RAISED
                f["slide_out"] = self.slide = err.slide
                self.stopped = True
                continue
            self.slide = slide
            f["status"] = FIX_SOLVED
            f["slide_out"], f["clock_bias"], f["x"], f["y"], f["z"] = slide, cb, *pos
            f["pseudorange"] = pr
        return out


def same_slide(a, b) -> bool:
    """fix_same_slide: the device's chain check, 4 units in the last place."""
    return abs(a - b) <= 4.0 * 2.0 ** -52 * abs(b)


def device_passes(compute, rec, rows, resets, carried):
    """The device's fix kernels (gypsum_b200/csrc/fix.cu) on one call, from the receiver's decisions: rec, rows and
    resets are ReceiverOracle.call's records, .rows and .resets, carried the slide entering the call (None: none), and
    compute(rows, receiver_timestamp, slide) the fix (a FIX_DTYPE record; the host core makes this exact for the
    device).  Pass 1 fixes every millisecond from its segment's slide (the last reset's, or the carried one); pass 2
    from pass 1's slide at the previous fix of the segment (at a reset: the reset value); a pass-2 fix whose slide is
    not within 4 ulp of pass 1's is a miss; from the first miss on, up to the first raise, every fix that does not start
    a segment and whose entering slide is not bit-equal to the slide the fix before it left is fixed again from that
    slide (k_fix_repair).  Fixes after a singular raise, which the device computes and then discards, are not modelled.
    Returns a dict: pass1 and out (ms -> record: pass 1's, and the final one), first_miss / first_raise (None: none),
    repaired (the milliseconds k_fix_repair fixes again) and slide (what the call carries to the next)."""
    fixing = [m for m in range(len(rec)) if rec[m]["status"] in (FIX_SOLVED, FIX_RAISED)]

    def fix(m, s):
        r = rec[m]
        if r["n_ready"] > 4:  # the non-square system: raised before anything changes
            f = r.copy()
            f["status"], f["slide_in"], f["slide_out"] = FIX_RAISED, s, s
            return f
        return compute(rows[m], r["receiver_timestamp"], s)

    seg, prev, prevs, pass1, out = carried, None, {}, {}, {}
    for m in range(len(rec)):
        if m in resets:
            seg, prev = resets[m], None
        if rec[m]["status"] not in (FIX_SOLVED, FIX_RAISED):
            continue
        pass1[m] = fix(m, seg)
        s = seg if prev is None else pass1[prev]["slide_out"]
        out[m] = pass1[m] if s == seg else fix(m, s)
        prevs[m], prev = prev, m
    miss = [m for m in fixing if not same_slide(out[m]["slide_out"], pass1[m]["slide_out"])]
    raised = [m for m in fixing if out[m]["status"] == FIX_RAISED]
    first_miss = miss[0] if miss else None
    first_raise = raised[0] if raised else len(rec)
    repaired = []
    if first_miss is not None:
        last = first_miss
        for m in fixing:
            if m <= first_miss:
                continue
            if m > first_raise:
                break
            s = out[last]["slide_out"]
            if prevs[m] is not None and not out[m]["slide_in"] == s:
                out[m] = fix(m, s)
                repaired.append(m)
                if out[m]["status"] == FIX_RAISED:
                    first_raise = min(first_raise, m)
            last = m
    out = {m: f for m, f in out.items() if m <= first_raise}
    if first_raise < len(rec):
        slide = float(out[first_raise]["slide_out"])
    elif fixing and fixing[-1] >= max(resets, default=-1):
        slide = float(out[fixing[-1]]["slide_out"])
    else:
        slide = resets[max(resets)] if resets else carried
    return {"pass1": pass1, "out": out, "first_miss": first_miss, "repaired": repaired,
            "first_raise": first_raise if first_raise < len(rec) else None, "slide": slide}


def golden_fix_rows(z, name: str, call: int) -> np.ndarray:
    """The recorded fixes of one call: float64 [n_ms, 15] (see tools/make_golden_fix.py)."""
    f = z[f"{name}_fix"]
    return f[f[:, 0] == call]


def golden_calls(z, name: str):
    """[(receiver timestamps, [per channel: ([(kind, words, trailing_edge, ms)], drop_ms)])] of one timeline."""
    out = []
    for c, (n_ms, chans) in enumerate(orb.golden_calls(z, name)):
        rx = golden_fix_rows(z, name, c)[:, 2]
        assert len(rx) == n_ms
        out.append((rx, [([(k, w, te, m) for k, w, _, te, m in events], drop) for events, drop in chans]))
    return out
