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
        self.rows = {}
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
