"""CPU oracle of the position fix's least-squares mode (gb200_tracker_set_fix_solver), on top of oracle/fix_oracle.py,
whose reference path it leaves alone.  Where five or more satellites are ready the reference's np.linalg.solve raises;
this mode runs the same _compute_position over all of them with np.linalg.lstsq(J, -r) in place of solve (Gauss-Newton)
and goes on.  Four ready rows take fx.compute_position unchanged.  TEST INFRASTRUCTURE, like the oracle package."""
from __future__ import annotations

import math

import numpy as np

from oracle import fix_oracle as fx
from oracle import nav_oracle as nav
from oracle import orbit_oracle as orb


def compute_position(rows, receiver_timestamp, slide, info=None):
    """fx.compute_position for four rows; for more, the same rounds and iterations with each step the least-squares
    solution.  Raises np.linalg.LinAlgError with `.slide` where lstsq reports rank < 4 (its default rcond).  info: an
    optional dict that receives "last_step", the largest component of the last iteration's step (metres / seconds)."""
    if len(rows) == 4:
        return fx.compute_position(rows, receiver_timestamp, slide)
    sx = [r[1] for r in rows]
    sy = [r[2] for r in rows]
    sz = [r[3] for r in rows]
    gx = gy = gz = 0
    cb = 0
    pr0 = None

    def residuals(ts):
        return np.array([((gx - x) ** 2 + (gy - y) ** 2 + (gz - z) ** 2 - ((fx.SPEED_OF_LIGHT * (t - cb)) ** 2))
                         for x, y, z, t in zip(sx, sy, sz, ts)])

    def jacobian(ts):
        return np.array([[2 * (gx - x), 2 * (gy - y), 2 * (gz - z), 2 * (math.pow(fx.SPEED_OF_LIGHT, 2) * (t - cb))]
                         for x, y, z, t in zip(sx, sy, sz, ts)])

    v = None
    for _ in range(5):
        ts = [(slide + receiver_timestamp) - r[0] for r in rows]
        if pr0 is None:
            pr0 = ts
        res, jac = residuals(ts), jacobian(ts)
        for _ in range(20):
            v, _, rank, _ = np.linalg.lstsq(jac, -res, rcond=None)
            if rank < 4:
                err = np.linalg.LinAlgError(f"rank {rank} least-squares system")
                err.slide = slide
                raise err
            gx += v[0]
            gy += v[1]
            gz += v[2]
            cb += v[3]
            res, jac = residuals(ts), jacobian(ts)
        slide -= cb
    if info is not None:
        info["last_step"] = (float(np.abs(v[:3]).max()), float(abs(v[3])))
    return slide, cb, (gx, gy, gz), pr0[:4]


class ReceiverOracle(fx.ReceiverOracle):
    """fx.ReceiverOracle in the least-squares mode: five or more ready satellites are fixed instead of raising; only a
    singular four-row system or a rank-deficient larger one stops the receiver.  self.rows holds all ready rows."""

    def call(self, chans, receiver_timestamps, teacher=None, sample=None) -> np.ndarray:
        """As fx.ReceiverOracle.call (the same receiver order, drops, resets, teacher and sample)."""
        n_ms = len(receiver_timestamps)
        by = [{} for _ in chans]
        for ch, (events, _) in enumerate(chans):
            for kind, w, te, m in events:
                by[ch].setdefault(m, []).append((kind, w, te))
        drops = [d for _, d in chans]
        tracked = [True] * len(chans)
        self.rows, self.resets = {}, {}
        out = np.zeros(n_ms, dtype=fx.FIX_DTYPE)
        for m in range(n_ms):
            f = out[m]
            f["receiver_timestamp"] = receiver_timestamps[m]
            for k in ("slide_in", "slide_out", "clock_bias", "x", "y", "z", "pseudorange"):
                f[k] = np.nan
            f["channel"] = -1
            if not self.stopped and any(tracked[ch] and m != drops[ch] and not self.sats[ch].frozen
                                        and any(k == nav.KIND_RAISED for k, _, _ in by[ch].get(m, ()))
                                        for ch in range(len(chans))):
                self.stopped = True
            if self.stopped:
                f["status"] = fx.FIX_STOPPED
                continue
            for ch, d in enumerate(drops):
                if m == d and tracked[ch]:
                    self.sats[ch].lost()
                    self._touch(ch)
                    tracked[ch] = False
            for ch in range(len(chans)):
                if tracked[ch]:
                    self.sats[ch].prn_observed()
            for ch in range(len(chans)):
                if tracked[ch]:
                    for kind, w, te in by[ch].get(m, ()):
                        if kind == nav.KIND_SUBFRAME:
                            fields = orb.parse(w)
                            self._touch(ch)
                            self.sats[ch].subframe(fields, te)
                            self.slide = fields["tow_seconds"] - te
                            self.resets[m] = self.slide
            ready = [ch for ch in self.order if self._ready(ch)]
            f["n_ready"] = len(ready)
            f["channel"][:min(4, len(ready))] = ready[:4]
            if len(ready) < 4 or self.slide is None:
                f["status"] = fx.FIX_NONE
                continue
            if teacher is not None:
                self.slide = float(teacher[m]["slide_in"])
            f["slide_in"] = self.slide
            if teacher is not None and sample is not None and m not in sample:
                f["status"] = fx.FIX_SOLVED
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
                f["status"] = fx.FIX_RAISED
                f["slide_out"] = self.slide = err.slide
                self.stopped = True
                continue
            self.slide = slide
            f["status"] = fx.FIX_SOLVED
            f["slide_out"], f["clock_bias"], f["x"], f["y"], f["z"] = slide, cb, *pos
            f["pseudorange"] = pr
        return out


def device_passes(compute, rec, rows, resets, carried):
    """fx.device_passes in the least-squares mode: every fixing millisecond, five or more rows included, goes through
    compute(rows, receiver_timestamp, slide) with all of its rows."""
    four = rec.copy()
    four["n_ready"] = np.minimum(four["n_ready"], 4)  # fx.device_passes raises above four without calling compute
    return fx.device_passes(compute, four, rows, resets, carried)
