"""Float64 restatement of the per-channel C/N0 and phase-lock estimator (gypsum_b200/csrc/signal_core.cuh, DESIGN.md
section 8e), for the signal tests.  Every sum runs in millisecond order, one Python float operation at a time, so that
it rounds as the host and device cores do."""
import math

import numpy as np

MIN_MS, MAX_MS = 20, 60000  # the window lengths the estimator accepts; fewer counted records than MIN_MS: status 0
FOUR_OVER_PI = 4.0 / math.pi  # a Rayleigh variable's power over its mean squared
NONE, SIGNAL, NOISE = 0, 1, 2  # SIGNAL_DTYPE["status"]
MARGIN_DB = 1.0

FIELDS = ("receiver_timestamp", "cn0_dbhz", "prompt_power", "noise_power", "pll_lock", "first_ms", "ms_index", "n_ms",
          "locked_ms", "status")


def noise_floor_dbhz(n):
    """The estimate for noise alone at n samples per millisecond: |P|^2 is then the largest of n exponentials, whose
    mean over the noise power is the harmonic number H_n."""
    h = 0.0
    for k in range(1, n + 1):
        h += 1.0 / k
    return 10.0 * math.log10((h - 1.0) / 1e-3)


def planted_cn0_dbhz(amplitude, sigma, fs):
    """C/N0 of a tone of this amplitude in complex noise of variance sigma^2 per sample at fs samples per second."""
    return 10.0 * math.log10(amplitude * amplitude * fs / (sigma * sigma))


def _div(a, b):
    with np.errstate(all="ignore"):
        return float(np.float64(a) / np.float64(b))


def estimate(i2, q2, pn, n, floor_dbhz):
    """(cn0, prompt power, noise power, PLI, status) of a window's sums over n records."""
    m2 = _div(i2 + q2, n)
    noise = FOUR_OVER_PI * _div(pn, n)
    pli = _div(i2 - q2, i2 + q2)
    cn0 = math.nan
    if n < MIN_MS or not (math.isfinite(i2) and math.isfinite(q2) and math.isfinite(pn)):
        status = NONE
    elif m2 > noise:
        cn0 = 10.0 * math.log10(_div(m2 - noise, noise * 1e-3))
        status = SIGNAL if cn0 >= floor_dbhz + MARGIN_DB else NOISE
    else:
        status = NOISE
    return cn0, m2, noise, pli, status


class SignalOracle:
    """One channel's estimator, kept across calls like the device's."""

    def __init__(self, window_ms, floor_dbhz):
        self.w, self.floor = int(window_ms), float(floor_dbhz)
        self.i2 = self.q2 = self.pn = 0.0
        self.n = self.locked = 0
        self.t0 = 0.0
        self.consumed = 0
        self.stopped = False

    def _emit(self, ms_index):
        cn0, m2, noise, pli, status = estimate(self.i2, self.q2, self.pn, self.n, self.floor)
        row = (self.t0, cn0, m2, noise, pli, self.consumed - self.n, ms_index, self.n, self.locked, status)
        self.i2 = self.q2 = self.pn = 0.0
        self.n = self.locked = 0
        return row

    def feed(self, peak_re, peak_im, strength, locked, lost, start_times):
        """One call over its records' fields (prompt I and Q and strength as float32, then float64): a list of window
        rows in FIELDS order."""
        out = []
        if self.stopped:
            return out
        for k in range(len(start_times)):
            if lost[k]:
                if self.n:
                    out.append(self._emit(k - 1))
                self.stopped = True
                break
            if self.n == 0:
                self.t0 = float(start_times[k])
            i, q, s = float(np.float32(peak_re[k])), float(np.float32(peak_im[k])), float(np.float32(strength[k]))
            i2, q2 = i * i, q * q
            self.i2 += i2
            self.q2 += q2
            self.pn += _div(i2 + q2, s * s)
            self.n += 1
            self.locked += 1 if locked[k] else 0
            self.consumed += 1
            if self.n == self.w:
                out.append(self._emit(k))
        return out


def windows_of_rows(rows, lost_at, window_ms, floor_dbhz, start_times):
    """The windows of one golden tracker file's rows (columns 0-2: prompt I, Q and strength) in one call; the row at
    lost_at (>= 0) is lost."""
    n = len(start_times)
    re, im, st = (np.zeros(n) for _ in range(3))
    m = min(n, len(rows))
    re[:m], im[:m], st[:m] = rows[:m, 0], rows[:m, 1], rows[:m, 2]
    lost = np.zeros(n, dtype=np.int32)
    if lost_at >= 0:
        lost[lost_at] = 1
    return SignalOracle(window_ms, floor_dbhz).feed(re, im, st, np.zeros(n, np.int32), lost, start_times)
