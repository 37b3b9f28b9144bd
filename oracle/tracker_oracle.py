"""CPU oracle (numpy, float64) for the tracking loop of gypsum/tracker.py.  TEST INFRASTRUCTURE -- see
oracle/__init__.py.  Pinned against the live reference tracker through tests/golden/tracker_*.npz
(tools/make_golden_tracker.py)."""
from __future__ import annotations

import collections
import math

import numpy as np

from oracle.gypsum_oracle import correlate_1ms, peak_strength, replica


class LostLock(Exception):
    """tracker.py:33 LostSatelliteLockError."""


def constellation_rotation(peaks: np.ndarray):
    """utils.py:119-131."""
    left = peaks[peaks.real < 0]
    if len(left) < 2:
        return None
    m = np.mean(left)
    angle = 180 - (((np.arctan2(m.imag, m.real) / math.tau) * 360) % 180)
    return angle - 180 if angle > 90 else angle


def constellation_circularity(peaks: np.ndarray):
    """utils.py:134-144: 1 - min/max eigenvalue of the 2x2 sample covariance of (I, Q)."""
    if len(peaks) < 2:
        return None
    ev, _ = np.linalg.eig(np.cov(np.real(peaks), np.imag(peaks)))
    return 1 - (min(ev) / max(ev))


class TrackerOracle:
    """One channel.  Mirrors GpsSatelliteTracker + GpsSatelliteTrackingParameters (tracker.py:117-389)."""

    def __init__(self, sv: int, doppler: float, carrier_phase: float, code_phase: int, fs: int, n: int):
        self.prn = replica(sv, n)
        self.fs, self.n = fs, n
        self.doppler, self.carrier_phase, self.code_phase = float(doppler), float(carrier_phase), int(code_phase)
        self.phase = code_phase  # tracker.py:224
        self.t1ms = np.arange(n) / fs  # tracker.py:217-219
        self.errors = collections.deque(maxlen=5000)  # tracker.py:153
        self.peaks = collections.deque(maxlen=1000)  # tracker.py:149
        self.last_circularity_check = 0.0  # tracker.py:222

    def is_locked(self) -> bool:
        """tracker.py:157-203."""
        if len(self.errors) < 250:
            return False
        err = np.array(list(self.errors)[-250:])
        var_ok = np.var(err) < 900
        i_ok, rot_ok = True, True
        last = np.array(list(self.peaks)[-250:])
        if len(self.peaks) > 2:
            neg, pos = last[last.real < 0], last[last.real >= 0]
            mean_neg = np.mean(neg) if len(neg) >= 2 else 0
            nv = np.var(neg.real) if len(neg) >= 2 else 0
            pv = np.var(pos.real) if len(pos) >= 2 else 0
            i_ok = (nv + pv) / 2.0 < 2
            angle = 180 - (((np.arctan2(mean_neg.imag, mean_neg.real) / math.tau) * 360) % 180)
            centered = angle if angle < 90 else 180 - angle
            rot_ok = bool(centered < 6)  # tracker.py:197 abs(bool)
        return bool(var_ok and i_ok and rot_ok)

    def step(self, samples: np.ndarray, start_time: float, end_time: float) -> dict:
        """tracker.py:331-389 (process_samples) including :264-329 and :246-262."""
        t = self.t1ms + start_time
        y = samples * np.exp(-1j * ((2 * np.pi * self.doppler * t) + self.carrier_phase))
        p0 = self.code_phase
        # tracker.py:293-295: np.correlate (mode 'valid', equal lengths) = one dot product sum y * conj(replica)
        early = np.correlate(y, np.roll(self.prn, p0 - 1))[0]
        late = np.correlate(y, np.roll(self.prn, p0 + 1))[0]
        disc = ((early.real ** 2 + early.imag ** 2) - (late.real ** 2 + late.imag ** 2)) / 2
        self.phase += disc * 0.002
        self.code_phase = int(self.phase)
        self.phase %= 2046
        coh = correlate_1ms(y, np.roll(self.prn, p0))
        nc = np.abs(coh)
        k = int(np.argmax(nc))
        strength = float(peak_strength(nc))
        peak = complex(coh[k])
        symbol = int(np.sign(peak.real))
        delay = (self.code_phase / 2046) * 0.001
        self.peaks.append(peak)
        error = peak.real * peak.imag
        locked = self.is_locked()
        bw = 3 if locked else 6
        ts = 1.0 / self.fs
        alpha, beta = 4 * (1.0 / math.sqrt(2)) * bw * ts, 4 * (bw ** 2) * ts
        self.carrier_phase += error * alpha
        self.carrier_phase %= math.tau
        self.doppler += error * beta
        self.errors.append(error)
        out = dict(peak=peak, strength=strength, symbol=symbol, error=error, disc=float(disc), locked=locked,
                   code_phase=self.code_phase, start=start_time + delay, end=end_time + delay, early=complex(early),
                   late=complex(late), peak_offset=k,
                   # tracker.py:352-353 appends the loop state to the histories BEFORE the 6-second adjustment below
                   doppler_hist=self.doppler, carrier_phase_hist=self.carrier_phase)
        if start_time - self.last_circularity_check >= 6:  # tracker.py:370-387
            self.last_circularity_check = start_time
            pk = np.array(self.peaks)
            circ = constellation_circularity(pk)
            if circ is not None:
                if circ < 0.2:
                    raise LostLock(out)  # carries this millisecond's correlator outputs for the tests
                if circ < 0.93:
                    rot = constellation_rotation(pk)
                    if rot is not None:
                        self.doppler += -np.sign(rot) * 5
                        self.carrier_phase += np.sign(rot) * (math.pi / 2)
        out.update(doppler=self.doppler, carrier_phase=self.carrier_phase)
        return out


def synth_tracking_iq(seed: int, n: int, n_ms: int, fs: int, channels, sigma: float = 0.02, t0: float = 0.0) -> np.ndarray:
    """SURVEY.md 8d / F11: noise sigma per sample plus, per channel (sv, doppler_hz, doppler_rate_hz_s, code_phase,
    carrier_phase, amplitude), amplitude * code * data-bit (20 ms, random) * exp(j(2 pi (f t + rate t^2/2) + phi)), the
    first sample at stream time t0."""
    rng = np.random.default_rng(seed)
    total = n * n_ms
    x = (rng.standard_normal(total) + 1j * rng.standard_normal(total)) * (sigma / math.sqrt(2.0))
    t = np.arange(total) / fs + t0
    for sv, f, rate, tau_s, phi, amp in channels:
        code = np.tile(np.roll(replica(sv, n).real, tau_s), n_ms)
        bits = rng.integers(0, 2, size=n_ms // 20 + 2) * 2 - 1
        offset = int(rng.integers(0, 20))
        data = np.repeat(bits, 20 * n)[offset * n: offset * n + total]
        x = x + amp * code * data * np.exp(1j * (math.tau * (f * t + 0.5 * rate * t * t) + phi))
    return x.astype(np.complex64)


def chunk_times(k: int, fs: int, n: int):
    """antenna_sample_provider.py:88-89,120-124: timestamps are round(cursor / fs, 6)."""
    return round(k * n / fs, 6), round((k + 1) * n / fs, 6)
