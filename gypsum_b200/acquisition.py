"""Drop-in for reference gypsum/acquisition.py: GpsSatelliteDetector and its result records.

Same class, method names, arguments and selection semantics (acquisition.py:52-190); the per-bin correlation
work of every requested satellite is batched into one GPU call per refinement pass instead of one numpy
evaluation per (satellite, bin).
"""
from __future__ import annotations

import logging
import math
from dataclasses import dataclass

import numpy as np

from gypsum_b200 import _native
from gypsum_b200.constants import ACQUISITION_INTEGRATED_CORRELATION_STRENGTH_DETECTION_THRESHOLD
from gypsum_b200.utils import POOL, IntegrationType, _kind, chips_of_satellite

_logger = logging.getLogger(__name__)


@dataclass
class BestNonCoherentCorrelationProfile:  # acquisition.py:25-32
    doppler_shift: float
    non_coherent_correlation_profile: np.ndarray
    sample_offset_of_correlation_peak: int
    correlation_strength: float


@dataclass
class SatelliteAcquisitionAttemptResult:  # acquisition.py:35-41
    satellite_id: object
    doppler_shift: float
    carrier_wave_phase_shift: float
    prn_phase_shift: int
    correlation_strength: float


def code_shift(ms, n: int, doppler_hz):
    """The weak grid's realignment of millisecond ms (from the block's first) at Doppler f, in samples: rint(ms * N * f /
    f_L1), evaluated in the engine's order (kernels.cuh code_shift).  A closing satellite's code lag at that millisecond is
    its lag at the first sample minus this."""
    return np.rint(np.float64(ms) * n * np.asarray(doppler_hz, dtype=np.float64) / 1575.42e6)


def doppler_search_bins(center: float, spread: float) -> range:
    """acquisition.py:163-167: int() truncates toward zero, the upper end is excluded."""
    return range(int(center - spread), int(center + spread), int(spread / 10))


@dataclass
class _Best:
    doppler: int
    peak_index: int
    strength: float


class GpsSatelliteDetector:
    def __init__(self, satellites_by_id: dict) -> None:
        self.satellites_by_id = satellites_by_id
        self._chips_cache: dict = {}

    # -- helpers ---------------------------------------------------------------------------------------------
    def _chips(self, satellite_id, n: int) -> np.ndarray:
        key = (getattr(satellite_id, "id", satellite_id), n)
        c = self._chips_cache.get(key)
        if c is None:
            c = self._chips_cache[key] = chips_of_satellite(self.satellites_by_id[satellite_id], n)
        return c

    def _prepare(self, satellite_ids, antenna_data, stream_attributes):
        fs = int(stream_attributes.samples_per_second)
        n = int(stream_attributes.samples_per_prn_transmission)
        ent = POOL.get(fs, n)
        idx = POOL.ensure_table(ent, [self._chips(s, n) for s in satellite_ids])
        eng = ent["engine"]
        if hasattr(antenna_data, "bind") and hasattr(antenna_data, "n_ms"):
            # antenna_sample_provider.DeviceWindow: the samples are already on the device (receiver.py:219 without the copy)
            n_ms = int(antenna_data.n_ms)
            if n_ms == 0:
                raise ValueError("need at least one whole millisecond of samples")
            antenna_data.bind()
            return eng, idx, n, n_ms
        data = np.ascontiguousarray(antenna_data, dtype=np.complex64)
        n_ms = data.size // n
        if n_ms == 0:
            raise ValueError("need at least one whole millisecond of samples")
        eng.upload_iq(data[: n_ms * n])
        return eng, idx, n, n_ms

    @staticmethod
    def _scan(eng, prn_idx, centers, spread, n, n_ms) -> list[_Best]:
        """One refinement pass for every satellite at once (acquisition.py:154-190 per satellite)."""
        cell_prn, cell_dop, spans = [], [], []
        for p, c in zip(prn_idx, centers):
            bins = list(doppler_search_bins(c, spread))
            spans.append((len(cell_prn), len(bins)))
            cell_prn.extend([p] * len(bins))
            cell_dop.extend(bins)
        rec = eng.acquire_cells(cell_prn, cell_dop, n_ms, _native.NON_COHERENT)
        strength = _native.strength_from_records(rec, n)
        out = []
        for first, count in spans:
            peaks = rec["peak"][first:first + count]
            k = first + int(np.argmax(peaks))  # first bin with the largest np.max(profile), acquisition.py:180-182
            out.append(_Best(int(cell_dop[k]), int(rec["argmax"][k]), float(strength[k])))
        return out

    def _acquire_many(self, satellite_ids, antenna_data, stream_attributes) -> list[SatelliteAcquisitionAttemptResult]:
        """acquisition.py:70-152 for a batch of satellites: one gb200_detect call -- the ten refinement passes, the
        bin selection between them and the final coherent integration all run on the device."""
        if not satellite_ids:
            return []
        eng, prn_idx, n, n_ms = self._prepare(satellite_ids, antenna_data, stream_attributes)
        rec = eng.detect(prn_idx, n_ms)
        phase = np.angle(rec["probe_re"].astype(np.float64) + 1j * rec["probe_im"].astype(np.float64))
        return [
            SatelliteAcquisitionAttemptResult(
                satellite_id=sid, doppler_shift=int(rec["doppler"][i]), carrier_wave_phase_shift=phase[i],
                prn_phase_shift=int(rec["code_phase"][i]), correlation_strength=float(rec["strength"][i]),
            )
            for i, sid in enumerate(satellite_ids)
        ]

    def _acquire_many_stepwise(self, satellite_ids, antenna_data, stream_attributes) -> list[SatelliteAcquisitionAttemptResult]:
        """The same search driven pass by pass from the host (one gb200_acquire_cells call per pass); kept as the
        cross-check of the on-device driver and for callers that want to observe the passes."""
        if not satellite_ids:
            return []
        eng, prn_idx, n, n_ms = self._prepare(satellite_ids, antenna_data, stream_attributes)
        centers = [0.0] * len(satellite_ids)
        kept: list[_Best | None] = [None] * len(satellite_ids)
        spread = 7000.0
        while spread >= 10:
            found = self._scan(eng, prn_idx, centers, spread, n, n_ms)
            spread /= 2
            for i, b in enumerate(found):
                centers[i] = b.doppler
                if kept[i] is None or b.strength > kept[i].strength:
                    kept[i] = b
        # one coherent integration per satellite at the kept Doppler; phase at the non-coherent peak index
        rec = eng.acquire_cells(prn_idx, [k.doppler for k in kept], n_ms, _native.COHERENT,
                                probe_idx=[k.peak_index for k in kept])
        phase = np.angle(rec["probe_re"].astype(np.float64) + 1j * rec["probe_im"].astype(np.float64))
        return [
            SatelliteAcquisitionAttemptResult(
                satellite_id=sid, doppler_shift=k.doppler, carrier_wave_phase_shift=phase[i],
                prn_phase_shift=k.peak_index, correlation_strength=k.strength,
            )
            for i, (sid, k) in enumerate(zip(satellite_ids, kept))
        ]

    def acquire_weak_satellites(self, satellite_ids, antenna_data, stream_attributes, coherent_ms: int,
                                doppler_spread: float = 7000.0, doppler_step: float | None = None
                                ) -> list[SatelliteAcquisitionAttemptResult]:
        """Semi-coherent acquisition for satellites too weak for the reference's search: over the whole window (uploaded
        samples or a DeviceSampleRing window, a whole number of coherent_ms-ms segments), every satellite's profile
        sum_k |coherent sum of segment k| on the Doppler bins arange(-spread, spread + step / 2, step), step 500 /
        coherent_ms Hz by default, in one gb200_acquire_grid_semicoherent_best call.  Then one coherent integration of
        the first coherent_ms milliseconds at each satellite's best bin gives the carrier phase at its code phase.

        One result per satellite, NOT thresholded: the reference's strength threshold was set for its own statistic.
        Keep coherent_ms within a navigation data bit (20 ms): a bit edge inside a segment cancels part of it."""
        if isinstance(coherent_ms, bool) or int(coherent_ms) != coherent_ms or coherent_ms < 1:
            raise ValueError(f"coherent_ms must be a positive whole number of milliseconds (got {coherent_ms!r})")
        coherent_ms = int(coherent_ms)
        spread = float(doppler_spread)
        step = 500.0 / coherent_ms if doppler_step is None else float(doppler_step)
        if not (np.isfinite(spread) and spread >= 0.0):
            raise ValueError(f"doppler_spread must be finite and >= 0 (got {doppler_spread!r})")
        if not (np.isfinite(step) and step > 0.0):
            raise ValueError(f"doppler_step must be finite and > 0 (got {doppler_step!r})")
        if not satellite_ids:
            return []
        satellite_ids = list(satellite_ids)
        eng, prn_idx, n, n_ms = self._prepare(satellite_ids, antenna_data, stream_attributes)
        bins = np.arange(-spread, spread + step / 2, step)
        best = eng.acquire_grid_semicoherent_best(1, n_ms, coherent_ms, prn_idx, bins)[0]
        rec = eng.acquire_cells(prn_idx, best["doppler"], coherent_ms, _native.COHERENT, probe_idx=best["code_phase"])
        phase = np.angle(rec["probe_re"].astype(np.float64) + 1j * rec["probe_im"].astype(np.float64))
        return [
            SatelliteAcquisitionAttemptResult(
                satellite_id=sid, doppler_shift=float(best["doppler"][i]), carrier_wave_phase_shift=float(phase[i]),
                prn_phase_shift=int(best["code_phase"][i]), correlation_strength=float(best["strength"][i]),
            )
            for i, sid in enumerate(satellite_ids)
        ]

    def search_weak_satellites(self, satellite_ids, antenna_data, stream_attributes, coherent_ms: int = 20,
                               bit_phases: int = 4, doppler_spread: float = 7000.0, doppler_step: float | None = None
                               ) -> list[SatelliteAcquisitionAttemptResult]:
        """Weak-signal acquisition through navigation data bits and code Doppler: every satellite's semi-coherent profile
        (segments of coherent_ms ms) at each of bit_phases segment offsets coherent_ms / bit_phases ms apart, with each
        millisecond realigned by its code Doppler, on the Doppler bins arange(-spread, spread + step / 2, step) (step
        500 / coherent_ms Hz by default), in one gb200_acquire_grid_weak_best call.  The window (uploaded samples or a
        DeviceSampleRing window) is trimmed to the longest one the bit phases cover with whole segments.  Then one coherent
        integration over the first segment of each satellite's best bit phase, which lies inside one data bit, gives the
        carrier phase at its code phase, referred back to the window's first sample (modulo pi: the bit's sign is unknown).

        One result per satellite, NOT thresholded: the reference's strength threshold was set for its own statistic."""
        for name, v in (("coherent_ms", coherent_ms), ("bit_phases", bit_phases)):
            if isinstance(v, bool) or int(v) != v or v < 1:
                raise ValueError(f"{name} must be a positive whole number (got {v!r})")
        coherent_ms, bit_phases = int(coherent_ms), int(bit_phases)
        if coherent_ms % bit_phases:
            raise ValueError(f"bit_phases ({bit_phases}) must divide coherent_ms ({coherent_ms})")
        spread = float(doppler_spread)
        step = 500.0 / coherent_ms if doppler_step is None else float(doppler_step)
        if not (np.isfinite(spread) and spread >= 0.0):
            raise ValueError(f"doppler_spread must be finite and >= 0 (got {doppler_spread!r})")
        if not (np.isfinite(step) and step > 0.0):
            raise ValueError(f"doppler_step must be finite and > 0 (got {doppler_step!r})")
        if not satellite_ids:
            return []
        satellite_ids = list(satellite_ids)
        eng, prn_idx, n, n_ms = self._prepare(satellite_ids, antenna_data, stream_attributes)
        delta = coherent_ms // bit_phases
        k = (n_ms - (bit_phases - 1) * delta) // coherent_ms
        if k < 1:
            raise ValueError(f"a {n_ms}-ms window holds no {coherent_ms}-ms segment at each of {bit_phases} bit phases "
                             f"(needs {coherent_ms + (bit_phases - 1) * delta} ms)")
        bins = np.arange(-spread, spread + step / 2, step)
        best = eng.acquire_grid_weak_best(1, k * coherent_ms + (bit_phases - 1) * delta, coherent_ms, bit_phases, prn_idx,
                                          bins)[0]
        phase_of = best["bin"] // bins.size
        phase = np.zeros(len(satellite_ids))
        on_device = hasattr(antenna_data, "bind")
        for j in np.unique(phase_of):
            first = int(j) * delta  # the phase's first segment: milliseconds first .. first + coherent_ms - 1
            if first and on_device:
                antenna_data.ring.native.bind_newest(n_ms - first)
            elif first:
                eng.upload_iq(np.ascontiguousarray(antenna_data, dtype=np.complex64)[first * n:(first + coherent_ms) * n])
            sel = np.flatnonzero(phase_of == j)
            f = best["doppler"][sel]
            # the code phase at the segment's first sample, where the probe's correlation peaks
            probe = (best["code_phase"][sel] - code_shift(first, n, f).astype(np.int64)) % n
            rec = eng.acquire_cells(np.asarray(prn_idx)[sel], f, coherent_ms, _native.COHERENT, probe_idx=probe)
            z = rec["probe_re"].astype(np.float64) + 1j * rec["probe_im"].astype(np.float64)
            phase[sel] = np.angle(z * np.exp(-1j * math.tau * f * first * 1e-3))
        return [
            SatelliteAcquisitionAttemptResult(
                satellite_id=sid, doppler_shift=float(best["doppler"][i]), carrier_wave_phase_shift=float(phase[i]),
                prn_phase_shift=int(best["code_phase"][i]), correlation_strength=float(best["strength"][i]),
            )
            for i, sid in enumerate(satellite_ids)
        ]

    # -- the reference's methods ---------------------------------------------------------------------------------
    def detect_satellites_in_antenna_data(self, satellites_to_search_for, antenna_data, stream_attributes):
        """acquisition.py:52-68."""
        results = self._acquire_many(list(satellites_to_search_for), antenna_data, stream_attributes)
        detected = []
        for r in results:
            if r.correlation_strength > ACQUISITION_INTEGRATED_CORRELATION_STRENGTH_DETECTION_THRESHOLD:
                _logger.info(f"Correlation strength above threshold, successfully detected satellite {r.satellite_id}!")
                detected.append(r)
        return detected

    def _attempt_acquisition_for_satellite_id(self, satellite_id, samples_for_integration_period, stream_attributes):
        """acquisition.py:70-152."""
        return self._acquire_many([satellite_id], samples_for_integration_period, stream_attributes)[0]

    def get_best_doppler_shift_estimation(self, center_doppler_shift, doppler_shift_spread, antenna_data,
                                          stream_attributes, satellite_id) -> BestNonCoherentCorrelationProfile:
        """acquisition.py:154-190, including the full profile of the winning bin."""
        eng, idx, n, n_ms = self._prepare([satellite_id], antenna_data, stream_attributes)
        b = self._scan(eng, idx, [center_doppler_shift], doppler_shift_spread, n, n_ms)[0]
        prof = eng.correlation_profile(idx[0], b.doppler, n_ms, _native.NON_COHERENT).astype(np.float64)
        return BestNonCoherentCorrelationProfile(b.doppler, prof, b.peak_index, b.strength)

    def get_integrated_correlation_with_doppler_shifted_prn(self, integration_type, antenna_data, stream_attributes,
                                                            doppler_shift, prn_as_complex) -> np.ndarray:
        """acquisition.py:192-219 minus its write-only memo (cache read is disabled at :205; nothing is kept here)."""
        from gypsum_b200.utils import integrate_correlation_with_doppler_shifted_prn

        return integrate_correlation_with_doppler_shifted_prn(integration_type, antenna_data, stream_attributes,
                                                              doppler_shift, prn_as_complex)


__all__ = ["GpsSatelliteDetector", "SatelliteAcquisitionAttemptResult", "BestNonCoherentCorrelationProfile",
           "IntegrationType", "doppler_search_bins"]
_ = _kind  # re-exported for callers that translate enums
