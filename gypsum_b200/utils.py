"""Drop-in for the DSP helpers of reference gypsum/utils.py that sit on the correlation path.

Same names, argument order and return types as the reference (utils.py:23-25, :59-73, :77-108, :111-116); the
arithmetic runs on the GPU through the C ABI.  Values come back widened to float64/complex128 like the
reference's, computed in float32 (tolerance: DESIGN.md section 6).
"""
from __future__ import annotations

import math
from enum import Enum, auto

import numpy as np

from gypsum_b200 import _native


class IntegrationType(Enum):  # utils.py:23-25
    Coherent = auto()
    NonCoherent = auto()


def _kind(integration_type) -> int:
    name = getattr(integration_type, "name", None)
    if name == "Coherent":
        return _native.COHERENT
    if name == "NonCoherent":
        return _native.NON_COHERENT
    raise ValueError("Unexpected integration type")  # utils.py:106


class _EnginePool:
    """One engine per (device, fs, N); each keeps a growing table of replica codes keyed by their chips."""

    def __init__(self):
        self._engines = {}

    def get(self, fs: int, n: int, device: int = 0):
        key = (device, int(fs), int(n))
        ent = self._engines.get(key)
        if ent is None:
            ent = {"engine": _native.Engine(fs, n, device), "codes": {}, "table": []}
            self._engines[key] = ent
        return ent

    def replica_index(self, ent, chips: np.ndarray) -> int:
        return self.ensure_table(ent, [chips])[0]

    def ensure_table(self, ent, chips_list) -> list[int]:
        """Register several codes with a single device upload."""
        new = False
        out = []
        for chips in chips_list:
            k = chips.tobytes()
            idx = ent["codes"].get(k)
            if idx is None:
                idx = len(ent["table"])
                ent["table"].append(chips)
                ent["codes"][k] = idx
                new = True
            out.append(idx)
        if new:
            ent["engine"].set_replicas(np.stack(ent["table"]))
        return out


POOL = _EnginePool()


class NotAChipReplica(ValueError):
    """The replica is not chips repeated N/1023 times: the FFT kernels cannot take it, the direct kernel can."""


def chips_of_replica(prn_as_complex: np.ndarray, n: int) -> tuple[np.ndarray, int]:
    """Recover (chips uint8[1023], roll) from a replica of the reference's form
    roll(repeat(+-1 chips, s), roll) (satellite.py:20-31; tracker.py:286 rolls it).  Anything else raises NotAChipReplica
    (a ValueError): the detector and tracker reject it, the public helpers below fall back to the generic kernel."""
    x = np.asarray(prn_as_complex)
    if x.shape != (n,):
        raise ValueError(f"replica must have {n} samples")
    s = n // 1023
    xr = np.real(x)
    if np.any(np.imag(x) != 0) or np.any(np.abs(xr) != 1):
        raise NotAChipReplica("replica must be a +-1 chip sequence (GpsSatellite.prn_as_complex)")
    for p in range(s):
        y = np.roll(xr, -p)
        c = y[::s]
        if np.array_equal(np.repeat(c, s), y):
            return (c > 0).astype(np.uint8), p
    raise NotAChipReplica("replica is not chips repeated samples_per_ms/1023 times")


def chips_of_satellite(satellite, n: int) -> np.ndarray:
    """chips uint8[1023] of a satellite: its PRN code when its replica has n/1023 samples per chip, else recovered from its
    replica (prn_as_complex), which must not be rolled."""
    code = getattr(getattr(satellite, "prn_code", None), "inner", None)
    if code is not None and getattr(satellite, "scale_factor", n // 1023) == n // 1023:
        return np.ascontiguousarray(np.asarray(code) != 0, dtype=np.uint8)
    chips, roll = chips_of_replica(satellite.prn_as_complex, n)
    if roll:
        raise ValueError("satellite replica must not be rolled")
    return chips


def _profile(x: np.ndarray, fs: int, n: int, n_ms: int, prn_replica, doppler: float, kind: int) -> np.ndarray:
    """The correlation profile of the n_ms milliseconds x against the replica at doppler, widened as the reference's:
    through the replica table when the replica is chips (the roll undone on the result), else correlated directly."""
    rep = np.asarray(prn_replica)
    if rep.shape != (n,):
        raise ValueError(f"replica must have {n} samples")
    wide = np.complex128 if kind == _native.COHERENT else np.float64
    if not math.isfinite(doppler):  # a NaN carrier: every value of the reference's profile is NaN (the engine refuses it)
        return np.full(n, complex(math.nan, math.nan) if kind == _native.COHERENT else math.nan, dtype=wide)
    ent = POOL.get(fs, n)
    eng = ent["engine"]
    try:
        chips, roll = chips_of_replica(rep, n)
    except NotAChipReplica:  # any other replica: direct circular correlation on the device
        eng.upload_iq(x)
        return eng.correlation_profile_replica(rep, doppler, n_ms, kind).astype(wide)
    idx = POOL.replica_index(ent, chips)
    eng.upload_iq(x)
    prof = eng.correlation_profile(idx, doppler, n_ms, kind).astype(wide)
    return np.roll(prof, -roll) if roll else prof


def frequency_domain_correlation(antenna_samples: np.ndarray, prn_replica: np.ndarray) -> np.ndarray:
    """utils.py:59-73: circular cross-correlation ifft(fft(x) conj(fft(prn))) of one millisecond -> complex128[N]."""
    x = np.ascontiguousarray(antenna_samples, dtype=np.complex64)
    return _profile(x, x.size * 1000, x.size, 1, prn_replica, 0.0, _native.COHERENT)


def integrate_correlation_with_doppler_shifted_prn(
    integration_type, antenna_data: np.ndarray, stream_attributes, doppler_shift: float, prn_as_complex: np.ndarray
) -> np.ndarray:
    """utils.py:77-108.  float64[N] (NonCoherent: sum over ms of |corr|) or complex128[N] (Coherent)."""
    kind = _kind(integration_type)
    fs = int(stream_attributes.samples_per_second)
    n = int(stream_attributes.samples_per_prn_transmission)
    data = np.ascontiguousarray(antenna_data, dtype=np.complex64)
    n_ms = data.size // n  # utils.py:34-38: a trailing partial chunk is dropped
    if n_ms == 0:
        return np.zeros(n, dtype=complex if kind == _native.COHERENT else np.float64)
    return _profile(data[: n_ms * n], fs, n, n_ms, prn_as_complex, float(doppler_shift), kind)


def get_normalized_correlation_peak_strength(profile: np.ndarray) -> float:
    """utils.py:111-116 (host helper for callers that hold a full profile)."""
    peak = np.max(profile)
    return peak / np.mean(profile[profile != peak])
