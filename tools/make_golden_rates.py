"""Generate tests/golden/acquisition_rates.npz by running the LIVE reference (/root/reference) at the sample rates the
other acquisition fixtures do not cover: 5.115, 6.138, 8.184, 10.230 and 12.276 Msps (S = 5, 6, 8, 10, 12).

Same pattern and input bytes as tools/make_golden.py (the `_Bytes` / `_Sat` shims, oracle.synth_iq).  It records
  * per rate, M = 2: one planted cell's utils.py:77 non-coherent and coherent profiles and its strength.  The planted
    code phase is n - 1, on the last polyphase branch;
  * at 5.115 and 12.276 Msps, M = 4: acquisition.py:70-152 for three satellites (two planted, one absent) and the
    detector's acquisition.py:52-68 answer for the same three.
Run:  python tools/make_golden_rates.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, "/root/reference")

from gypsum.acquisition import GpsSatelliteDetector  # noqa: E402
from gypsum.antenna_sample_provider import SampleProviderAttributes  # noqa: E402
from gypsum.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals  # noqa: E402
from gypsum.satellite import GpsSatellite  # noqa: E402
from gypsum.utils import (  # noqa: E402
    IntegrationType,
    get_normalized_correlation_peak_strength,
    integrate_correlation_with_doppler_shifted_prn,
)

from oracle import gypsum_oracle as o  # noqa: E402  (only for synth_iq: identical input bytes everywhere)

OUT = os.path.join(ROOT, "tests", "golden", "acquisition_rates.npz")
PROFILE_SEED, PROFILE_MS = 4321, 2
# S -> (sv, Doppler of the recorded cell).  The planted satellite sits 0.25 Hz off the cell, at code phase n - 1.
PROFILE_CELLS = {5: (14, 2345.0), 6: (7, -4250.0), 8: (21, 6500.0), 10: (30, -1250.0), 12: (2, 9000.0)}
DETECT_MS = 4
# S -> (seed, planted, svs); the last satellite of each list is not in the signal
DETECT_CASES = {
    5: (55, [(14, 2345.0, 5114, 0.9, 0.12), (3, -4100.0, 2600, 2.2, 0.1)], [14, 3, 20]),
    12: (66, [(9, 3650.0, 12275, 0.4, 0.08), (27, -6200.0, 6007, 1.7, 0.08)], [9, 27, 5]),
}


class _Bytes(np.ndarray):
    """acquisition.py:203 calls ndarray.tostring(), removed in numpy 2.x; supply it from the caller side so the
    reference file runs unmodified."""

    def tostring(self):
        return self.tobytes()


class _Sat:
    def __init__(self, sat):
        self.satellite_id = sat.satellite_id
        self.prn_as_complex = sat.prn_as_complex.view(_Bytes)


def main():
    codes = generate_replica_prn_signals()
    rec = {}
    for s, (sv, f) in PROFILE_CELLS.items():
        n = 1023 * s
        fs = n * 1000
        planted = [(sv, f + 0.25, n - 1, 0.6, 0.3)]
        x = o.synth_iq(PROFILE_SEED, n, PROFILE_MS, fs, planted)
        attrs = SampleProviderAttributes(fs, n)
        prn = GpsSatellite(GpsSatelliteId(sv), codes[GpsSatelliteId(sv)], s).prn_as_complex
        nc = integrate_correlation_with_doppler_shifted_prn(IntegrationType.NonCoherent, x, attrs, f, prn)
        co = integrate_correlation_with_doppler_shifted_prn(IntegrationType.Coherent, x, attrs, f, prn)
        key = f"cell_n{n}"
        rec[f"{key}__sv"], rec[f"{key}__doppler"] = np.int64(sv), np.float64(f)
        rec[f"{key}__planted"] = np.array(planted, dtype=np.float64)
        rec[f"{key}__noncoherent"], rec[f"{key}__coherent"] = nc, co
        rec[f"{key}__strength"] = np.float64(get_normalized_correlation_peak_strength(nc))
    for s, (seed, planted, svs) in DETECT_CASES.items():
        n = 1023 * s
        fs = n * 1000
        x = o.synth_iq(seed, n, DETECT_MS, fs, planted)
        attrs = SampleProviderAttributes(fs, n)
        sats = {GpsSatelliteId(i): _Sat(GpsSatellite(GpsSatelliteId(i), codes[GpsSatelliteId(i)], s)) for i in svs}
        det = GpsSatelliteDetector(sats)
        rows = []
        for sv in svs:
            r = det._attempt_acquisition_for_satellite_id(GpsSatelliteId(sv), x, attrs)
            rows.append([sv, r.doppler_shift, r.carrier_wave_phase_shift, r.prn_phase_shift, r.correlation_strength])
        found = det.detect_satellites_in_antenna_data([GpsSatelliteId(sv) for sv in svs], x, attrs)
        key = f"detect_n{n}"
        rec[f"{key}__seed"], rec[f"{key}__n_ms"] = np.int64(seed), np.int64(DETECT_MS)
        rec[f"{key}__planted"], rec[f"{key}__svs"] = np.array(planted, dtype=np.float64), np.array(svs)
        rec[f"{key}__results"] = np.array(rows, dtype=np.float64)
        rec[f"{key}__detected"] = np.array([r.satellite_id.id for r in found])
    rec["profile_seed"], rec["profile_ms"] = np.int64(PROFILE_SEED), np.int64(PROFILE_MS)
    np.savez_compressed(OUT, **rec)
    print("golden written:", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
