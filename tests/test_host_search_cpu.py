"""Host-side acquisition logic without a GPU: GpsSatelliteDetector's pass-by-pass search (bin ranges with int()
truncation, first bin with the largest maximum, re-centring, strictly-stronger keep, coherent phase at the kept index,
detection threshold) driven through a stand-in engine whose cells are evaluated by the float64 oracle, against the
results recorded from the live reference detector (tests/golden/detector_n2046.npz).  The stand-in is test
infrastructure: it implements the four engine calls the host code makes, nothing of the product."""
import os

import numpy as np

from gpu_support import Attrs
from gypsum_b200 import _native
from oracle import gypsum_oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class OracleEngine:
    """upload_iq / set_replicas / acquire_cells / correlation_profile with the oracle's arithmetic."""

    def __init__(self, fs, n):
        self.fs, self.n, self.calls = fs, n, []

    def set_replicas(self, chips):
        self.replicas = [np.repeat(2.0 * c.astype(np.float64) - 1.0, self.n // 1023).astype(complex) for c in np.asarray(chips)]

    def upload_iq(self, x):
        self.x = np.asarray(x)

    def _profile(self, prn, dop, n_ms, kind):
        which = o.COHERENT if kind == _native.COHERENT else o.NON_COHERENT
        return o.integrate(which, self.x[: n_ms * self.n], self.fs, self.n, float(dop), self.replicas[prn])

    def acquire_cells(self, prn_idx, doppler_hz, n_ms, kind=_native.NON_COHERENT, probe_idx=None):
        self.calls.append((len(prn_idx), kind))
        rec = np.zeros(len(prn_idx), dtype=_native.RECORD_DTYPE)
        for i, (p, f) in enumerate(zip(prn_idx, doppler_hz)):
            prof = self._profile(p, f, n_ms, kind)
            mag = np.abs(prof)
            rec["peak"][i], rec["argmax"][i] = mag.max(), int(mag.argmax())
            rec["sum"][i], rec["count"][i] = mag.sum(), int(np.count_nonzero(mag == mag.max()))
            if probe_idx is not None and probe_idx[i] >= 0:
                rec["probe_re"][i], rec["probe_im"][i] = prof[probe_idx[i]].real, prof[probe_idx[i]].imag
        return rec

    def correlation_profile(self, prn, dop, n_ms, kind):
        prof = self._profile(prn, dop, n_ms, kind)
        return prof if kind == _native.COHERENT else np.abs(prof)

    def correlation_profile_replica(self, replica, dop, n_ms, kind):
        which = o.COHERENT if kind == _native.COHERENT else o.NON_COHERENT
        self.generic_calls = getattr(self, "generic_calls", 0) + 1
        return o.integrate(which, self.x[: n_ms * self.n], self.fs, self.n, float(dop), np.asarray(replica, dtype=complex))


def test_pass_by_pass_search_reproduces_the_reference_detector(monkeypatch):
    from gypsum_b200 import utils
    from gypsum_b200.acquisition import GpsSatelliteDetector, doppler_search_bins
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite

    z = np.load(os.path.join(ROOT, "tests", "golden", "detector_n2046.npz"))
    planted = [(int(p[0]), p[1], int(p[2]), p[3], p[4]) for p in z["planted"]]
    x = o.synth_iq(int(z["seed"]), 2046, 10, 2046000, planted)
    eng = OracleEngine(2046000, 2046)
    ent = {"engine": eng, "codes": {}, "table": []}
    monkeypatch.setattr(utils.POOL, "get", lambda fs, n, device=0: ent)
    codes = generate_replica_prn_signals()
    det = GpsSatelliteDetector({sid: GpsSatellite(sid, code, 2) for sid, code in codes.items()})
    rows = {int(r[0]): r for r in z["results"]}
    ids = [GpsSatelliteId(sv) for sv in (25, 1, 3)]  # two planted satellites and a noise-only one
    got = det._acquire_many_stepwise(ids, x, Attrs(2046000, 2046))
    # ten non-coherent passes of (20 | 28) bins per satellite + one coherent call
    assert [c[1] for c in eng.calls] == [_native.NON_COHERENT] * 10 + [_native.COHERENT]
    assert sum(c[0] for c in eng.calls[:10]) == 3 * 222
    for r in got:
        ref = rows[r.satellite_id.id]
        # float64 cells: every decision of the reference, exactly; values to the float32 fields of the 32-byte record
        assert (r.doppler_shift, r.prn_phase_shift) == (int(ref[1]), int(ref[3]))
        assert abs(r.correlation_strength - ref[4]) <= 2e-7 * ref[4]
        d = abs(r.carrier_wave_phase_shift - ref[2])
        assert min(d, 2 * np.pi - d) <= 1e-6
    # acquisition.py:163-167: int() truncates toward zero and the upper end is excluded
    assert list(doppler_search_bins(0.0, 7000.0))[:2] == [-7000, -6300] and len(doppler_search_bins(0.0, 7000.0)) == 20
    assert list(doppler_search_bins(-3258.0, 13.671875)) == list(range(-3271, -3244, 1))
    best = det.get_best_doppler_shift_estimation(0.0, 7000.0, x, Attrs(2046000, 2046), GpsSatelliteId(25))
    assert best.sample_offset_of_correlation_peak == int(best.non_coherent_correlation_profile.argmax()) == 777
    assert best.doppler_shift in doppler_search_bins(0.0, 7000.0)


def test_drop_in_utils_wrappers_argument_handling(monkeypatch):
    """utils.py:59-108 as the host code implements it around the engine: a replica rolled by any number of samples (the
    tracker rolls by the code phase, tracker.py:286), a trailing partial millisecond (dropped, utils.py:34-38), no whole
    millisecond at all, the integration-type error -- each compared with the oracle called the reference's way."""
    import pytest

    from gypsum_b200 import utils
    from gypsum_b200.utils import (IntegrationType, frequency_domain_correlation,
                                   integrate_correlation_with_doppler_shifted_prn)

    n, fs = 4092, 4092000
    eng = OracleEngine(fs, n)
    ent = {"engine": eng, "codes": {}, "table": []}
    monkeypatch.setattr(utils.POOL, "get", lambda fs_, n_, device=0: ent)

    A = Attrs(fs, n)

    x = o.synth_iq(3, n, 3, fs, [(9, 1250.0, 1001, 0.4, 0.3)])
    rep = o.replica(9, n)
    for roll in (0, 1, 3, 4, 1001, n - 1):  # within a chip (4 samples per chip), whole chips, both
        r = np.roll(rep, roll)
        want = o.integrate(o.NON_COHERENT, x, fs, n, 1250.0, r)
        got = integrate_correlation_with_doppler_shifted_prn(IntegrationType.NonCoherent, x, A, 1250.0, r)
        assert got.dtype == np.float64 and np.abs(got - want).max() <= 1e-9 * want.max(), roll
    ragged = np.concatenate([x, x[:100]])
    want = o.integrate(o.COHERENT, x, fs, n, -300.0, rep)
    got = integrate_correlation_with_doppler_shifted_prn(IntegrationType.Coherent, ragged, A, -300.0, rep)
    assert got.dtype == np.complex128 and np.abs(got - want).max() <= 1e-9 * np.abs(want).max()
    empty = integrate_correlation_with_doppler_shifted_prn(IntegrationType.NonCoherent, x[: n - 1], A, 0.0, rep)
    assert empty.shape == (n,) and not empty.any()
    one = frequency_domain_correlation(x[:n], np.roll(rep, 6))
    assert np.abs(one - o.correlate_1ms(x[:n].astype(np.complex128), np.roll(rep, 6))).max() <= 1e-9 * np.abs(one).max()
    with pytest.raises(ValueError, match="Unexpected integration type"):
        integrate_correlation_with_doppler_shifted_prn("coherent", x, A, 0.0, rep)
    # a replica that is NOT chips repeated N/1023 times goes to the generic (direct-correlation) entry point, like any
    # array the reference's function would accept (utils.py:59-73): scaled, complex, arbitrary
    rng = np.random.default_rng(0)
    odd = (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    for r in (rep * 0.5, odd):
        want = o.integrate(o.COHERENT, x, fs, n, 0.0, r)
        got = integrate_correlation_with_doppler_shifted_prn(IntegrationType.Coherent, x, A, 0.0, r)
        assert got.dtype == np.complex128 and np.abs(got - want).max() <= 1e-6 * np.abs(want).max()
    one = frequency_domain_correlation(x[:n], odd)
    assert np.abs(one - o.correlate_1ms(x[:n].astype(np.complex128), odd)).max() <= 1e-6 * np.abs(one).max()
    assert eng.generic_calls == 3
    with pytest.raises(ValueError):
        integrate_correlation_with_doppler_shifted_prn(IntegrationType.Coherent, x, A, 0.0, rep[:-1])  # wrong length
