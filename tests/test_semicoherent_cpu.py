"""The semi-coherent oracle (tests/semicoherent_support.py) against the oracle's two integration types, and the
sensitivity the mode exists for, decided on the float64 oracle alone.

integrate_semicoherent with one-millisecond segments is the non-coherent profile bit for bit; with one segment over the
whole window it is the magnitude of the coherent profile.  The vectorised grid form agrees with it.  The planted satellite
of the sensitivity case (C/N0 30.3 dB-Hz, data bits every 20 ms aligned to the segments) is lost by a 20-ms non-coherent
search over a 50-Hz grid and found by T = 10, K = 2 at its code phase and within one bin of its Doppler."""
import numpy as np
import pytest

import semicoherent_support as ss
from acq_support import MAG_TOL, vector_grid
from oracle import gypsum_oracle as o

FS, N = 2046000, 2046


def _iq(seed, n_ms, planted=((9, 730.0, 1023, 0.5, 0.2),), nav_bits=False):
    return o.synth_iq(seed, N, n_ms, FS, list(planted), nav_bits=nav_bits)


@pytest.mark.parametrize("n_ms", [1, 3, 6])
def test_one_ms_segments_are_the_non_coherent_profile_exactly(n_ms):
    x = _iq(10 + n_ms, n_ms)
    for f in (730.0, -1250.5, -0.0):
        want = o.integrate(o.NON_COHERENT, x, FS, N, f, o.replica(9, N))
        got = ss.integrate_semicoherent(x, FS, N, f, o.replica(9, N), 1)
        assert np.array_equal(got, want), (n_ms, f)


@pytest.mark.parametrize("n_ms", [1, 4, 10])
def test_one_segment_is_the_coherent_magnitude(n_ms):
    x = _iq(20 + n_ms, n_ms)
    for f in (730.0, 4321.25):
        want = np.abs(o.integrate(o.COHERENT, x, FS, N, f, o.replica(9, N)))
        got = ss.integrate_semicoherent(x, FS, N, f, o.replica(9, N), n_ms)
        assert np.abs(got - want).max() <= 1e-12 * want.max(), (n_ms, f)


def test_partial_segments_are_refused():
    x = _iq(1, 5)
    for t in (0, 2, 3, 4, 6):
        with pytest.raises(ValueError):
            ss.integrate_semicoherent(x, FS, N, 0.0, o.replica(9, N), t)


@pytest.mark.parametrize("t", [1, 2, 3, 6])
def test_vectorised_grid_is_the_oracle(t):
    x = _iq(30 + t, 6, planted=((9, 730.0, 1023, 0.5, 0.2), (14, -500.0, 0, 1.0, 0.2)))
    svs, dop = [9, 14, 21], np.array([-500.0, 0.0, 730.0])
    peak, arg, total, count = ss.vector_semicoherent(x, FS, N, svs, dop, t)
    for a, sv in enumerate(svs):
        for b, f in enumerate(dop):
            prof = ss.integrate_semicoherent(x, FS, N, f, o.replica(sv, N), t)
            assert abs(peak[a, b] - prof.max()) <= 1e-12 * prof.max()
            assert abs(total[a, b] - prof.sum()) <= 1e-12 * prof.sum()
            assert arg[a, b] == prof.argmax() and count[a, b] == np.count_nonzero(prof == prof.max())
    # one-millisecond segments: the non-coherent grid, within float64 rounding of its own vectorised form
    if t == 1:
        ref = vector_grid(x, FS, N, svs, dop)
        assert np.abs(peak - ref[0]).max() <= MAG_TOL * 1e-6 * ref[0].max() and np.array_equal(arg, ref[1])


def test_semicoherent_finds_a_satellite_the_non_coherent_search_misses():
    x = ss.sensitivity_iq()
    nc_peak, nc_arg, _, _, _ = vector_grid(x, ss.SENS_FS, ss.SENS_N, ss.SENS_SVS, ss.SENS_BINS)
    b, tau, above = ss.search_decision(nc_peak, nc_arg)
    assert tau != ss.SENS_CODE_PHASE or not above, "the 20-ms non-coherent search should miss this satellite"
    peak, arg, _, _ = ss.vector_semicoherent(x, ss.SENS_FS, ss.SENS_N, ss.SENS_SVS, ss.SENS_BINS, 10)
    b, tau, above = ss.search_decision(peak, arg)
    assert tau == ss.SENS_CODE_PHASE and above
    assert abs(ss.SENS_BINS[b] - ss.SENS_DOPPLER) <= 50.0
