"""The weak grid's float64 oracle (tests/weak_support.py) on its own: it reduces to the semi-coherent oracle, its shifts
follow the C expression, and on planted signals it finds what bit edges and code Doppler hide from the semi-coherent
grid (DESIGN.md section 8f, weak grids)."""
import ctypes
import ctypes.util

import numpy as np
import pytest

import semicoherent_support as ss
import weak_support as ws
from oracle import gypsum_oracle as o

FS, N = 2046000, 2046


def test_one_phase_without_shifts_is_the_semicoherent_oracle_bit_for_bit():
    """B = 1 at Dopplers whose shifts are all zero over the window (|f| * M * N < f_L1 / 2)."""
    x = o.synth_iq(21, N, 12, FS, [(5, 600.0, 333, 0.4, 0.3)])
    r = o.replica(5, N)
    for f, t in ((600.0, 4), (-0.0, 3), (-1500.0, 12), (2000.0, 1)):
        assert all(ws.shift(m, N, f) == 0 for m in range(12)), f
        assert np.array_equal(ws.integrate_weak(x, FS, N, f, r, t, 1)[0], ss.integrate_semicoherent(x, FS, N, f, r, t)), f


def test_each_phase_is_the_semicoherent_oracle_of_the_window_from_its_offset():
    x = o.synth_iq(22, N, 22, FS, [(5, 600.0, 333, 0.4, 0.3)])
    r = o.replica(5, N)
    prof = ws.integrate_weak(x, FS, N, 600.0, r, 8, 4)  # phase step 2: 6 ms of offsets and K = 2
    for j in range(4):
        want = ss.integrate_semicoherent(x[2 * j * N:(2 * j + 16) * N], FS, N, 600.0, r, 8)
        np.testing.assert_allclose(prof[j], want, rtol=1e-12, atol=1e-9 * want.max())


def test_partial_segments_are_refused():
    for m, t, b in ((17, 8, 4), (13, 8, 4), (5, 6, 1), (10, 4, 3), (4, 0, 1), (4, 2, 0)):
        with pytest.raises(ValueError):
            ws.weak_shape(m, t, b)
    assert ws.weak_shape(14, 8, 4) == (2, 1) and ws.weak_shape(95, 20, 4) == (5, 4) and ws.weak_shape(7, 1, 1) == (1, 7)


def test_zero_doppler_shifts_nothing():
    for m in (0, 1, 999, 10 ** 6):
        for f in (0.0, -0.0):
            assert ws.shift(m, N, f) == 0 and ws.shift(m, 16368, f) == 0


def test_shift_rounding_matches_the_c_expression():
    """rint of the same float64 product, in the same order, through the C library's rint: ties go to even, both signs,
    and the values either side of each tie."""
    libm = ctypes.CDLL(ctypes.util.find_library("m"))
    libm.rint.restype, libm.rint.argtypes = ctypes.c_double, [ctypes.c_double]
    from gypsum_b200.acquisition import code_shift

    cases = []
    for m, n in ((1, 1023), (7, 2046), (500, 2046), (999, 16368)):
        for q in (0.5, 1.5, 2.5, 3.5, 7.5):
            f = q * 1575.42e6 / (m * n)  # m * N * f / f_L1 is q, up to the last bit
            for g in (f, np.nextafter(f, 0.0), np.nextafter(f, np.inf)):
                cases += [(m, n, g), (m, n, -g)]
    for m, n, f in cases:
        c = libm.rint(float(m) * n * f / 1575.42e6)
        assert ws.shift(m, n, f) == c == code_shift(m, n, f), (m, n, f)
    assert ws.shift(1, 2, 1575.42e6 / 4) == 0.0 and ws.shift(3, 2, 1575.42e6 / 4) == 2.0  # 0.5 -> 0, 1.5 -> 2
    assert ws.shift(1, 2, -1575.42e6 / 4) == 0.0 and ws.shift(3, 2, -1575.42e6 / 4) == -2.0


def test_generator_without_doppler_or_bits_is_synth_iq():
    planted = [(25, 0.0, 777, 0.3, 0.3)]
    x = o.synth_iq(4, N, 3, FS, planted)
    # the first of the two bits holds the partial code period before sample 777
    y = ws.synth_weak_iq(4, N, 3, FS, [p + (0, [1.0, 1.0]) for p in planted])
    np.testing.assert_allclose(y, x, atol=1e-6)


def test_a_bit_edge_in_every_segment_hides_the_satellite_from_one_phase():
    """Bits alternating every 20 ms with edges 10 ms into every 20-ms segment of phase 0: with B = 1 the planted cell
    cancels down to the noise and the search picks a neighbouring Doppler bin (a mid-segment sign flip looks like a
    25-Hz offset); B = 2 and B = 4 find the exact code phase and Doppler on the phase that starts at a bit edge."""
    x = ws.bit_phase_iq()
    planted_bin = int(np.flatnonzero(ws.BIT_BINS == ws.BIT_DOPPLER)[0])
    b1 = ws.vector_weak(x, ws.BIT_FS, ws.BIT_N, ws.BIT_SVS, ws.BIT_BINS, 20, 1)
    (_, f1), _, _ = ws.search_decision(b1[0], b1[1], ws.BIT_BINS)
    assert f1 != ws.BIT_DOPPLER
    assert b1[0][0, 0, planted_bin] < b1[0][1:].max()  # the planted cell is below the best noise PRN's
    for b, m, j in ((2, 90, 1), (4, 95, 2)):
        got = ws.vector_weak(x[:m * ws.BIT_N], ws.BIT_FS, ws.BIT_N, ws.BIT_SVS, ws.BIT_BINS, 20, b)
        assert ws.search_decision(got[0], got[1], ws.BIT_BINS) == ((j, ws.BIT_DOPPLER), ws.BIT_CODE_PHASE, True), b


# The weak case: 29.0 dB-Hz (amplitude 0.0197 on noise of unit variance), random bits with edges 11 ms into the
# recording, 95 ms at T = 20, B = 4 (K = 4 per phase) against the semi-coherent T = 20 grid over the first 80 ms (K = 4).
WEAK_SEED, WEAK_BIT_PHASE, WEAK_AMP = 3, 11, 0.01970367272436974
WEAK_SV, WEAK_DOPPLER, WEAK_CODE_PHASE = 19, 2150.0, 1337
WEAK_SVS = [WEAK_SV, 2, 6, 13, 24, 28]
WEAK_BINS = np.arange(2000.0, 2301.0, 25.0)


def weak_case_iq():
    return ws.synth_weak_iq(WEAK_SEED, N, 95, FS, [(WEAK_SV, WEAK_DOPPLER, WEAK_CODE_PHASE, 1.1, WEAK_AMP, WEAK_BIT_PHASE,
                                                     None)])


def test_weak_satellite_with_random_bits_at_a_random_phase():
    """The weak grid finds the exact code phase and Doppler on bit phase 2 (10 ms, the closest to the edges at 11 ms),
    above every noise PRN by 1.61x; the semi-coherent grid, whose segments straddle the edges, lands one 25-Hz bin off
    with a margin of 1.25x."""
    x = weak_case_iq()
    w = ws.vector_weak(x, FS, N, WEAK_SVS, WEAK_BINS, 20, 4)
    assert ws.search_decision(w[0], w[1], WEAK_BINS) == ((2, WEAK_DOPPLER), WEAK_CODE_PHASE, True)
    assert w[0][0].max() >= 1.6 * w[0][1:].max()
    s = ss.vector_semicoherent(x[:80 * N], FS, N, WEAK_SVS, WEAK_BINS, 20)
    b, tau, above = ss.search_decision(s[0], s[1])
    assert WEAK_BINS[b] != WEAK_DOPPLER and s[0][0].max() < 1.3 * s[0][1:].max()


def test_code_doppler_realignment_over_one_second():
    """1 s at 2.046 Msps and 6 kHz, where the code drifts 7.8 samples: the realigned non-coherent profile (T = 1) peaks
    on the planted code phase with 0.990 of a zero-Doppler control's peak (at least 0.95 asserted; the rest is the up to
    1/2-sample rounding of each shift), and the unaligned profile's peak is 2.6x lower (2.4x asserted), 6 samples off."""
    planted = dict(sv=9, tau=700, amp=0.1)
    x = ws.synth_weak_iq(3, N, 1000, FS, [(planted["sv"], 6000.0, planted["tau"], 0.2, planted["amp"], 0, [1.0] * 60)])
    c = ws.synth_weak_iq(3, N, 1000, FS, [(planted["sv"], 0.0, planted["tau"], 0.2, planted["amp"], 0, [1.0] * 60)])
    r = o.replica(planted["sv"], N)
    aligned = ws.integrate_weak(x, FS, N, 6000.0, r, 1, 1)[0]
    control = ws.integrate_weak(c, FS, N, 0.0, r, 1, 1)[0]
    unaligned = o.integrate(o.NON_COHERENT, x, FS, N, 6000.0, r)
    assert int(np.argmax(aligned)) == planted["tau"] == int(np.argmax(control))
    assert aligned.max() >= 0.95 * control.max()
    assert unaligned.max() * 2.4 <= aligned.max()
    assert int(np.argmax(unaligned)) != planted["tau"]
