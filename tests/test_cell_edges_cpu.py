"""The per-cell entry points' host rules, without a GPU: gb200_acquire_cells' automatic kernel choice at its two thresholds
(restated in acq_support.fused_choice), the drop-in helpers' recovery of a rolled chip replica at every roll residue, and
their answer for a non-finite Doppler, which the engine refuses: the reference's profile, NaN at every lag."""
import math

import numpy as np
import pytest

from acq_support import FUSED_CELL_LIMIT, FUSED_RATES, choice_list, fused_choice, rate, vector_cells
from gpu_support import Attrs
from oracle import gypsum_oracle as o

ALL_RATES = [1, 2, 3, 4, 5, 6, 8, 10, 12, 16]
CHOICES = {"unique_at": False, "unique_past": True, "size_at": True, "size_past": False}


def rolls(s):
    """Replica rolls at every residue the helpers' roll undo meets: 0, 1, S - 1, S, S + 1, N - S and N - 1."""
    n, _ = rate(s)
    return sorted({0, 1, s - 1, s, s + 1, n - s, n - 1})


@pytest.mark.parametrize("case", list(CHOICES))
def test_fused_choice_at_its_thresholds(case):
    """Each list lands exactly at or one past its threshold, and the restated rule picks the kernel named for it at S = 2
    and 4, the split kernels at every other rate and whenever a profile is wanted.  -0.0 and 0.0 are one distinct value:
    counted apart, the list at the distinct-Doppler threshold would cross it."""
    prns, dop, m = choice_list(case, 2, 3)
    n_cells, n_unique = dop.size, len({float(f) for f in dop})
    assert prns.size == n_cells and (np.signbit(dop) & (dop == 0)).any() and ((~np.signbit(dop)) & (dop == 0)).any()
    bitwise = len({f.tobytes() for f in dop})
    assert bitwise == n_unique + 1
    if case.startswith("unique"):
        assert n_cells % 4 == 0 and n_cells * m > FUSED_CELL_LIMIT
        assert n_unique == n_cells // 4 + (case == "unique_past")
        if case == "unique_at":
            assert bitwise * 4 > n_cells  # a count that told -0.0 from 0.0 would choose the fused kernel here
    else:
        assert n_cells * m == FUSED_CELL_LIMIT + (case == "size_past") and n_unique * 4 <= n_cells
    for s in ALL_RATES:
        assert fused_choice(s, dop, m) == (CHOICES[case] and s in FUSED_RATES), (case, s)
        assert not fused_choice(s, dop, m, profile=True)


def test_fused_choice_small_lists():
    """One cell, or any list of at most 8192 cell-milliseconds, takes the fused kernel at S = 2 and 4 even when every cell
    shares one Doppler."""
    for s in FUSED_RATES:
        assert fused_choice(s, [0.0], 20)
        assert fused_choice(s, [1500.0] * 409, 20) and not fused_choice(s, [1500.0] * 410, 20)
        assert fused_choice(s, [-0.0, 0.0] * 4096, 1) and not fused_choice(s, [-0.0, 0.0] * 4096 + [0.0], 1)


@pytest.mark.parametrize("s", ALL_RATES)
def test_chips_of_replica_every_roll(s):
    """chips_of_replica(roll(replica, k)) == (the code rolled by k // S chips, k % S) at every listed roll, and those
    chips repeated and rolled by the residue give the replica back; a +-1 sequence that is not chip-repeated, or a complex
    one, is NotAChipReplica."""
    from gypsum_b200 import utils

    n, _ = rate(s)
    for sv in (1, 25):
        for k in rolls(s):
            rep = np.roll(o.replica(sv, n), k)
            chips, p = utils.chips_of_replica(rep, n)
            assert p == k % s, (s, k)
            assert np.array_equal(chips, np.roll(o.ca_code(sv), k // s).astype(np.uint8)), (s, k)
            assert np.array_equal(np.roll(np.repeat(2.0 * chips - 1.0, s), p), rep.real), (s, k)
    if s > 1:
        seq = np.repeat(2.0 * o.ca_code(3) - 1.0, s)
        seq[s // 2] = -seq[s // 2]  # one sample off its chip
        with pytest.raises(utils.NotAChipReplica):
            utils.chips_of_replica(seq, n)
    with pytest.raises(utils.NotAChipReplica):
        utils.chips_of_replica(o.replica(3, n) * 1j, n)


@pytest.mark.parametrize("doppler", [math.nan, math.inf, -math.inf], ids=["nan", "inf", "minus_inf"])
def test_drop_in_non_finite_doppler_is_the_reference_profile(monkeypatch, doppler):
    """integrate_correlation_with_doppler_shifted_prn at a non-finite Doppler == o.integrate: every value NaN (both parts
    for Coherent), same dtype and length, at every rate, for chip and generic replicas and a trailing partial chunk, without creating
    an engine; fewer samples than a millisecond still give the reference's zeros."""
    from gypsum_b200 import utils

    def no_engine(*_):
        raise AssertionError("an engine was created for a non-finite Doppler")

    monkeypatch.setattr(utils.POOL, "get", no_engine)
    rng = np.random.default_rng(5)
    for s in ALL_RATES:
        n, fs = rate(s)
        x = o.synth_iq(s, n, 2, fs, [(5, 1500.0, n - 1, 0.3, 0.5)])
        data = np.concatenate([x, x[:17]])
        generic = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
        for rep in (np.roll(o.replica(5, n), s + 1), generic):
            for it, kind in ((utils.IntegrationType.NonCoherent, o.NON_COHERENT), (utils.IntegrationType.Coherent, o.COHERENT)):
                got = utils.integrate_correlation_with_doppler_shifted_prn(it, data, Attrs(fs, n), doppler, rep)
                with np.errstate(invalid="ignore"):
                    want = o.integrate(kind, data, fs, n, doppler, rep.astype(complex))
                assert got.dtype == want.dtype and got.shape == want.shape, (s, kind)
                # every real and imaginary part NaN in both; numpy's FFT leaves some with the sign bit set, some without
                assert np.isnan(want.view(np.float64)).all() and np.isnan(got.view(np.float64)).all(), (s, kind)
                short = utils.integrate_correlation_with_doppler_shifted_prn(it, x[:n - 1], Attrs(fs, n), doppler, rep)
                assert short.tobytes() == o.integrate(kind, x[:n - 1], fs, n, doppler, rep.astype(complex)).tobytes()


def test_vector_cells_matches_integrate():
    """vector_cells == o.integrate cell by cell (count and argmax exact, magnitudes within 1e-12, probe values at their
    lags) on an unsorted list with repeated cells, -0.0 next to 0.0 and repeated Dopplers of other PRNs, both kinds."""
    s = 2
    n, fs = rate(s)
    x = o.synth_iq(8, n, 3, fs, [(5, 1500.0, n - 1, 0.3, 0.7), (1, -3000.25, 0, 0.3, 0.7)])
    svs = [5, 1, 5, 32, 1, 5, 17]
    dop = np.array([1500.0, -3000.25, -0.0, 1500.0, -3000.25, 1500.0, 0.0])
    probe = np.array([n - 1, 0, 1, s - 1, n - s, n - 1, 511 * s + 1])
    for kind in (o.NON_COHERENT, o.COHERENT):
        peak, arg, total, count, val = vector_cells(x, fs, n, svs, dop, kind, probe)
        for i, (sv, f) in enumerate(zip(svs, dop)):
            prof = o.integrate(kind, x, fs, n, f, o.replica(sv, n))
            mag = np.abs(prof)
            assert (arg[i], count[i]) == (int(mag.argmax()), int(np.count_nonzero(mag == mag.max()))), (kind, i)
            assert abs(peak[i] - mag.max()) <= 1e-12 * mag.max() and abs(total[i] - mag.sum()) <= 1e-12 * mag.sum()
            assert abs(val[i] - prof[probe[i]]) <= 1e-12 * mag.max(), (kind, i)
        assert (arg[[0, 5]] == n - 1).all() and arg[1] == 0
