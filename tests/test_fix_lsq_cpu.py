"""The position fix's least-squares mode on the CPU: fix_core.cuh's least-squares solve compiled for the host
(tests/emu/fix_emu.cu) on exact pseudoranges from a planted position with 5 to 12 satellites, against the
least-squares oracle (tests/fix_lsq_oracle.py, np.linalg.lstsq) on perturbed rows and on the five-ready golden timelines,
the four-row case against the reference mode, and the rank-deficient raise."""
import os

import numpy as np
import pytest

import fix_lsq_oracle as lo
from fix_support import BIAS_S, MANY_BIAS_S, MANY_POS_M, MANY_SLIDE_ULPS, POS_M, fix_emulator, slide_tol
from oracle import fix_oracle as fx
from oracle import orbit_oracle as orb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# least squares against numpy's SVD where Gauss-Newton has converged (perturbed rows: numpy's last step below 1e-6 m),
# a small multiple of the measured spread (DESIGN.md §8c: position 2.4e-5 m with 5 rows, 4.4e-9 m with 6 to 12; clock
# bias 3.8e-14 s; slide 0 ulp)
LSQ_POS_M, LSQ_BIAS_S, LSQ_SLIDE_ULPS = 1e-4, 2e-13, 4


@pytest.fixture(scope="module")
def lsq_emu():
    return fix_emulator()


def satellites(seed, n):
    """n satellite positions from realistic planted ephemerides (as tests/test_fix_cpu.py's, with more rows)."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        sv = orb.OrbitOracle()
        eph = orb.realistic_ephemeris(rng, 1 + k)
        for sf in (1, 2, 3):
            sv.subframe(orb.parse(orb.words_of(orb.encode_subframe(sf, 5000, eph))), 1.0)
        sv.count, sv.counting = 1234 + 7 * k, True
        tow, _ = sv.time_of_week()
        out.append((tow, *sv.position(tow)))
    return out


def planted_rows(sats, pos, bias, rx, slide, tow_noise=None):
    """Rows whose pseudoranges are exact for the receiver at pos with clock bias `bias`, plus tow_noise[i] seconds."""
    rows = []
    for i, (_, x, y, z) in enumerate(sats):
        rng_ = np.sqrt((pos[0] - x) ** 2 + (pos[1] - y) ** 2 + (pos[2] - z) ** 2)
        noise = 0.0 if tow_noise is None else tow_noise[i]
        rows.append(((slide + rx) - (rng_ / fx.SPEED_OF_LIGHT + bias) + noise, x, y, z))
    return rows


CASES = [((-2.7e6, -4.3e6, 3.9e6), 0.0123), ((4.0e6, 3.0e5, 4.9e6), -0.071), ((1.1e6, -6.2e6, 1.0e5), 0.0)]


@pytest.mark.parametrize("n", [5, 6, 8, 12])
def test_least_squares_recovers_a_planted_position(lsq_emu, n):
    """Exact pseudoranges from a planted receiver position and clock bias over n rows: the least-squares core recovers
    both within the reference mode's bounds.  The residuals are zero, so this does not depend on numpy."""
    worst = 0.0
    for seed, (pos, bias) in enumerate(CASES):
        rows = planted_rows(satellites(100 + seed, n), pos, bias, 0.5, 0.0)
        got = lsq_emu(rows, 0.5, 0.0)
        assert got["status"] == fx.FIX_SOLVED
        err = max(abs(got[k] - p) for k, p in zip("xyz", pos))
        worst = max(worst, err)
        assert err <= POS_M, err
        assert abs(got["slide_out"] - (0.0 - bias)) <= BIAS_S and abs(got["clock_bias"]) <= BIAS_S
        assert np.array_equal(got["pseudorange"], [(0.0 + 0.5) - r[0] for r in rows[:4]])
    print(f"n = {n}: planted position recovered within {worst:.3g} m")


@pytest.mark.parametrize("n", [5, 6, 8, 12])
def test_perturbed_rows_against_numpy(lsq_emu, n):
    """Rows whose times of week disagree by up to 1e-7 s (30 m of range), at a realistic slide: the host core against
    np.linalg.lstsq's Gauss-Newton within LSQ_*, where the oracle's last step shows it has converged."""
    rng = np.random.default_rng(7 + n)
    worst = [0.0, 0.0, 0.0]
    steps = [0.0, 0.0]
    for seed, (pos, bias) in enumerate(CASES):
        sats = satellites(200 + seed, n)
        rx = 3.0 + seed
        slide = sats[0][0] - 0.07 - rx  # a reset's slide: about 4e5 s, as on the receiver
        rows = planted_rows(sats, pos, bias, rx, slide, rng.uniform(-1e-7, 1e-7, n))
        got = lsq_emu(rows, rx, slide)
        info = {}
        want = lo.compute_position(rows, rx, slide, info)
        assert got["status"] == fx.FIX_SOLVED
        steps = [max(a, b) for a, b in zip(steps, info["last_step"])]
        assert info["last_step"][0] < 1e-6, info  # converged: the bound below is not set on a moving iterate
        worst[0] = max(worst[0], abs(got["slide_out"] - want[0]) / (2.0 ** -52 * abs(want[0])))
        worst[1] = max(worst[1], abs(got["clock_bias"] - want[1]))
        worst[2] = max(worst[2], *(abs(got[k] - w) for k, w in zip("xyz", want[2])))
        assert np.abs(got["pseudorange"] - want[3]).max() <= 4 * 2.0 ** -52 * abs(slide)
        # 30 m of inconsistency moves the solution by metres, not kilometres
        assert max(abs(got[k] - p) for k, p in zip("xyz", pos)) < 1e3
    print(f"n = {n}: host vs numpy slide {worst[0]:.3g} ulp, clock bias {worst[1]:.3g} s, position {worst[2]:.3g} m; "
          f"numpy's last step {steps[0]:.3g} m / {steps[1]:.3g} s")
    assert worst[0] <= LSQ_SLIDE_ULPS and worst[1] <= LSQ_BIAS_S and worst[2] <= LSQ_POS_M, worst


@pytest.mark.parametrize("name", [("fix", "five"), ("fix_repair", "gap_five")], ids=["five", "gap_five"])
def test_golden_five_ready_against_numpy(lsq_emu, name):
    """Every five-ready fix of the golden timelines in the least-squares oracle's chain, from the oracle's slide_in:
    the host core against numpy within MANY_*, the oracle's last step reported beside it."""
    z = np.load(os.path.join(ROOT, "tests", "golden", f"{name[0]}.npz"))
    rcv, worst, steps, n5 = None, [0.0, 0.0, 0.0], [0.0, 0.0], 0
    for rx, chans in fx.golden_calls(z, name[1]):
        rcv = rcv or lo.ReceiverOracle(len(chans))
        rec = rcv.call(chans, rx)
        assert not (rec["status"] == fx.FIX_RAISED).any()
        for m in np.flatnonzero((rec["status"] == fx.FIX_SOLVED) & (rec["n_ready"] >= 5)):
            r = rec[m]
            got = lsq_emu(rcv.rows[m], r["receiver_timestamp"], r["slide_in"])
            assert got["status"] == fx.FIX_SOLVED and got["slide_in"] == r["slide_in"]
            assert np.array_equal(got["pseudorange"], r["pseudorange"])
            if n5 % 50 == 0:
                info = {}
                lo.compute_position(rcv.rows[m], r["receiver_timestamp"], r["slide_in"], info)
                steps = [max(a, b) for a, b in zip(steps, info["last_step"])]
            n5 += 1
            worst[0] = max(worst[0], abs(got["slide_out"] - r["slide_out"]) / (2.0 ** -52 * abs(r["slide_out"])))
            worst[1] = max(worst[1], abs(got["clock_bias"] - r["clock_bias"]))
            worst[2] = max(worst[2], *(abs(got[k] - r[k]) for k in "xyz"))
    assert n5 >= 600
    print(f"{name[1]}: {n5} five-ready fixes; host vs numpy slide {worst[0]:.3g} ulp, clock bias {worst[1]:.3g} s, "
          f"position {worst[2]:.3g} m; numpy's last step up to {steps[0]:.3g} m / {steps[1]:.3g} s")
    assert worst[0] <= MANY_SLIDE_ULPS and worst[1] <= MANY_BIAS_S and worst[2] <= MANY_POS_M, worst


@pytest.mark.parametrize("name", ["realistic", "lost", "five"])
def test_four_rows_are_the_reference_fix(lsq_emu, name):
    """Four ready rows take the reference mode's code path: the host core's record is the reference oracle's within the
    reference mode's bounds, and the oracle's least-squares mode equals the reference oracle bit for bit up to the
    first five-ready millisecond."""
    z = np.load(os.path.join(ROOT, "tests", "golden", "fix.npz"))
    ref = ls = None
    n = 0
    for rx, chans in fx.golden_calls(z, name):
        ref = ref or fx.ReceiverOracle(len(chans))
        ls = ls or lo.ReceiverOracle(len(chans))
        a, b = ref.call(chans, rx), ls.call(chans, rx)
        five = np.flatnonzero(a["n_ready"] >= 5)
        end = five[0] if len(five) else len(a)
        assert a[:end].tobytes() == b[:end].tobytes()
        for m in np.flatnonzero(b["status"] == fx.FIX_SOLVED):
            if b[m]["n_ready"] == 4:
                got, want = lsq_emu(ls.rows[m], rx[m], b[m]["slide_in"]), a[m]
                assert got["status"] == want["status"] and got["slide_in"] == want["slide_in"], m
                assert abs(got["slide_out"] - want["slide_out"]) <= slide_tol(want["slide_out"]), m
                assert np.abs(got["pseudorange"] - want["pseudorange"]).max() <= slide_tol(want["slide_in"]), m
                assert abs(got["clock_bias"] - want["clock_bias"]) <= BIAS_S, m
                assert max(abs(got[k] - want[k]) for k in "xyz") <= POS_M, m
                n += 1
        if len(five):
            break
    assert n >= 100


def test_identical_rows_raise(lsq_emu):
    """Five identical rows: rank 1.  The oracle's lstsq reports it and raises with the entering slide; the host core
    raises there too and leaves the solution unset."""
    row = satellites(3, 1)[0]
    rows = [row] * 5
    rx, slide = 2.0, row[0] - 0.07 - 2.0
    with pytest.raises(np.linalg.LinAlgError) as err:
        lo.compute_position(rows, rx, slide)
    assert err.value.slide == slide
    got = lsq_emu(rows, rx, slide)
    assert got["status"] == fx.FIX_RAISED and got["slide_in"] == got["slide_out"] == slide and np.isnan(got["x"])


def test_five_ready_chain_model(lsq_emu):
    """What DESIGN.md §8c reports of the two passes in this mode, from the device model on the host core: on `five` the
    non-converging five-row fixes depend on their entering slide, so the chain check misses at the first fix after the
    five-ready millisecond and the repair runs the rest of the segment serially; on `gap_five` the miss is the clock
    jump's, as in the reference mode.  Either way the records are the serial chain's, so they agree with the oracle's."""
    want = {"five": (401, 298), "gap_five": (350, 49)}
    for npz, name in (("fix", "five"), ("fix_repair", "gap_five")):
        z = np.load(os.path.join(ROOT, "tests", "golden", f"{npz}.npz"))
        rcv, carried, misses = None, None, []
        for rx, chans in fx.golden_calls(z, name):
            rcv = rcv or lo.ReceiverOracle(len(chans))
            rec = rcv.call(chans, rx)
            d = lo.device_passes(lsq_emu, rec, rcv.rows, rcv.resets, carried)
            carried = d["slide"]
            misses.append((d["first_miss"], len(d["repaired"])))
            for m, f in d["out"].items():
                assert f["status"] == rec[m]["status"]
                assert abs(f["slide_out"] - rec[m]["slide_out"]) <= MANY_SLIDE_ULPS * 2.0 ** -52 * abs(rec[m]["slide_out"])
        print(f"{name}: (first miss, repaired) per call {misses}")
        assert misses == [want[name], (None, 0)]
