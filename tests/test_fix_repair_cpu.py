"""The position fix's serial repair on the CPU, on timelines recorded from the live reference's GpsWorldModel with a
receiver-clock jump inside a segment (tests/golden/fix_repair.npz, tools/make_golden_fix.py).  A jump puts the fix from
the segment's reset slide (the device's pass 1) on the other root of the squared-range equations while the serial chain
stays on its own, so the device's chain check misses and k_fix_repair runs (DESIGN.md §8c).  fx.device_passes models the
device's passes over the host core (fix_core.cuh compiled for the host): it predicts the first miss and the fixes the
repair recomputes, and shows on the CPU that every gap timeline needs the repair."""
import os

import numpy as np
import pytest

from fix_support import BIAS_S, POS_M, fix_emulator, slide_tol
from oracle import fix_oracle as fx

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "fix_repair.npz")
TIMELINES = ["gap_mid", "gap_two", "gap_back", "gap_first", "gap_carry", "gap_five", "gap_raise", "singular"]
# timeline -> (call, first miss, fixes the repair recomputes in each call), from the host core on the oracle's rows
MISSES = {
    "gap_mid": (0, 600, [299, 0]),  # 601-899, up to the reset at 900
    "gap_two": (0, 600, [598, 0]),  # 601-899, then 1201-1499 after the second jump, across the reset at 900
    "gap_back": (0, 600, [150, 0]),  # 601-750: the jump back at 750 returns the chain to pass 1's root
    "gap_first": (0, 301, [598, 0]),  # 302-899
    "gap_carry": (0, 1300, [199, 0]),  # 1301-1499; call 1 starts from the repaired slide
    "gap_five": (0, 350, [49, 0]),  # 351-399; the LinAlgError at 400 is a reset millisecond
    "gap_raise": (0, 400, [99, 0]),  # 401-499; the decoder raise stops the receiver at 500
}


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def fix_emu():
    return fix_emulator()


def model_timeline(z, name, compute):
    """Per call: the oracle's records and the device model's passes on the oracle's rows, the slide carried across."""
    rcv, carried, out = None, None, []
    for rx, chans in fx.golden_calls(z, name):
        rcv = rcv or fx.ReceiverOracle(len(chans))
        rec = rcv.call(chans, rx)
        d = fx.device_passes(compute, rec, rcv.rows, rcv.resets, carried)
        carried = d["slide"]
        out.append((rec, d))
    return out, rcv


def test_golden_lists_every_timeline(golden):
    assert list(golden["timelines"]) == TIMELINES


@pytest.mark.parametrize("name", TIMELINES)
def test_oracle_equals_reference(golden, name):
    """Status, ready count, rows, slides and solution of the oracle equal the reference's bit for bit."""
    rcv = None
    for c, (rx, chans) in enumerate(fx.golden_calls(golden, name)):
        rcv = rcv or fx.ReceiverOracle(len(chans))
        got = rcv.call(chans, rx)
        want = fx.golden_fix_rows(golden, name, c)
        assert np.array_equal(got["status"], want[:, 3].astype(int))
        assert np.array_equal(got["n_ready"], want[:, 4].astype(int))
        assert np.array_equal(got["channel"], want[:, 11:15].astype(int))
        fixing = np.isin(got["status"], [fx.FIX_SOLVED, fx.FIX_RAISED])
        assert np.array_equal(got["slide_in"][fixing], want[fixing, 5])
        assert np.array_equal(got["slide_out"][fixing], want[fixing, 6])
        for k, col in (("clock_bias", 7), ("x", 8), ("y", 9), ("z", 10)):
            assert np.array_equal(got[k], want[:, col], equal_nan=True), k


@pytest.mark.parametrize("name", list(MISSES))
def test_every_gap_timeline_misses(golden, fix_emu, name):
    """The device model on the host core: the chain check misses where the jump lands, pass 1 alone is on the other
    root there (about 0.177 s off in the slide), and the repair recomputes the predicted fixes, none in call 1."""
    calls, _ = model_timeline(golden, name, fix_emu)
    call, miss, repaired = MISSES[name]
    assert [d["first_miss"] for _, d in calls] == [miss if c == call else None for c in range(len(calls))]
    assert [len(d["repaired"]) for _, d in calls] == repaired
    rec, d = calls[call]
    off = abs(d["pass1"][miss]["slide_out"] - rec[miss]["slide_out"])
    assert 0.1 < off < 0.3, off
    wrong = [m for m, f in d["pass1"].items() if m in d["out"] and not fx.same_slide(f["slide_out"], rec[m]["slide_out"])]
    assert wrong[0] == miss
    print(f"{name}: first miss at ms {miss}, pass 1 wrong at {len(wrong)} ms by up to "
          f"{max(abs(d['pass1'][m]['slide_out'] - rec[m]['slide_out']) for m in wrong):.3g} s, "
          f"repaired {len(d['repaired'])} fixes")


@pytest.mark.parametrize("name", TIMELINES)
def test_repaired_chain_against_the_oracle(golden, fix_emu, name):
    """What the device's records come to after the repair (the host core, chained from the first miss on) against the
    reference's serial chain: status exact, slides and round-0 pseudoranges within 4 ulp, clock bias within 1e-14 s,
    position within 2e-6 m, and the slide carried to the next call within 4 ulp."""
    calls, rcv = model_timeline(golden, name, fix_emu)
    worst = [0.0, 0.0, 0.0]
    for rec, d in calls:
        fixing = np.flatnonzero(np.isin(rec["status"], [fx.FIX_SOLVED, fx.FIX_RAISED]))
        assert sorted(d["out"]) == list(fixing)
        for m in fixing:
            got, want = d["out"][m], rec[m]
            assert got["status"] == want["status"], m
            for k in ("slide_in", "slide_out"):
                assert abs(got[k] - want[k]) <= slide_tol(want[k]), (m, k)
                worst[0] = max(worst[0], abs(got[k] - want[k]))
            if want["status"] == fx.FIX_SOLVED:
                worst[0] = max(worst[0], np.abs(got["pseudorange"] - want["pseudorange"]).max())
                assert np.abs(got["pseudorange"] - want["pseudorange"]).max() <= slide_tol(want["slide_in"]), m
                worst[1] = max(worst[1], abs(got["clock_bias"] - want["clock_bias"]))
                worst[2] = max(worst[2], *(abs(got[k] - want[k]) for k in "xyz"))
    if rcv.slide is not None:
        assert abs(calls[-1][1]["slide"] - rcv.slide) <= slide_tol(rcv.slide)
    print(f"{name}: worst slide / pseudorange {worst[0]:.3g} s, clock bias {worst[1]:.3g} s, position {worst[2]:.3g} m")
    assert worst[1] <= BIAS_S and worst[2] <= POS_M, worst


def test_gap_five_stops_the_repair_at_the_raise(golden, fix_emu):
    """The repair stops at the LinAlgError; the raise's slides are those the reset at its millisecond set, and nothing
    after it is fixed."""
    calls, _ = model_timeline(golden, "gap_five", fix_emu)
    _, d = calls[0]
    assert d["first_raise"] == 400 and max(d["out"]) == 400
    want = fx.golden_fix_rows(golden, "gap_five", 0)
    assert want[400, 3] == fx.FIX_RAISED and (want[401:, 3] == fx.FIX_STOPPED).all()
    assert d["out"][400]["slide_in"] == d["out"][400]["slide_out"] == want[400, 5] == want[400, 6]


def test_singular_matrix(golden, fix_emu):
    """Two channels of different PRNs on one ephemeris and schedule give bit-identical rows; the reference raises
    "Singular matrix" at the first fix and stops, and the host core raises there too, leaving the slide it entered with."""
    want = fx.golden_fix_rows(golden, "singular", 0)
    raised = np.flatnonzero(want[:, 3] == fx.FIX_RAISED)
    assert list(raised) == [300] and (want[301:, 3] == fx.FIX_STOPPED).all() and (want[:300, 3] == fx.FIX_NONE).all()
    assert (fx.golden_fix_rows(golden, "singular", 1)[:, 3] == fx.FIX_STOPPED).all()
    rcv = fx.ReceiverOracle(4)
    rx, chans = fx.golden_calls(golden, "singular")[0]
    rcv.call(chans, rx)
    rows = np.array(rcv.rows[300])
    assert list(want[300, 11:15]) == [0, 1, 2, 3] and rows[2].tobytes() == rows[3].tobytes()
    got = fix_emu(rows, want[300, 2], want[300, 5])
    assert got["status"] == fx.FIX_RAISED
    assert got["slide_in"] == want[300, 5] and got["slide_out"] == want[300, 6] and np.isnan(got["x"])
