"""The position-fix kernels' serial repair on the device (fix.cu through gb200_tracker_position_fixes), on the timelines
with a receiver-clock jump recorded from the live reference's GpsWorldModel (tests/golden/fix_repair.npz).  On each of
them the chain check misses and k_fix_repair runs; fx.device_passes over the host core and the device's own
observations predicts every record and the repair count exactly (tests/test_fix_repair_cpu.py runs the same model on
the CPU)."""
import os

import numpy as np
import pytest

from fix_support import ChainCheck, fix_emulator, rows_at, run_golden, slide_tol
from gpu_support import make_engine
from oracle import fix_oracle as fx

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "fix_repair.npz")
GAPS = ["gap_mid", "gap_two", "gap_back", "gap_first", "gap_carry", "gap_five", "gap_raise"]
N, FS = 2046, 2046000


@pytest.fixture(scope="module")
def engine(native_lib):
    e = make_engine(FS, N)
    yield e
    e.close()


@pytest.fixture(scope="module")
def fix_emu():
    return fix_emulator()


@pytest.mark.parametrize("name", GAPS + ["singular"])
def test_repair_on_the_device(engine, fix_emu, name):
    """Against the recording and the oracle: status, ready count and rows exact; slides and round-0 pseudoranges within
    4 ulp, clock bias within 1e-14 s, position within 2e-6 m.  Against the model of the passes on the device's own
    observations (fix_support.ChainCheck): every record bit for bit, and after every call receiver_state()'s slide the
    model's carried slide exactly, its order and stop the oracle's and its repair count the model's.  Every solved
    record is the host core's fix from its own slide_in; a fix that does not start a segment starts from the slide the
    fix before it left, exactly where the repair ran and within 4 ulp elsewhere; the last slide is the oracle's within
    4 ulp."""
    z, calls, out = run_golden(engine, GOLDEN, name)
    rcv = fx.ReceiverOracle(len(calls[0][1]))
    check = ChainCheck(fix_emu)
    for c, ((rx, chans), (got, obs, state)) in enumerate(zip(calls, out)):
        want = rcv.call(chans, rx)
        rec = fx.golden_fix_rows(z, name, c)
        assert np.array_equal(got["status"], rec[:, 3].astype(int))
        # the oracle's status, rows and numbers, the model of the passes bit for bit and receiver_state()
        model = check(want, rcv.resets, rcv.order, rcv.stopped, got, obs, state, what=c)
        fixing = np.flatnonzero(np.isin(want["status"], [fx.FIX_SOLVED, fx.FIX_RAISED]))
        for m in np.flatnonzero(want["status"] == fx.FIX_SOLVED):
            host = fix_emu(rows_at(obs, want[m]["channel"], m), got[m]["receiver_timestamp"], got[m]["slide_in"])
            assert host.tobytes()[:88] == got[m].tobytes()[:88] and host["status"] == got[m]["status"], m
        # the chain relation
        for a, b in zip(fixing[:-1], fixing[1:]):
            if b in rcv.resets or any(r in rcv.resets for r in range(a + 1, b)):
                assert got[b]["slide_in"] == rcv.resets[max(r for r in rcv.resets if r <= b)]
            elif model["first_miss"] is not None and b > model["first_miss"]:
                assert got[b]["slide_in"] == got[a]["slide_out"], b
            else:
                assert abs(got[b]["slide_in"] - got[a]["slide_out"]) <= slide_tol(got[a]["slide_out"]), b
        print(f"{name} call {c}: first miss {model['first_miss']}, repaired {len(model['repaired'])}, "
              f"receiver_state repaired {state['repaired']}")
    st = out[-1][2]
    assert st["order"] == rcv.order and st["stopped"] == rcv.stopped
    if rcv.slide is not None:
        assert abs(st["slide"] - rcv.slide) <= slide_tol(rcv.slide)
    if name in GAPS:
        assert out[0][2]["repaired"] > 0
    print(f"{name}: worst slide {check.worst[0]:.3g} ulp, clock bias {check.worst[1]:.3g} s, position "
          f"{check.worst[2]:.3g} m")


def test_carried_slide_needs_no_repair(engine):
    """gap_carry repairs to the end of call 0; call 1 continues from the repaired slide and repairs nothing."""
    _, _, out = run_golden(engine, GOLDEN, "gap_carry")
    (first, _, s0), (second, _, s1) = out
    assert s0["repaired"] > 0 and s1["repaired"] == s0["repaired"]
    assert (first["status"][-100:] == fx.FIX_SOLVED).all() and second["status"][0] == fx.FIX_SOLVED
    assert second[0]["slide_in"] == first[-1]["slide_out"]


def test_gap_five_stops_at_the_raise(engine):
    z, _, out = run_golden(engine, GOLDEN, "gap_five")
    got, _, state = out[0]
    assert np.flatnonzero(got["status"] == fx.FIX_RAISED).tolist() == [400]
    assert (got["status"][401:] == fx.FIX_STOPPED).all() and (out[1][0]["status"] == fx.FIX_STOPPED).all()
    assert state["stopped"] and state["slide"] == got[400]["slide_out"] == fx.golden_fix_rows(z, "gap_five", 0)[400, 6]


def test_singular_matrix_stops_the_receiver(engine):
    """Two channels with one ephemeris: the device raises at the millisecond the reference raised, with the slide the
    reference kept, and stops."""
    z, _, out = run_golden(engine, GOLDEN, "singular")
    want = fx.golden_fix_rows(z, "singular", 0)
    got, _, state = out[0]
    assert np.flatnonzero(got["status"] == fx.FIX_RAISED).tolist() == [300] == np.flatnonzero(want[:, 3] == 2).tolist()
    assert got[300]["slide_out"] == want[300, 6] and np.isnan(got[300]["x"])
    assert (got["status"][301:] == fx.FIX_STOPPED).all() and (out[1][0]["status"] == fx.FIX_STOPPED).all()
    assert state["stopped"] and out[1][2]["stopped"] and state["repaired"] == 0


def test_fixes_device_matches_host_on_a_repair(engine):
    _, _, host = run_golden(engine, GOLDEN, "gap_mid")
    _, _, dev = run_golden(engine, GOLDEN, "gap_mid", device_out=True)
    assert host[0][2]["repaired"] > 0
    for (a, _, _), (b, _, _) in zip(host, dev):
        assert a.tobytes() == b.tobytes()
