"""GPU parity of the position-fix kernels (fix.cu through gb200_tracker_position_fixes) against timelines recorded from
the live reference's GpsWorldModel (tests/golden/fix.npz) and the oracle, and end to end behind the tracking, bit,
subframe and orbit kernels on 60 s of IQ that carries four consistent planted ephemerides."""
import os

import numpy as np
import pytest

from fix_support import BIAS_S, POS_M, fix_emulator, parse_events, rows_at, run_golden, slide_tol
from gpu_support import make_engine
from oracle import fix_oracle as fx
from oracle import nav_oracle as nav
from oracle import orbit_oracle as orb
from oracle import tracker_oracle as t

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "fix.npz")
TIMELINES = ["realistic", "three", "gate", "lost", "five", "raise"]
N, FS = 2046, 2046000


@pytest.fixture(scope="module")
def engine(native_lib):
    e = make_engine(FS, N)
    yield e
    e.close()


@pytest.fixture(scope="module")
def fix_emu():
    return fix_emulator()


def _compare(got, want):
    """Status, ready count and rows exact; slides and round-0 pseudoranges within 4 ulp, clock bias within 1e-14 s,
    position within 2e-6 m.  Returns the largest slide / pseudorange, clock-bias and position differences."""
    assert np.array_equal(got["status"], want["status"])
    assert np.array_equal(got["n_ready"], want["n_ready"])
    assert np.array_equal(got["channel"], want["channel"])
    fixing = np.isin(want["status"], [fx.FIX_SOLVED, fx.FIX_RAISED])
    solved = want["status"] == fx.FIX_SOLVED
    worst = [0.0, 0.0, 0.0]
    if fixing.any():
        for k in ("slide_in", "slide_out"):
            d = np.abs(got[k][fixing] - want[k][fixing])
            worst[0] = max(worst[0], float(d.max()))
            assert (d <= slide_tol(want[k][fixing])).all(), k
    if solved.any():
        d = np.abs(got["pseudorange"][solved] - want["pseudorange"][solved]).max(axis=1)
        worst[0] = max(worst[0], float(d.max()))
        assert (d <= slide_tol(want["slide_in"][solved])).all()
        worst[1] = float(np.abs(got["clock_bias"][solved] - want["clock_bias"][solved]).max())
        worst[2] = max(float(np.abs(got[k][solved] - want[k][solved]).max()) for k in "xyz")
    assert worst[1] <= BIAS_S and worst[2] <= POS_M, worst
    assert np.isnan(got["x"][~solved]).all()
    return worst


@pytest.mark.parametrize("name", TIMELINES)
def test_golden_timelines_on_the_device(engine, fix_emu, name):
    """The recorded timelines through the kernels, receiver state carried across calls: status, ready count and rows
    exact, slides and solution within the bounds of the oracle's chain; every record equals the host core's fix from
    the record's own slide_in bit for bit; the chain relation holds (slide_in exact at a reset, else within 4 ulp of
    the previous fix's slide_out)."""
    z, calls, out = run_golden(engine, GOLDEN, name)
    rcv = fx.ReceiverOracle(len(calls[0][1]))
    worst = [0.0, 0.0, 0.0]
    for c, ((rx, chans), (got, obs, _)) in enumerate(zip(calls, out)):
        want = rcv.call(chans, rx)
        assert np.array_equal(got["status"], fx.golden_fix_rows(z, name, c)[:, 3].astype(int))
        worst = [max(a, b) for a, b in zip(worst, _compare(got, want))]
        for m in np.flatnonzero(got["status"] == fx.FIX_SOLVED):
            r = got[m]
            host = fix_emu(rows_at(obs, r["channel"], m), r["receiver_timestamp"], r["slide_in"])
            # the numbers (slides, solution, pseudoranges) and the status; the rows are the plan's
            assert host.tobytes()[:88] == r.tobytes()[:88] and host["status"] == r["status"], m
        # at a reset millisecond the slide is the reset value exactly; elsewhere it continues the chain
        fixing = np.flatnonzero(got["status"] == fx.FIX_SOLVED)
        for a, b in zip(fixing[:-1], fixing[1:]):
            if want[b]["slide_in"] == want[a]["slide_out"]:
                assert abs(got[b]["slide_in"] - got[a]["slide_out"]) <= slide_tol(got[a]["slide_out"])
            else:
                assert got[b]["slide_in"] == want[b]["slide_in"]
    st = out[-1][2]
    assert st["order"] == rcv.order and st["stopped"] == rcv.stopped and st["repaired"] == 0
    if rcv.slide is not None:
        assert abs(st["slide"] - rcv.slide) <= slide_tol(rcv.slide)
    print(f"{name}: worst slide / pseudorange {worst[0]:.3g} s, clock bias {worst[1]:.3g} s, position {worst[2]:.3g} m")


def test_fixes_device_matches_host(engine):
    _, _, host = run_golden(engine, GOLDEN, "lost")
    _, _, dev = run_golden(engine, GOLDEN, "lost", device_out=True)
    for (a, _, _), (b, _, _) in zip(host, dev):
        assert a.tobytes() == b.tobytes()


def test_state_errors(engine):
    from gypsum_b200 import _native

    z = np.load(GOLDEN)
    calls = fx.golden_calls(z, "realistic")
    trk = _native.Tracker(engine, [0, 1, 2, 3], [0.0] * 4, [0.0] * 4, [0] * 4)
    with pytest.raises(RuntimeError, match="no gb200_tracker_parse_subframes call"):
        trk.position_fixes([])
    assert trk.receiver_state() == {"slide": None, "stopped": False, "order": [], "repaired": 0}
    rx, chans = calls[0]
    parse_events(trk, chans, len(rx))
    with pytest.raises(ValueError, match="one start time per millisecond"):
        trk.position_fixes(rx[:-1])
    trk.position_fixes(rx)
    with pytest.raises(RuntimeError, match="already computed"):
        trk.position_fixes(rx)
    parse_events(trk, [([], -1)] * 4, 10)
    parse_events(trk, [([], -1)] * 4, 10)  # the fixes of the call before were skipped
    with pytest.raises(RuntimeError, match="gap"):
        trk.position_fixes(np.arange(10) * 0.001)
    trk.close()
    # parse calls before the first fix call may go without fixes
    trk = _native.Tracker(engine, [0, 1, 2, 3], [0.0] * 4, [0.0] * 4, [0] * 4)
    parse_events(trk, [([], -1)] * 4, 10)
    parse_events(trk, [([], -1)] * 4, 10)
    assert (trk.position_fixes(np.arange(10) * 0.001)["status"] == fx.FIX_NONE).all()
    trk.close()


def test_position_fix_behind_the_tracking_kernel(engine):
    """4 channels x 60 s at 2.046 Msps through TrackerBank -> integrate_bits -> decode_subframes -> parse_subframes ->
    position_fixes in 1-s calls.  Every channel carries the same TOW counts with its own ephemeris and starts its bits
    at the same millisecond, so the four complete together (after the decoder's phase search and subframes 1-3) and
    their times of week stay consistent.  Every record's status, ready count and rows match the oracle fed the device's
    own events and drops; its numbers match the oracle teacher-forced with the record's slide_in, on sampled
    milliseconds and on every millisecond around a reset or a change of the ready set.  The last seconds fix on every
    millisecond."""
    from gypsum_b200.antenna_sample_provider import SampleProviderAttributes
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import TrackerBank
    from gypsum_b200.world_model import solution_from_fix

    erng = np.random.default_rng(11)
    chans = []
    for i, (sv, dop, code, cph) in enumerate(((3, 500.3, 333, 1.0), (9, -1500.3, 999, 2.5), (17, 2500.3, 1555, 4.0),
                                              (30, -3000.3, 222, 5.5))):
        eph = orb.realistic_ephemeris(erng, sv)
        sfs = orb.ephemeris_subframes(eph, 11, first_id=1, tow0=20000, seed=i)
        chans.append((sv, dop, code, cph, 0.005, sfs, 7))
    attrs = SampleProviderAttributes(FS, N)
    codes = generate_replica_prn_signals()
    seeds = [(GpsSatellite(GpsSatelliteId(c[0]), codes[GpsSatelliteId(c[0])], N // 1023), round(c[1]), c[3], c[2])
             for c in chans]
    bank = TrackerBank(seeds, attrs)
    iq_chans = [(c[0], c[1], c[2], c[3], c[4], np.concatenate([np.asarray(sf, np.int8) for sf in c[5]]), c[6]) for c in chans]
    rcv = fx.ReceiverOracle(4)
    n_checked = n_marked = 0
    worst = [0.0, 0.0, 0.0]
    fixes = []
    for k0 in range(0, 60000, 1000):
        x = nav.synth_lnav_iq(21, N, FS, k0, 1000, iq_chans, sigma=0.01)
        tt = np.array([t.chunk_times(k, FS, N) for k in range(k0, k0 + 1000)])
        recs = bank.process(x, tt[:, 0])
        bits = bank.integrate_bits(tt[:, 0], tt[:, 1])
        sub = bank.decode_subframes()
        bank.parse_subframes()
        got = bank.position_fixes(tt[:, 0])
        fixes.append(got)
        # the oracle on the device's own events and drops, as tests/test_gpu_orbit.py feeds it
        per = []
        for c in range(4):
            events = [(int(e["kind"]), tuple(int(w) for w in e["words"]), float(e["trailing_edge_receiver_timestamp"]),
                       int(bits[c][int(e["bit_index"])]["ms_index"])) for e in sub[c]]
            drops = [m for kind, _, _, m in events if kind == nav.KIND_CANNOT] + list(np.flatnonzero(recs["lost"][c])[:1])
            per.append((events, int(min(drops)) if drops else -1))
        marks = {m for ev, _ in per for _, _, _, m in ev} | set(np.flatnonzero(np.diff(got["n_ready"])) + 1)
        near = {m + d for m in marks for d in (-1, 0, 1)}
        sample = set(range(0, 1000, 97)) | near
        want = rcv.call(per, tt[:, 0], teacher=got, sample=sample)
        assert np.array_equal(got["status"], want["status"]) and np.array_equal(got["channel"], want["channel"])
        sel = np.array(sorted(m for m in sample if 0 <= m < 1000 and want[m]["status"] == fx.FIX_SOLVED), dtype=int)
        if len(sel):
            worst = [max(a, b) for a, b in zip(worst, _compare(got[sel], want[sel]))]
            n_checked += len(sel)
            n_marked += len([m for m in sel if m in near])
    all_fix = np.concatenate(fixes)
    assert (all_fix[-5000:]["status"] == fx.FIX_SOLVED).all()
    # the fixes start near 42 s; the subframes at 48 and 54 s reset the slide while fixing, and the first fix changes
    # the ready set: each contributes its millisecond and the next one at least
    assert n_checked >= 100 and n_marked >= 6, (n_checked, n_marked)
    assert bank.native.receiver_state()["repaired"] == 0
    sol = solution_from_fix(all_fix[-1])
    assert np.isfinite([sol.clock_bias, sol.receiver_pos.x, sol.receiver_pos.y, sol.receiver_pos.z]).all()
    print(f"fixing ms {int((all_fix['status'] == 1).sum())}, first at {int(np.flatnonzero(all_fix['status'] == 1)[0])}; "
          f"checked against the oracle {n_checked}, {n_marked} of them around a reset or a ready-set change; worst slide / "
          f"pseudorange {worst[0]:.3g} s, clock bias {worst[1]:.3g} s, position {worst[2]:.3g} m")
    bank.native.close()
