"""The position fix's least-squares mode on the device (fix.cu through gb200_tracker_position_fixes after
gb200_tracker_set_fix_solver): the golden timelines, a scripted timeline of six channels whose ready set goes from 6 to 5
to 4 inside one segment, returns, and takes a receiver-clock jump, and 60 s of IQ through TrackerBank.  Against the
least-squares oracle (tests/fix_lsq_oracle.py) within the bounds of tests/fix_support.py, against the model of the
passes (every record bit for bit, and the repair count), and against the reference mode up to the first five-ready
millisecond (byte for byte)."""
import os

import numpy as np
import pytest

import fix_lsq_oracle as lo
from fix_support import (BIAS_S, MANY_BIAS_S, MANY_POS_M, MANY_SLIDE_ULPS, POS_M, SLIDE_ULPS, fix_emulator, parse_events,
                         ready_rows, run_calls, scripted_timeline)
from gpu_support import make_engine
from oracle import fix_oracle as fx
from oracle import nav_oracle as nav
from oracle import orbit_oracle as orb
from oracle import tracker_oracle as t

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, FS = 2046, 2046000
GOLDEN = [("fix", "realistic"), ("fix", "lost"), ("fix", "five"), ("fix", "raise"), ("fix_repair", "gap_five"),
          ("fix_repair", "gap_mid"), ("fix_repair", "singular")]


@pytest.fixture(scope="module")
def engine(native_lib):
    e = make_engine(FS, N)
    yield e
    e.close()


@pytest.fixture(scope="module")
def lsq_emu():
    return fix_emulator()


def _check(calls, got_calls, ref_calls, lsq_emu):
    """Against the oracle, the model of the passes and the reference-mode run; returns (first five-ready (call, ms),
    worst slide ulp / clock bias / position, repaired per call)."""
    rcv = lo.ReceiverOracle(len(calls[0][1]))
    carried, repaired, worst, first5, reference_left = None, 0, [0.0, 0.0, 0.0], None, True
    per_call = []
    for c, ((rx, chans), (got, obs, state), (ref, _, _)) in enumerate(zip(calls, got_calls, ref_calls)):
        want = rcv.call(chans, rx)
        assert np.array_equal(got["status"], want["status"]), c
        assert np.array_equal(got["n_ready"], want["n_ready"]) and np.array_equal(got["channel"], want["channel"]), c
        # byte for byte the reference mode's records up to the first five-ready millisecond
        five = np.flatnonzero((want["n_ready"] >= 5) & np.isin(want["status"], [fx.FIX_SOLVED, fx.FIX_RAISED]))
        if reference_left:
            end = five[0] if len(five) else len(got)
            assert got[:end].tobytes() == ref[:end].tobytes(), c
            if len(five):
                first5, reference_left = (c, int(five[0])), False
        fixing = np.flatnonzero(np.isin(want["status"], [fx.FIX_SOLVED, fx.FIX_RAISED]))
        solved = np.flatnonzero(want["status"] == fx.FIX_SOLVED)
        pos_m, bias_s, ulps = (MANY_POS_M, MANY_BIAS_S, MANY_SLIDE_ULPS) if not reference_left else (POS_M, BIAS_S, SLIDE_ULPS)
        for k in ("slide_in", "slide_out"):
            d = np.abs(got[k][fixing] - want[k][fixing]) / (2.0 ** -52 * np.abs(want[k][fixing]))
            assert (d <= ulps).all(), k
            worst[0] = max([worst[0], *d])
        if len(solved):
            worst[1] = max(worst[1], float(np.abs(got["clock_bias"][solved] - want["clock_bias"][solved]).max()))
            worst[2] = max([worst[2], *(float(np.abs(got[k][solved] - want[k][solved]).max()) for k in "xyz")])
            assert worst[1] <= bias_s and worst[2] <= pos_m, worst
        assert np.isnan(got["x"][got["status"] != fx.FIX_SOLVED]).all()
        # the model of the passes on the device's own observations: every record bit for bit, and the repair count
        rows = {m: ready_rows(obs, state["order"], m) for m in fixing}
        assert all(len(rows[m]) == want[m]["n_ready"] for m in fixing)
        model = lo.device_passes(lsq_emu, want, rows, rcv.resets, carried)
        carried = model["slide"]
        assert sorted(model["out"]) == list(fixing)
        for m in fixing:
            p = model["out"][m]
            assert p.tobytes()[:88] == got[m].tobytes()[:88] and p["status"] == got[m]["status"], (c, m)
        repaired += len(model["repaired"])
        assert state["repaired"] == repaired, (c, state["repaired"], repaired)
        per_call.append((model["first_miss"], len(model["repaired"])))
    st = got_calls[-1][2]
    assert st["order"] == rcv.order and st["stopped"] == rcv.stopped
    if rcv.slide is not None:
        assert abs(st["slide"] - rcv.slide) <= MANY_SLIDE_ULPS * 2.0 ** -52 * abs(rcv.slide)
    return first5, worst, per_call


@pytest.mark.parametrize("name", GOLDEN, ids=[n for _, n in GOLDEN])
def test_golden_timelines_least_squares(engine, lsq_emu, name):
    """The recorded timelines in the least-squares mode.  Status, ready count and rows are the least-squares oracle's;
    the numbers are within the bounds; every record before the first five-ready millisecond is the reference mode's
    byte for byte; each record is the model of the passes' bit for bit, and the repair count is the model's.  In `five`
    and `gap_five` the fixes go on past ms 400, where the reference mode stops."""
    z = np.load(os.path.join(ROOT, "tests", "golden", f"{name[0]}.npz"))
    calls = fx.golden_calls(z, name[1])
    got = run_calls(engine, calls, solver="least_squares")
    ref = run_calls(engine, calls, solver="reference")
    first5, worst, per_call = _check(calls, got, ref, lsq_emu)
    if name[1] in ("five", "gap_five"):
        assert first5 == (0, 400)
        assert (got[0][0]["status"][400:] == fx.FIX_SOLVED).all() and (got[1][0]["status"] == fx.FIX_SOLVED).all()
        assert (ref[0][0]["status"][401:] == fx.FIX_STOPPED).all()
    if name[1] == "singular":
        assert np.flatnonzero(got[0][0]["status"] == fx.FIX_RAISED).tolist() == [300] and got[0][2]["stopped"]
    print(f"{name[1]}: first five-ready {first5}; (first miss, repaired) per call {per_call}; worst slide "
          f"{worst[0]:.3g} ulp, clock bias {worst[1]:.3g} s, position {worst[2]:.3g} m")


def test_scripted_six_channels(engine, lsq_emu):
    """scripted_timeline(): the ready set goes 6 -> 5 -> 4 inside call 0's first fixing segment, channels 4 and 5
    return with call 1's subframe, and the clock jump in call 1 makes the repair solve six rows.  Checked as the golden
    timelines are."""
    calls = scripted_timeline()
    got = run_calls(engine, calls, solver="least_squares")
    ref = run_calls(engine, calls, solver="reference")
    first5, worst, per_call = _check(calls, got, ref, lsq_emu)
    r0, r1 = got[0][0], got[1][0]
    assert first5 == (0, 300)
    assert (r0["n_ready"][300:600] == 6).all() and (r0["n_ready"][600:700] == 5).all()
    assert (r0["n_ready"][700:] == 4).all() and (r0["status"][300:] == fx.FIX_SOLVED).all()
    assert (r1["n_ready"][200:] == 6).all() and (r1["status"] == fx.FIX_SOLVED).all()
    assert per_call[1][1] > 0 and got[1][2]["repaired"] > got[0][2]["repaired"]
    assert ref[0][0]["status"][300] == fx.FIX_RAISED and (ref[0][0]["status"][301:] == fx.FIX_STOPPED).all()
    print(f"scripted: (first miss, repaired) per call {per_call}; worst slide {worst[0]:.3g} ulp, clock bias "
          f"{worst[1]:.3g} s, position {worst[2]:.3g} m")


def test_fix_solver_errors(engine):
    from gypsum_b200 import _native

    trk = _native.Tracker(engine, [0, 1, 2, 3], [0.0] * 4, [0.0] * 4, [0] * 4)
    with pytest.raises(ValueError, match="fix solver"):
        trk.set_fix_solver("svd")
    with pytest.raises(ValueError):
        engine._check(engine._lib.gb200_tracker_set_fix_solver(trk._h, 7), "gb200_tracker_set_fix_solver")
    trk.set_fix_solver("least_squares")
    trk.set_fix_solver("reference")  # as often as wanted before the first fix call
    parse_events(trk, [([], -1)] * 4, 10)
    trk.position_fixes(np.arange(10) * 0.001)
    with pytest.raises(RuntimeError, match="first fix call"):
        trk.set_fix_solver("least_squares")
    trk.close()


def test_least_squares_behind_the_tracking_kernel(engine):
    """6 channels x 60 s at 2.046 Msps through TrackerBank(fix_solver="least_squares") -> integrate_bits ->
    decode_subframes -> parse_subframes -> position_fixes in 1-s calls, as tests/test_gpu_fix.py runs four.  Every
    record's status, ready count and rows match the least-squares oracle fed the device's own events and drops; its
    numbers match the oracle teacher-forced with the record's slide_in, on sampled milliseconds and around every reset
    and ready-set change.  The last seconds fix on every millisecond with five or more ready (the oracle, fed the same
    events, agrees on which).  A reference-mode bank on the same IQ stops at its first five-ready millisecond."""
    from gypsum_b200.antenna_sample_provider import SampleProviderAttributes
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import TrackerBank
    from gypsum_b200.world_model import solution_from_fix

    erng = np.random.default_rng(13)
    chans = []
    for i, (sv, dop, code, cph) in enumerate(((3, 500.3, 333, 1.0), (9, -1500.3, 999, 2.5), (17, 2500.3, 1555, 4.0),
                                              (30, -3000.3, 222, 5.5), (12, 1200.3, 1777, 0.5),
                                              (22, -700.3, 600, 3.0))):
        eph = orb.realistic_ephemeris(erng, sv)
        sfs = orb.ephemeris_subframes(eph, 11, first_id=1, tow0=20000, seed=i)
        chans.append((sv, dop, code, cph, 0.005, sfs, 7))
    attrs = SampleProviderAttributes(FS, N)
    codes = generate_replica_prn_signals()
    seeds = [(GpsSatellite(GpsSatelliteId(c[0]), codes[GpsSatelliteId(c[0])], N // 1023), round(c[1]), c[3], c[2])
             for c in chans]
    bank = TrackerBank(seeds, attrs, fix_solver="least_squares")
    ref_bank = TrackerBank(seeds, attrs)
    iq_chans = [(c[0], c[1], c[2], c[3], c[4], np.concatenate([np.asarray(sf, np.int8) for sf in c[5]]), c[6]) for c in chans]
    n_ch = len(chans)
    rcv = lo.ReceiverOracle(n_ch)
    n_checked = n_marked = 0
    worst = [0.0, 0.0, 0.0]
    fixes, ref_fixes = [], []
    for k0 in range(0, 60000, 1000):
        x = nav.synth_lnav_iq(21, N, FS, k0, 1000, iq_chans, sigma=0.01)
        tt = np.array([t.chunk_times(k, FS, N) for k in range(k0, k0 + 1000)])
        for b in (ref_bank, bank):
            recs = b.process(x, tt[:, 0])
            bits = b.integrate_bits(tt[:, 0], tt[:, 1])
            sub = b.decode_subframes()
            b.parse_subframes()
            (fixes if b is bank else ref_fixes).append(b.position_fixes(tt[:, 0]))
        got = fixes[-1]
        per = []
        for c in range(n_ch):
            events = [(int(e["kind"]), tuple(int(w) for w in e["words"]), float(e["trailing_edge_receiver_timestamp"]),
                       int(bits[c][int(e["bit_index"])]["ms_index"])) for e in sub[c]]
            drops = [m for kind, _, _, m in events if kind == nav.KIND_CANNOT] + list(np.flatnonzero(recs["lost"][c])[:1])
            per.append((events, int(min(drops)) if drops else -1))
        marks = {m for ev, _ in per for _, _, _, m in ev} | set(np.flatnonzero(np.diff(got["n_ready"])) + 1)
        near = {m + d for m in marks for d in (-1, 0, 1)}
        sample = set(range(0, 1000, 97)) | near
        want = rcv.call(per, tt[:, 0], teacher=got, sample=sample)
        assert np.array_equal(got["status"], want["status"]) and np.array_equal(got["channel"], want["channel"])
        assert np.array_equal(got["n_ready"], want["n_ready"])
        sel = np.array(sorted(m for m in sample if 0 <= m < 1000 and want[m]["status"] == fx.FIX_SOLVED), dtype=int)
        for m in sel:
            g, w = got[m], want[m]
            many = w["n_ready"] > 4
            pos_m, bias_s, ulps = (MANY_POS_M, MANY_BIAS_S, MANY_SLIDE_ULPS) if many else (POS_M, BIAS_S, SLIDE_ULPS)
            ds = abs(g["slide_out"] - w["slide_out"]) / (2.0 ** -52 * abs(w["slide_out"]))
            db, dp = abs(g["clock_bias"] - w["clock_bias"]), max(abs(g[k] - w[k]) for k in "xyz")
            assert g["slide_in"] == w["slide_in"] and ds <= ulps and db <= bias_s and dp <= pos_m, (k0, m, ds, db, dp)
            worst = [max(worst[0], ds), max(worst[1], db), max(worst[2], dp)]
        n_checked += len(sel)
        n_marked += len([m for m in sel if m in near])
    all_fix, all_ref = np.concatenate(fixes), np.concatenate(ref_fixes)
    # every millisecond of the last 5 s fixed over more than four rows, where the reference mode has stopped
    assert (all_fix[-5000:]["status"] == fx.FIX_SOLVED).all() and (all_fix[-5000:]["n_ready"] > 4).all()
    assert n_checked >= 100 and n_marked >= 6, (n_checked, n_marked)
    five = np.flatnonzero((all_ref["n_ready"] >= 5) & (all_ref["status"] != fx.FIX_NONE))
    assert len(five) and all_ref[five[0]]["status"] == fx.FIX_RAISED
    assert (all_ref["status"][five[0] + 1:] == fx.FIX_STOPPED).all()
    sol = solution_from_fix(all_fix[-1])
    assert np.isfinite([sol.clock_bias, sol.receiver_pos.x, sol.receiver_pos.y, sol.receiver_pos.z]).all()
    print(f"fixing ms {int((all_fix['status'] == 1).sum())}, first at {int(np.flatnonzero(all_fix['status'] == 1)[0])}; "
          f"reference mode raised at {int(five[0])}; checked against the oracle {n_checked}, {n_marked} of them around "
          f"a reset or a ready-set change; worst slide {worst[0]:.3g} ulp, clock bias {worst[1]:.3g} s, position "
          f"{worst[2]:.3g} m; repaired {bank.native.receiver_state()['repaired']}; ready counts of the last 5 s "
          f"{np.bincount(all_fix[-5000:]['n_ready']).tolist()}")
    bank.native.close()
    ref_bank.native.close()
