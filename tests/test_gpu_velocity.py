"""The velocity fix on the device (velocity.cu through gb200_tracker_velocity_fixes): the recorded fix timelines
(tests/golden/fix.npz) with Dopplers planted from the geometry of the device's own fixes, the least-squares mode on a
scripted six-channel timeline, the reference mode's raise, the device variant, the error cases, and 60 s of IQ through
TrackerBank.  Against the planted values and the float64 oracle (tests/velocity_oracle.py) within the bounds of
tests/velocity_support.py, and against the host build of the same core (tests/emu/velocity_emu.cu): only sin, cos and
atan2, in the satellite velocity and the latitude and longitude, may round differently there."""
import os

import numpy as np
import pytest

import velocity_oracle as vo
from fix_support import parse_events
from gpu_support import make_engine
from oracle import fix_oracle as fx
from oracle import nav_oracle as nav
from oracle import orbit_oracle as orb
from oracle import tracker_oracle as t
from test_gpu_fix_lsq import scripted_timeline
from velocity_support import DOP_REL, DRIFT_SS, VEL_MS, velocity_emulator

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "fix.npz")
TIMELINES = ["realistic", "three", "gate", "lost", "five", "raise"]
N, FS = 2046, 2046000
# the device against the host build: relative to the velocity's scale times GDOP, and to DOP; degrees and metres
HOST_REL, HOST_DEG, HOST_M = 1e-12, 1e-12, 1e-6
V_PLANT, DRIFT_PLANT = np.array([12.5, -40.25, 3.0]), 2.5e-9
NUMBERS = list(vo.VELOCITY_DTYPE.names[1:14])


@pytest.fixture(scope="module")
def engine(native_lib):
    e = make_engine(FS, N)
    yield e
    e.close()


@pytest.fixture(scope="module")
def emu():
    return velocity_emulator()


def rows_of(fix, obs, order, m):
    """The channels the velocity of a solved fix uses: its four, or every ready channel in the world model's order."""
    if fix["n_ready"] == 4:
        return [int(c) for c in fix["channel"]]
    return [c for c in order if (obs[c, m]["flags"] & 6) == 6]


def sat_rows(obs, params, chans, m, satellite):
    return np.array([[obs[c, m]["x"], obs[c, m]["y"], obs[c, m]["z"], *satellite(params[c, m], obs[c, m]["tow"])]
                     for c in chans])


def planted(fixes, obs, params, order):
    """[n_channels][n_ms] Dopplers that V_PLANT and DRIFT_PLANT measure at every solved fix's position (0 elsewhere)."""
    dopp = np.zeros(obs.shape)
    for m in np.flatnonzero(fixes["status"] == fx.FIX_SOLVED):
        f = fixes[m]
        chans = rows_of(f, obs, order, m)
        sat = sat_rows(obs, params, chans, m, vo.satellite_velocity)
        dopp[chans, m] = vo.dopplers(sat, (f["x"], f["y"], f["z"]), V_PLANT, DRIFT_PLANT)
    return dopp


def expected(emu, fixes, obs, params, dopp, order, sample=None):
    """(host core, oracle) records of one call, on the sampled milliseconds (None: all)."""
    satellite, compute, _ = emu
    host = np.zeros(len(fixes), dtype=vo.VELOCITY_DTYPE)
    for k in NUMBERS:
        host[k] = np.nan
    host["receiver_timestamp"] = fixes["receiver_timestamp"]
    orc = host.copy()
    ms = np.flatnonzero(fixes["status"] == fx.FIX_SOLVED)
    for m in ms if sample is None else [m for m in ms if m in sample]:
        f = fixes[m]
        chans = rows_of(f, obs, order, m)
        r, rx = (f["x"], f["y"], f["z"]), f["receiver_timestamp"]
        d = np.array([dopp[c, m] for c in chans])[:, None]
        host[m] = compute(np.hstack([sat_rows(obs, params, chans, m, satellite), d]), r, rx)
        orc[m] = vo.solve(np.hstack([sat_rows(obs, params, chans, m, vo.satellite_velocity), d]), r, rx)
    return host, orc


def compare(got, fixes, host, orc, sample=None, plant=False):
    """Status and rows against the fix records; every number against the host core (tight) and the oracle (the
    bounds), and the plants.  Returns [worst velocity, drift, DOP relative against the oracle, byte-identical records
    against the host core, records checked]."""
    assert np.array_equal(got["receiver_timestamp"], fixes["receiver_timestamp"])
    solved = fixes["status"] == fx.FIX_SOLVED
    assert (got["status"][~solved] == vo.VEL_NONE).all() and (got["n_rows"][~solved] == 0).all()
    assert all(np.isnan(got[k][~solved]).all() for k in NUMBERS)
    assert (got["status"][solved] == vo.VEL_SOLVED).all()
    assert np.array_equal(got["n_rows"][solved], fixes["n_ready"][solved])
    assert (got["reserved"] == 0).all()
    worst = [0.0, 0.0, 0.0, 0, 0]
    for m in np.flatnonzero(solved):
        if sample is not None and m not in sample:
            continue
        g, h, o = got[m], host[m], orc[m]
        assert g["status"] == h["status"] == o["status"] and g["n_rows"] == h["n_rows"] == o["n_rows"], m
        scale = max(1.0, *(abs(h[k]) for k in ("vx", "vy", "vz"))) * max(1.0, h["gdop"])
        for k in ("vx", "vy", "vz"):
            assert abs(g[k] - h[k]) <= HOST_REL * scale, (m, k, g[k], h[k])
        assert abs(g["clock_drift"] - h["clock_drift"]) <= HOST_REL * scale / vo.C_LIGHT, m
        for k in ("gdop", "pdop", "hdop", "vdop", "tdop"):
            assert abs(g[k] - h[k]) <= HOST_REL * abs(h[k]), (m, k, g[k], h[k])
        # with planted Dopplers the residuals are rounding: relative to the velocity's scale, like the velocity
        assert (np.isnan(g["residual_rms"]) and np.isnan(h["residual_rms"])) or \
            abs(g["residual_rms"] - h["residual_rms"]) <= HOST_REL * max(scale, abs(h["residual_rms"]))
        assert abs(g["latitude_deg"] - h["latitude_deg"]) <= HOST_DEG and abs(g["longitude_deg"] - h["longitude_deg"]) <= HOST_DEG
        assert abs(g["height"] - h["height"]) <= HOST_M
        worst[3] += g.tobytes() == h.tobytes()
        worst[4] += 1
        want = (V_PLANT, DRIFT_PLANT) if plant else ((o["vx"], o["vy"], o["vz"]), o["clock_drift"])
        dv = max(abs(g[k] - w) for k, w in zip(("vx", "vy", "vz"), want[0]))
        dd = abs(g["clock_drift"] - want[1])
        dop = max(abs(g[k] - o[k]) / abs(o[k]) for k in ("gdop", "pdop", "hdop", "vdop", "tdop"))
        worst[:3] = [max(worst[0], dv), max(worst[1], dd), max(worst[2], dop)]
        assert dv <= VEL_MS and dd <= DRIFT_SS and dop <= DOP_REL, (m, dv, dd, dop)
        if g["n_rows"] > 4:
            assert abs(g["residual_rms"] - o["residual_rms"]) <= DOP_REL * max(scale, o["residual_rms"])
        else:
            assert np.isnan(g["residual_rms"])
    return worst


def run_planted(engine, emu, calls, solver="reference"):
    """A timeline through one tracker, call after call: position_fixes, then velocity_fixes with planted Dopplers.
    Returns per call (velocity records, fix records), and the worst differences."""
    import torch

    from gypsum_b200 import _native

    n_ch = len(calls[0][1])
    trk = _native.Tracker(engine, list(range(n_ch)), [0.0] * n_ch, [0.0] * n_ch, [0] * n_ch)
    trk.set_fix_solver(solver)
    sv, out, worst = None, [], [0.0, 0.0, 0.0, 0, 0]
    for rx, chans in calls:
        parse_events(trk, chans, len(rx))
        fixes = trk.position_fixes(rx)
        obs, order = trk.observations(), trk.receiver_state()["order"]
        params, sv = vo.params_timeline(chans, len(rx), sv)
        dopp = planted(fixes, obs, params, order)
        d = torch.from_numpy(dopp).cuda()
        got = trk.velocity_fixes(d.data_ptr())
        host, orc = expected(emu, fixes, obs, params, dopp, order)
        w = compare(got, fixes, host, orc, plant=True)
        worst = [max(a, b) for a, b in zip(worst[:3], w[:3])] + [worst[3] + w[3], worst[4] + w[4]]
        out.append((got, fixes))
    trk.close()
    return out, worst


@pytest.mark.parametrize("name", TIMELINES)
def test_golden_timelines_planted(engine, emu, name):
    """The recorded fix timelines with Dopplers planted from each solved fix's geometry: the planted velocity and
    drift come back within the bounds, every number is the host core's (bounds for sin / cos / atan2 only) and the
    oracle's; every millisecond without a solved fix has status 0."""
    calls = fx.golden_calls(np.load(GOLDEN), name)
    out, worst = run_planted(engine, emu, calls)
    n_solved = sum(int((f["status"] == fx.FIX_SOLVED).sum()) for _, f in out)
    assert worst[4] == n_solved
    print(f"{name}: {n_solved} solved; worst velocity {worst[0]:.3g} m/s, drift {worst[1]:.3g} s/s, DOP {worst[2]:.3g} "
          f"relative; byte-identical to the host core {worst[3]} of {worst[4]}")


def test_least_squares_scripted_six_channels(engine, emu):
    """tests/test_gpu_fix_lsq.py's scripted timeline in the least-squares mode: the velocity's rows follow the ready set
    6 -> 5 -> 4 inside call 0's segment and are six again in call 1, where the chain repair recomputed fixes."""
    out, worst = run_planted(engine, emu, scripted_timeline(), solver="least_squares")
    (v0, f0), (v1, _) = out
    assert (v0["n_rows"][300:600] == 6).all() and (v0["n_rows"][600:700] == 5).all() and (v0["n_rows"][700:] == 4).all()
    assert (v0["status"][300:] == vo.VEL_SOLVED).all() and (v0["status"][:300] == vo.VEL_NONE).all()
    assert (v1["n_rows"][200:] == 6).all() and (v1["status"] == vo.VEL_SOLVED).all()
    assert np.isfinite(v0["residual_rms"][300:700]).all() and np.isnan(v0["residual_rms"][700:]).all()
    print(f"scripted: worst velocity {worst[0]:.3g} m/s, drift {worst[1]:.3g} s/s, DOP {worst[2]:.3g} relative; "
          f"byte-identical to the host core {worst[3]} of {worst[4]}")


def test_reference_mode_raise(engine, emu):
    """`five` in the reference mode: the fix raises at ms 400 and the receiver stops, so the velocity has status 0 from
    the raise on."""
    out, _ = run_planted(engine, emu, fx.golden_calls(np.load(GOLDEN), "five"))
    (v0, f0), rest = out[0], out[1:]
    assert f0["status"][400] == fx.FIX_RAISED
    assert (v0["status"][400:] == vo.VEL_NONE).all() and (v0["status"][:400][f0["status"][:400] == fx.FIX_SOLVED] == 1).all()
    assert all((v["status"] == vo.VEL_NONE).all() for v, _ in rest)


def test_device_variant_and_repeat(engine):
    """velocity_fixes_device equals velocity_fixes with the kept fixes and with a caller's fix buffer; two calls give
    identical bytes; fixes written to caller memory by position_fixes_device are read from there."""
    import torch

    from gypsum_b200 import _native

    calls = fx.golden_calls(np.load(GOLDEN), "lost")
    trk = _native.Tracker(engine, [0, 1, 2, 3], [0.0] * 4, [0.0] * 4, [0] * 4)
    rng = np.random.default_rng(3)
    n_checked = 0
    for k, (rx, chans) in enumerate(calls):
        parse_events(trk, chans, len(rx))
        d = torch.from_numpy(rng.uniform(-4000, 4000, size=(4, len(rx)))).cuda()
        size = len(rx) * _native.VELOCITY_DTYPE.itemsize
        if k % 2 == 0:
            fixes = trk.position_fixes(rx)
            fdev = torch.from_numpy(fixes.view(np.uint8).copy()).cuda()
            a = trk.velocity_fixes(d.data_ptr())
            assert a.tobytes() == trk.velocity_fixes(d.data_ptr()).tobytes()
            assert a.tobytes() == trk.velocity_fixes(d.data_ptr(), fdev.data_ptr()).tobytes()
            out = torch.empty(size, dtype=torch.uint8, device="cuda")
            trk.velocity_fixes_device(out.data_ptr(), d.data_ptr())
            torch.cuda.synchronize()
            assert out.cpu().numpy().tobytes() == a.tobytes()
        else:
            fdev = torch.empty(len(rx) * _native.FIX_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
            trk.position_fixes_device(rx, fdev.data_ptr())
            with pytest.raises(RuntimeError, match="pass that buffer"):
                trk.velocity_fixes(d.data_ptr())
            a = trk.velocity_fixes(d.data_ptr(), fdev.data_ptr())
            out = torch.empty(size, dtype=torch.uint8, device="cuda")
            trk.velocity_fixes_device(out.data_ptr(), d.data_ptr(), fdev.data_ptr())
            torch.cuda.synchronize()
            assert out.cpu().numpy().tobytes() == a.tobytes()
        n_checked += int((a["status"] == vo.VEL_SOLVED).sum())
    assert n_checked > 0
    trk.close()


def test_velocity_errors(engine):
    """ESTATE: no parse call; the parse call's fixes not computed; fixes in caller memory (above); no tracking records
    behind a parse call fed a caller's events.  EINVAL: a null output."""
    import torch

    from gypsum_b200 import _native

    trk = _native.Tracker(engine, [0, 1, 2, 3], [0.0] * 4, [0.0] * 4, [0] * 4)
    d = torch.zeros((4, 10), dtype=torch.float64, device="cuda")
    with pytest.raises(RuntimeError, match="no gb200_tracker_parse_subframes call"):
        trk.velocity_fixes(d.data_ptr())
    parse_events(trk, [([], -1)] * 4, 10)
    with pytest.raises(RuntimeError, match="not computed yet"):
        trk.velocity_fixes(d.data_ptr())
    trk.position_fixes(np.arange(10) * 0.001)
    with pytest.raises(RuntimeError, match="pass doppler_device"):
        trk.velocity_fixes()
    v = trk.velocity_fixes(d.data_ptr())
    assert (v["status"] == vo.VEL_NONE).all() and np.array_equal(v["receiver_timestamp"], np.arange(10) * 0.001)
    with pytest.raises(ValueError):
        engine._check(engine._lib.gb200_tracker_velocity_fixes(trk._h, d.data_ptr(), None, None), "velocity")
    with pytest.raises(ValueError):
        engine._check(engine._lib.gb200_tracker_velocity_fixes_device(trk._h, d.data_ptr(), None, None), "velocity")
    parse_events(trk, [([], -1)] * 4, 10)
    with pytest.raises(RuntimeError, match="not computed yet"):
        trk.velocity_fixes(d.data_ptr())
    trk.close()


def test_velocity_behind_the_tracking_kernel(engine, emu):
    """4 channels x 60 s at 2.046 Msps through TrackerBank -> integrate_bits -> decode_subframes -> parse_subframes ->
    position_fixes -> velocity_fixes in 1-s calls, the IQ of tests/test_gpu_fix.py's end-to-end test.  The Dopplers
    planted in that IQ are constants unrelated to the satellites' geometry, so the velocities mean nothing physically:
    this checks parity only.  Every record's status and rows follow the fix records; its numbers match the oracle fed
    the device's own tracker Doppler records, observations and fix records, on sampled milliseconds and around every
    subframe.  A process call after the parse call replaces the records the default Doppler reads (ESTATE)."""
    from gypsum_b200.antenna_sample_provider import SampleProviderAttributes
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import TrackerBank

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
    sv, worst, n_solved = None, [0.0, 0.0, 0.0, 0, 0], 0
    for k0 in range(0, 60000, 1000):
        x = nav.synth_lnav_iq(21, N, FS, k0, 1000, iq_chans, sigma=0.01)
        tt = np.array([t.chunk_times(k, FS, N) for k in range(k0, k0 + 1000)])
        recs = bank.process(x, tt[:, 0])
        bits = bank.integrate_bits(tt[:, 0], tt[:, 1])
        sub = bank.decode_subframes()
        bank.parse_subframes()
        fixes = bank.position_fixes(tt[:, 0])
        got = bank.velocity_fixes()
        per = []
        for c in range(4):
            events = [(int(e["kind"]), tuple(int(w) for w in e["words"]), float(e["trailing_edge_receiver_timestamp"]),
                       int(bits[c][int(e["bit_index"])]["ms_index"])) for e in sub[c]]
            drops = [m for kind, _, _, m in events if kind == nav.KIND_CANNOT] + list(np.flatnonzero(recs["lost"][c])[:1])
            per.append((events, int(min(drops)) if drops else -1))
        params, sv = vo.params_timeline(per, 1000, sv)
        marks = {m for ev, _ in per for _, _, _, m in ev}
        sample = set(range(0, 1000, 37)) | {m + d for m in marks for d in (-1, 0, 1)}
        obs, order = bank.observations(), bank.native.receiver_state()["order"]
        oracle_in = (fixes, obs, params, np.ascontiguousarray(recs["doppler"]), order)
        host, orc = expected(emu, *oracle_in, sample=sample)
        w = compare(got, fixes, host, orc, sample=sample)
        worst = [max(a, b) for a, b in zip(worst[:3], w[:3])] + [worst[3] + w[3], worst[4] + w[4]]
        n_solved += int((got["status"] == vo.VEL_SOLVED).sum())
    assert n_solved >= 5000 and worst[4] >= 100, (n_solved, worst)
    tt = np.array([t.chunk_times(k, FS, N) for k in range(60000, 60010)])
    bank.process(nav.synth_lnav_iq(21, N, FS, 60000, 10, iq_chans, sigma=0.01), tt[:, 0])
    with pytest.raises(RuntimeError, match="pass doppler_device"):
        bank.velocity_fixes()
    print(f"solved {n_solved}; checked {worst[4]}: worst velocity {worst[0]:.3g} m/s, drift {worst[1]:.3g} s/s, DOP "
          f"{worst[2]:.3g} relative; byte-identical to the host core {worst[3]}")
    bank.native.close()

