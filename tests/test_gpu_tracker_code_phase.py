"""The tracker's "samples" code-phase mode on the device (DESIGN.md §7): k_track_channels / k_track_channels_wide with
the DLL wrapped at N and k_integrate_bits stamping with code_phase / N, at every rate and at code phases across
[0, N), against the float64 tracker oracle wrapped at N (tests/code_phase_support.py); the drop-in pools of both modes
on one engine; and the chain from tracking to position fixes at 16.368 Msps on satellites at code phases of 2046 and
more, which the reference mode loses."""
import concurrent.futures
import multiprocessing

import numpy as np
import pytest

from code_phase_support import ALL_RATES, WrapOracle, amplitude, oracle_rows, planted_channels, planted_phases
from gpu_support import Attrs, EngineCache
from oracle import fix_oracle as fx
from oracle import nav_oracle as nav
from oracle import orbit_oracle as orb
from oracle import tracker_oracle as t
from tracker_support import assert_follows_reference, assert_ms_matches_oracle, start_times

pytestmark = pytest.mark.gpu
FREE_MS = 6100    # past the 6-second constellation check
ORACLE_MS = 300   # free-running oracle milliseconds per channel (about 10 ms each at 16.368 Msps)


@pytest.fixture(scope="module")
def engines(native_lib):
    cache = EngineCache()
    yield cache
    cache.close()


def _oracle_rows_parallel(jobs):
    ctx = multiprocessing.get_context("spawn")
    with concurrent.futures.ProcessPoolExecutor(max_workers=min(len(jobs), ctx.cpu_count() or 1), mp_context=ctx) as pool:
        return list(pool.map(oracle_rows, jobs))


def _bind_repeated(eng, base, n_ms):
    """Binds n_ms milliseconds of `base` repeated end to end as the engine's device IQ; returns the tensor to keep."""
    import torch

    n = eng.samples_per_ms
    reps = -(-n_ms * n // base.size)
    xd = torch.from_numpy(base.view(np.float32)).cuda().repeat(reps)[: n_ms * n * 2].contiguous()
    torch.cuda.synchronize()
    eng.bind_iq_device(xd.data_ptr(), n_ms * n)
    return xd


@pytest.mark.parametrize("s", ALL_RATES)
def test_samples_mode_keeps_every_code_phase(engines, s):
    """A samples-mode bank with channels at N - 1, on every polyphase branch and at 2046 and 2047 where N > 2046, runs
    free for 6.1 s over a 1-s recording repeated (whole-Hz Dopplers keep the carrier continuous): no channel is lost,
    the 6-second check runs, and each channel stays within two chips and a sample of its planted code phase, counted
    modulo N.  Over the first 300 ms every channel follows the oracle wrapped at N (tracker_support bounds,
    per-millisecond proofs).  The reference mode on the same IQ follows the oracle wrapped at 2046 and, at S >= 3,
    moves every channel at 2047 or more to code phase mod 2046 after millisecond 0, off its signal: the loss this mode
    removes.  (One at 2046 whose first DLL step takes it below 2046 is kept.)"""
    from gypsum_b200 import _native

    n, fs = 1023 * s, 1023000 * s
    phases = planted_phases(s)
    chans = [(sv, float(round(f)), 0.0, cp, phi, amp) for sv, f, _, cp, phi, amp in planted_channels(s, phases)]
    seeds = [(sv - 1, f, 0.0, cp) for sv, f, _, cp, _, _ in chans]
    base = t.synth_tracking_iq(500 + s, n, 1000, fs, chans)
    eng = engines(n)
    ts = start_times(FREE_MS, fs, n)
    keep = _bind_repeated(eng, base, FREE_MS)
    bank = _native.Tracker(eng, *[list(v) for v in zip(*seeds)])
    bank.set_code_phase_mode("samples")
    rec = bank.process(FREE_MS, ts)
    bank.close()
    ref = _native.Tracker(eng, *[list(v) for v in zip(*seeds)])
    rec_ref = ref.process(3, ts[:3])
    ref.close()
    del keep
    assert not rec["lost"].any()
    assert ts[6000] == 6.0
    for c, cp in enumerate(phases):
        d = (rec["code_phase"][c].astype(np.int64) - cp) % n
        assert np.minimum(d, n - d).max() <= 2 * s + 1, (c, cp)
    jobs = [(base[:ORACLE_MS * n], n, fs, (sv + 1, f, p, cp), ORACLE_MS, n) for sv, f, p, cp in seeds]
    jobs += [(base[:3 * n], n, fs, (sv + 1, f, p, cp), 3, 2046) for sv, f, p, cp in seeds]
    got = _oracle_rows_parallel(jobs)
    for c, cp in enumerate(phases):
        rows, lost_at = got[c]
        assert lost_at < 0 and len(rows) == ORACLE_MS
        assert_follows_reference(rec[c, :ORACLE_MS], rows, histories=True)
        rows_ref, _ = got[len(phases) + c]
        assert_follows_reference(rec_ref[c], rows_ref, histories=True)
        if cp >= 2047:  # at cp mod 2046 from millisecond 1 on: a multiple of 1023 samples off the signal
            d = (int(rec_ref["code_phase"][c, 1]) - cp) % n
            assert min(d, n - d) >= 1000, c
    assert (s >= 3) == any(cp >= 2047 for cp in phases)


@pytest.mark.parametrize("s", ALL_RATES)
def test_accumulator_crosses_the_wrap_teacher_forced(engines, s):
    """At an amplitude where one DLL step is several samples, each millisecond's signal one sample early of the oracle's
    code phase drives the accumulator up from N - 3 across N - 1 -> 0 (tracker.py:298-303 with the modulus N); the
    device, set to the oracle's state each millisecond, matches its correlators and loop update every millisecond."""
    from gypsum_b200 import _native

    n, fs = 1023 * s, 1023000 * s
    eng = engines(n)
    trk = _native.Tracker(eng, [24], [1500.0], [0.0], [n - 3])
    trk.set_code_phase_mode("samples")
    tr = WrapOracle(25, 1500.0, 0.0, n - 3, fs, n, wrap=n)
    tr.phase = n - 2.5
    seen = []
    for k in range(60):
        a, b = t.chunk_times(k, fs, n)
        xk = t.synth_tracking_iq(700 + k, n, 1, fs, [(25, 1500.0, 0.0, (tr.code_phase - 1) % n, 0.3, 150.0 / n)], t0=a)
        trk.set_state(0, tr.doppler, tr.carrier_phase, float(tr.phase), tr.code_phase)
        eng.upload_iq(xk)
        rec = trk.process(1, [a])[0, 0]
        r = tr.step(xk, a, b)
        assert_ms_matches_oracle(rec, r, k)
        assert abs(rec["phase_acc"] - tr.phase) <= 1e-3 and 0 <= rec["phase_acc"] < n, k
        seen.append(r["code_phase"])
        if max(seen) >= n - 1 and seen[-1] < n // 2:
            break
    assert max(seen) >= n - 1 and seen[-1] < n // 2, seen
    trk.close()


def test_bit_stamps_in_samples_mode(engines):
    """integrate_bits on a samples-mode bank at 16.368 Msps: every event equals the host integrator fed the device's
    own records through _pseudosymbol with the modulus N, timestamps bit for bit."""
    from gypsum_b200 import _native
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId
    from gypsum_b200.navigation_bit_integrator import NavigationBitIntegrator
    from gypsum_b200.tracker import BitValue, _pseudosymbol

    s, n_ms = 16, 2000
    n, fs = 1023 * s, 1023000 * s
    phases = [2046, 7777, 12345, n - 1]
    chans = [(3 + c, 700.3 - 400 * c, 0.0, cp, 0.5, amplitude(s)) for c, cp in enumerate(phases)]
    x = t.synth_tracking_iq(41, n, n_ms, fs, chans)
    tt = np.array([t.chunk_times(k, fs, n) for k in range(n_ms)])
    eng = engines(n)
    eng.upload_iq(x)
    trk = _native.Tracker(eng, [c[0] - 1 for c in chans], [round(c[1]) for c in chans], [0.0] * 4, phases)
    trk.set_code_phase_mode("samples")
    rec = trk.process(n_ms, tt[:, 0])
    events = trk.integrate_bits(n_ms, tt[:, 0], tt[:, 1])
    trk.close()
    code = {BitValue.ONE: 1, BitValue.ZERO: 0, BitValue.UNKNOWN: -1}
    for c in range(4):
        assert not rec["lost"][c].any() and (rec["code_phase"][c] >= 2000).all(), c
        integ = NavigationBitIntegrator(GpsSatelliteId(chans[c][0]))
        want = []
        for k in range(n_ms):
            for e in integ.process_pseudosymbol(tt[k, 0], _pseudosymbol(rec[c, k], tt[k, 0], tt[k, 1], n)):
                want.append((k, e.receiver_timestamp, e.trailing_edge_receiver_timestamp, code[e.bit_value]))
        got = [(int(e["ms_index"]), float(e["receiver_timestamp"]), float(e["trailing_edge_receiver_timestamp"]),
                int(e["bit_value"])) for e in events[c]]
        assert got == want and len(got) >= 90, c


def test_drop_in_pools_of_both_modes_share_one_engine(native_lib):
    """Drop-in GpsSatelliteTrackers at 16.368 Msps fed through a DeviceSampleRing, one call per millisecond: two in the
    samples mode at code phases 7777 and 12345 and one in the reference mode at 777, interleaved on one engine.  Each
    mode batches in its own pool; each tracker's pseudosymbols, stamps and loop state equal a TrackerBank of its mode,
    the stamps being its records' chunk times plus code_phase / wrap ms."""
    from gypsum_b200 import _native
    from gypsum_b200.antenna_sample_provider import AntennaSampleChunk, DeviceSampleRing, SampleProviderAttributes
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import GpsSatelliteTracker, GpsSatelliteTrackingParameters, TrackerBank, _pseudosymbol

    s, n_ms = 16, 300
    n, fs = 1023 * s, 1023000 * s
    attrs = SampleProviderAttributes(fs, n)
    plan = [(25, 1500.3, 7777, "samples"), (7, -2212.7, 777, "reference"), (12, 640.4, 12345, "samples")]
    x = t.synth_tracking_iq(51, n, n_ms, fs, [(sv, f, 0.0, cp, 0.3, amplitude(s)) for sv, f, cp, _ in plan])
    tt = np.array([t.chunk_times(k, fs, n) for k in range(n_ms)])
    codes = generate_replica_prn_signals()
    sats = {sv: GpsSatellite(GpsSatelliteId(sv), codes[GpsSatelliteId(sv)], s) for sv, *_ in plan}
    recs = []
    for sv, f, cp, mode in plan:
        bank = TrackerBank([(sats[sv], round(f), 0.0, cp)], attrs, code_phase=mode)
        recs.append(bank.process(x, tt[:, 0])[0])
        bank.native.close()
    trks = [GpsSatelliteTracker(GpsSatelliteTrackingParameters(satellite=sats[sv], current_doppler_shift=round(f),
                                                               current_carrier_wave_phase_shift=0.0,
                                                               current_prn_code_phase_shift=cp, doppler_shifts=[]),
                                attrs, keep_correlation_profiles=False, code_phase=mode) for sv, f, cp, mode in plan]
    assert trks[0]._pool is trks[2]._pool and trks[0]._pool is not trks[1]._pool
    ring = DeviceSampleRing(attrs, 10)
    got = [[] for _ in plan]
    for k in range(n_ms):
        chunk = ring.append(AntennaSampleChunk(tt[k, 0], tt[k, 1], x[k * n:(k + 1) * n]))
        for c, trk in enumerate(trks):
            ps = trk.process_samples(chunk)
            got[c].append((ps.pseudosymbol.as_val(), ps.start_of_pseudosymbol, ps.end_of_pseudosymbol))
    for c, (sv, f, cp, mode) in enumerate(plan):
        wrap = n if mode == "samples" else 2046
        want = []
        for k in range(n_ms):
            ps = _pseudosymbol(recs[c][k], tt[k, 0], tt[k, 1], wrap)
            want.append((ps.pseudosymbol.as_val(), ps.start_of_pseudosymbol, ps.end_of_pseudosymbol))
        assert got[c] == want, c
        p = trks[c].tracking_params
        assert (p.current_doppler_shift, p.current_prn_code_phase_shift, trks[c].phase) == (
            recs[c][-1]["doppler"], recs[c][-1]["code_phase"], recs[c][-1]["phase_acc"]), c
        assert not recs[c]["lost"].any() and abs(int(recs[c][-1]["code_phase"]) - cp) <= 2 * s, c
        trks[c].close()
    ring.native.close()


def test_mode_errors(engines):
    """ESTATE once a bank or a pool has tracked (or a bank has integrated bits), EINVAL and ValueError for an unknown
    mode; before that the mode may be set again."""
    from gypsum_b200 import _native
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import GpsSatelliteTracker, GpsSatelliteTrackingParameters, TrackerBank

    n = 2046
    eng = engines(n)
    eng.upload_iq(np.zeros(2 * n, dtype=np.complex64))
    bank = _native.Tracker(eng, [0], [0.0], [0.0], [5])
    with pytest.raises(ValueError, match="code-phase mode"):
        bank.set_code_phase_mode("chips")
    assert eng._lib.gb200_tracker_set_code_phase_mode(bank._h, 2) == _native.EINVAL
    assert eng._lib.gb200_tracker_set_code_phase_mode(None, 1) == _native.EINVAL
    bank.set_code_phase_mode("samples")
    bank.set_code_phase_mode("reference")
    bank.process(1, [0.0])
    with pytest.raises(RuntimeError, match="first tracking call"):
        bank.set_code_phase_mode("samples")
    assert eng._lib.gb200_tracker_set_code_phase_mode(bank._h, 1) == _native.ESTATE
    bank.close()
    import torch

    out = torch.empty(_native.TRACK_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    bank = _native.Tracker(eng, [0], [0.0], [0.0], [5])
    bank.process_device(1, np.zeros(1), out.data_ptr())
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="first tracking call"):
        bank.set_code_phase_mode("samples")
    bank.close()
    recs = np.zeros(20, _native.TRACK_DTYPE)
    recs["symbol"] = 1
    dev = torch.from_numpy(recs.view(np.uint8)).cuda()
    bank = _native.Tracker(eng, [0], [0.0], [0.0], [5])
    bank.integrate_bits(20, np.arange(20) * 1e-3, np.arange(1, 21) * 1e-3, dev.data_ptr())
    with pytest.raises(RuntimeError, match="first tracking call"):
        bank.set_code_phase_mode("samples")
    bank.close()
    pool = _native.Tracker.pool(eng, 2)
    pool.set_code_phase_mode("samples")
    pool.reset_channel(1, 0, 0.0, 0.0, 5)
    pool.process_channels([1], 1, [0.0])
    with pytest.raises(RuntimeError, match="first tracking call"):
        pool.set_code_phase_mode("reference")
    pool.close()
    codes = generate_replica_prn_signals()
    sat = GpsSatellite(GpsSatelliteId(1), codes[GpsSatelliteId(1)], 2)
    with pytest.raises(ValueError, match="code-phase mode"):
        TrackerBank([(sat, 0.0, 0.0, 5)], Attrs(2046000, n), code_phase="chips")
    params = GpsSatelliteTrackingParameters(satellite=sat, current_doppler_shift=0.0, current_carrier_wave_phase_shift=0.0,
                                            current_prn_code_phase_shift=5, doppler_shifts=[])
    with pytest.raises(ValueError, match="code-phase mode"):
        GpsSatelliteTracker(params, Attrs(2046000, n), code_phase="chips")


E2E_PHASES = [2400, 8000, 12000, 16000]  # at 16.368 Msps; / 8 at 2.046 Msps
POS_M_16368 = 2e-5
# how far the two rates' subframe stamps may differ: each rate's DLL drifts from the planted phase on its own over the
# minute (the reference's loop; 3.4 chips apart on one channel), far less than the >= 1.03 ms the reference's stamping
# would put between them
STAMP_AGREEMENT_S = 2e-5


def _lnav_scenario(n):
    """test_gpu_fix's four satellites with consistent ephemerides, at code phases E2E_PHASES scaled to n samples per
    ms and the same signal-to-noise ratio per millisecond at every rate."""
    erng = np.random.default_rng(11)
    chans = []
    for i, (sv, dop, cph) in enumerate(((3, 500.3, 1.0), (9, -1500.3, 2.5), (17, 2500.3, 4.0), (30, -3000.3, 5.5))):
        eph = orb.realistic_ephemeris(erng, sv)
        sfs = orb.ephemeris_subframes(eph, 11, first_id=1, tow0=20000, seed=i)
        chans.append((sv, dop, E2E_PHASES[i] * n // 16368, cph, 0.005 * np.sqrt(2046 / n), sfs, 7))
    return chans


def _run_lnav(n, per_second):
    """60 s of the scenario through every bank in 1-s calls; per_second(k0, x, tt) runs after each upload."""
    fs = 1000 * n
    chans = _lnav_scenario(n)
    iq_chans = [(c[0], c[1], c[2], c[3], c[4], np.concatenate([np.asarray(sf, np.int8) for sf in c[5]]), c[6]) for c in chans]
    for k0 in range(0, 60000, 1000):
        x = nav.synth_lnav_iq(21, n, fs, k0, 1000, iq_chans, sigma=0.01)
        tt = np.array([t.chunk_times(k, fs, n) for k in range(k0, k0 + 1000)])
        per_second(k0, x, tt)
    return chans


def _seeds(chans, n):
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite

    codes = generate_replica_prn_signals()
    return [(GpsSatellite(GpsSatelliteId(c[0]), codes[GpsSatelliteId(c[0])], n // 1023), round(c[1]), c[3], c[2])
            for c in chans]


def test_position_fixes_at_16368_ksps_from_code_phases_past_2046(native_lib):
    """4 channels x 60 s at 16.368 Msps, code phases 2400 to 16000, through a samples-mode TrackerBank -> integrate_bits
    -> decode_subframes -> parse_subframes -> position_fixes in 1-s calls: no channel is lost, every decoded subframe is
    a planted one, at least a whole 6-s subframe segment of milliseconds is fixed, and every record matches the fix
    oracle fed the device's own events and drops within test_gpu_fix's bounds, the position within 2e-5 m.  A
    reference-mode bank on the same IQ moves every channel off its signal after millisecond 0; a default bank equals it
    byte for byte (records, bits, subframes).  The same scenario at 2.046 Msps with the code phases / 8 gives
    subframes whose trailing-edge stamps agree with these within 20 us: each rate's DLL drifts a few chips from the
    planted phase on its own over the minute, while stamping cp / 2046 at 16.368 Msps would put them 1.03 to 6.8 ms
    apart."""
    from gypsum_b200.antenna_sample_provider import SampleProviderAttributes
    from gypsum_b200.tracker import TrackerBank
    from fix_support import BIAS_S, slide_tol

    n = 16368
    chans = _lnav_scenario(n)
    attrs = SampleProviderAttributes(1000 * n, n)
    seeds = _seeds(chans, n)
    bank = TrackerBank(seeds, attrs, code_phase="samples")
    ref = TrackerBank(seeds, attrs, code_phase="reference")
    dflt = TrackerBank(seeds, attrs)
    rcv = fx.ReceiverOracle(4)
    fixes, subframes, ref_off = [], [[] for _ in range(4)], [0] * 4
    lost = [[] for _ in range(4)]
    n_checked = 0
    worst_m = [0.0]

    def per_second(k0, x, tt):
        nonlocal n_checked
        recs = bank.process(x, tt[:, 0])
        bits = bank.integrate_bits(tt[:, 0], tt[:, 1])
        sub = bank.decode_subframes()
        bank.parse_subframes()
        got = bank.position_fixes(tt[:, 0])
        fixes.append(got)
        per = []
        for c in range(4):
            subframes[c] += [e for e in sub[c] if int(e["kind"]) == nav.KIND_SUBFRAME]
            lost[c] += [k0 + int(k) for k in np.flatnonzero(recs["lost"][c] == 1)]
            events = [(int(e["kind"]), tuple(int(w) for w in e["words"]), float(e["trailing_edge_receiver_timestamp"]),
                       int(bits[c][int(e["bit_index"])]["ms_index"])) for e in sub[c]]
            drops = [m for kind, _, _, m in events if kind == nav.KIND_CANNOT] + list(np.flatnonzero(recs["lost"][c])[:1])
            per.append((events, int(min(drops)) if drops else -1))
        marks = {m for ev, _ in per for _, _, _, m in ev} | set(np.flatnonzero(np.diff(got["n_ready"])) + 1)
        sample = set(range(0, 1000, 97)) | {m + d for m in marks for d in (-1, 0, 1)}
        want = rcv.call(per, tt[:, 0], teacher=got, sample=sample)
        assert np.array_equal(got["status"], want["status"]) and np.array_equal(got["channel"], want["channel"])
        sel = np.array(sorted(m for m in sample if 0 <= m < 1000 and want[m]["status"] == fx.FIX_SOLVED), dtype=int)
        if len(sel):
            g, w = got[sel], want[sel]
            for key in ("slide_in", "slide_out", "pseudorange"):
                tol = slide_tol(w["slide_in"])
                assert (np.abs(g[key] - w[key]).reshape(len(sel), -1).max(axis=1) <= tol).all(), key
            assert np.abs(g["clock_bias"] - w["clock_bias"]).max() <= BIAS_S
            worst_m[0] = max(worst_m[0], max(float(np.abs(g[k] - w[k]).max()) for k in "xyz"))
            n_checked += len(sel)
        out = []
        for b in (ref, dflt):
            r = b.process(x, tt[:, 0])
            out.append((r, b.integrate_bits(tt[:, 0], tt[:, 1]), b.decode_subframes()))
        (r0, b0, s0), (r1, b1, s1) = out
        assert r0.tobytes() == r1.tobytes()
        for c in range(4):
            assert b0[c].tobytes() == b1[c].tobytes() and s0[c].tobytes() == s1[c].tobytes(), c
            if k0 == 0:  # at cp mod 2046 from millisecond 1 on: a multiple of 1023 samples off the signal
                d = (int(r0["code_phase"][c, 1]) - E2E_PHASES[c]) % n
                ref_off[c] = min(d, n - d)

    _run_lnav(n, per_second)
    all_fix = np.concatenate(fixes)
    solved = np.flatnonzero(all_fix["status"] == fx.FIX_SOLVED)
    # a whole 6-s subframe segment of fixes; later segments need every channel's next subframe, which the reference's
    # loop gains at 16.368 Msps do not decode every time (the planted subframes come back, not all of them)
    assert len(solved) >= 6000 and n_checked >= 60 and not any(lost), (len(solved), lost, [len(v) for v in subframes])
    # slides, pseudoranges and clock bias hold test_gpu_fix's bounds; the position, whose Newton steps round differently
    # in the two solvers, is held to 2e-5 m here (test_gpu_fix: 2e-6 m): with these four satellites' geometry the same
    # rounding moves it by up to 1.1e-5 m
    assert worst_m[0] <= POS_M_16368, worst_m
    print(f"fixing ms {int((all_fix['status'] == 1).sum())}, checked {n_checked}, worst position {worst_m[0]:.3g} m")
    for c in range(4):
        planted = [list(sf) for sf in chans[c][5]]
        assert len(subframes[c]) >= 4 and all(_native_bits(e) in planted for e in subframes[c]), c
        assert ref_off[c] >= 1000, c
    for b in (bank, ref, dflt):
        b.native.close()

    # the same delay at 2.046 Msps
    n2 = 2046
    chans2 = _lnav_scenario(n2)
    assert [c[2] * 8 for c in chans2] == E2E_PHASES
    low = TrackerBank(_seeds(chans2, n2), SampleProviderAttributes(1000 * n2, n2), code_phase="samples")
    low_sub = [[] for _ in range(4)]

    def per_second_low(k0, x, tt):
        low.process(x, tt[:, 0])
        low.integrate_bits(tt[:, 0], tt[:, 1])
        for c, ev in enumerate(low.decode_subframes()):
            low_sub[c] += [e for e in ev if int(e["kind"]) == nav.KIND_SUBFRAME]

    _run_lnav(n2, per_second_low)
    low.native.close()
    for c in range(4):
        hi = {tuple(_native_bits(e)): float(e["trailing_edge_receiver_timestamp"]) for e in subframes[c]}
        pairs = [(hi[tuple(_native_bits(e))], float(e["trailing_edge_receiver_timestamp"])) for e in low_sub[c]
                 if tuple(_native_bits(e)) in hi]
        assert len(pairs) >= 3, c
        worst = max(abs(a - b) for a, b in pairs)
        # stamping cp / 2046 at 16.368 Msps would put these subframes this far from the 2.046-Msps ones
        reference_offset = E2E_PHASES[c] * (1 / 2046 - 1 / 16368) * 1e-3
        assert reference_offset >= 1e-3 and worst <= STAMP_AGREEMENT_S <= reference_offset / 50, (c, worst)


def _native_bits(event):
    from gypsum_b200 import _native

    return _native.subframe_bits(event)
