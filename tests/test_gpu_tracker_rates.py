"""GPU tracking at every rate the engine acquires at other than 2.046 / 4.092 Msps: k_track_channels at S = 1, 3 and
k_track_channels_wide at S = 5 .. 16 (tracker.cu), against the tracker oracle and the live reference's trajectories
(tests/golden/tracker_fs1/fs8/fs16/fs16_long.npz).  Same bounds as tests/test_gpu_tracker.py
(tests/tracker_support.py)."""
import numpy as np
import pytest

from gpu_support import Attrs, EngineCache, run_child
from oracle import gypsum_oracle as o
from oracle import tracker_oracle as t
from tracker_support import assert_follows_reference, assert_ms_matches_oracle, load_tracker_case, start_times

pytestmark = pytest.mark.gpu
RATES = [1, 3, 5, 6, 8, 10, 12, 16]
N16, FS16 = 16368, 16368000

_FIRST_RUN_SCRIPT = r"""
import sys
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
from gpu_support import make_engine
from gypsum_b200 import _native
from oracle import tracker_oracle as t
from tracker_support import start_times

for s in (1, 3, 5, 16):
    n, fs = 1023 * s, 1023000 * s
    x = t.synth_tracking_iq(7, n, 20, fs, [(12, 640.4, 0.0, 1501, 0.7, 0.004)])
    eng = make_engine(fs, n)
    eng.upload_iq(x)
    trk = _native.Tracker(eng, [11], [640.0], [0.0], [1501])
    rec = trk.process(20, start_times(20, fs, n))[0]
    tr = t.TrackerOracle(12, 640.0, 0.0, 1501, fs, n)
    want = [tr.step(x[k * n:(k + 1) * n], *t.chunk_times(k, fs, n))["symbol"] for k in range(20)]
    assert not rec["lost"].any() and list(rec["symbol"]) == want, s
    trk.close()
    eng.close()
print("rates ok")
"""


def test_first_run_of_the_new_instantiations_in_a_child_process(native_lib):
    """Runs first, in its own process, so that a fault in a never-exercised kernel cannot disturb the CUDA context of
    the tests below."""
    run_child(_FIRST_RUN_SCRIPT, ok="rates ok")


@pytest.fixture(scope="module")
def engines(native_lib):
    cache = EngineCache()
    yield cache
    cache.close()


def _code_phase_geometry(s):
    """(name, code phase) of every edge of the early / prompt / late lags at S = s: phases 0 and N - 1, where p -+ 1 wraps;
    one phase on every polyphase branch p mod S; phases of N and above at S = 1; and the negative and >= 2046 phases that
    int() of an overshooting DLL accumulator gives (tracker.py:298-303)."""
    n = 1023 * s
    cases = [("zero", 0), ("one", 1), ("n-2", n - 2), ("n-1", n - 1)]
    cases += [(f"branch{r}", s * ((311 + 97 * r) % 1023) + r) for r in range(s)]
    cases += [("p2045", 2045)] + ([(f"p{p}", p) for p in (1023, 1024, 1535, 2044)] if s == 1 else [])
    cases += [("minus1", -1), ("minus2", -2), ("p2046", 2046), ("p2047", 2047)]
    seen, out = set(), []
    for name, p in cases:
        if p not in seen:
            seen.add(p)
            out.append(pytest.param(s, name, p, id=f"{s}-{name}"))
    return out


def _assert_named_edge(s, name, p):
    n = 1023 * s
    if name == "zero":
        assert p % n == 0  # early lag wraps to N - 1
    elif name == "n-1":
        assert p % n == n - 1  # late lag wraps to 0
    elif name.startswith("branch"):
        assert p % s == int(name[6:]) and 0 <= p < n  # prompt on branch r, E / L on its neighbours
    elif name.startswith("minus"):
        assert p < 0
    elif name in ("p2046", "p2047"):
        assert p >= 2046
    elif s == 1 and name.startswith("p"):
        assert p >= n  # past N at 1.023 Msps: np.roll is modular


GEOMETRY = [c for s in [1, 2, 3, 4, 5, 6, 8, 10, 12, 16] for c in _code_phase_geometry(s)]


@pytest.mark.parametrize("s,name,p", GEOMETRY)
def test_teacher_forced_correlators_at_every_rate(engines, s, name, p):
    """Each millisecond starts from the oracle's loop state with code phase p and the DLL accumulator the reference's
    int() and % 2046 leave with it: early / late / prompt outputs, the updated state and |prompt profile|.  The signal
    sits at p, p - 1 and p + 1, so the prompt, the early or the late tap is the peak: the last two at an amplitude
    that makes the planted lag the peak in every millisecond, the first at the one the golden rates use (at the prompt,
    |E| and |L| are nearly equal and their difference must stay above float32 rounding)."""
    from gypsum_b200 import _native

    _assert_named_edge(s, name, p)
    n, fs = 1023 * s, 1023000 * s
    phase = p + 0.3 if p >= 0 else p - 0.3
    acc = phase % 2046  # int(phase) == p
    assert int(phase) == p
    eng = engines(n)
    trk = _native.Tracker(eng, [24], [1500.0], [0.0], [p])
    tr = t.TrackerOracle(25, 1500.0, 0.0, p, fs, n)
    for d in (0, -1, 1):
        amp = 0.01 if d else (0.004 if s < 8 else 0.002)
        x = t.synth_tracking_iq(100 + s + d, n, 4, fs, [(25, 1500.3, 0.0, p + d, 0.3, amp)])
        for k in range(4):
            a, b = t.chunk_times(k, fs, n)
            tr.code_phase, tr.phase = p, acc
            trk.set_state(0, tr.doppler, tr.carrier_phase, acc, p)
            xk = x[k * n:(k + 1) * n]
            eng.upload_iq(xk)
            rec, prof = trk.process(1, [a], want_profiles=True)
            y = xk * np.exp(-1j * (2 * np.pi * tr.doppler * (tr.t1ms + a) + tr.carrier_phase))
            ref = np.abs(o.correlate_1ms(y, np.roll(tr.prn, p)))
            r = tr.step(xk, a, b)
            assert_ms_matches_oracle(rec[0, 0], r, (d, k))
            if d:  # the early (d = -1) or late tap is the peak, at rolled index N - 1 or 1
                assert r["peak_offset"] == d % n, (d, k)
                tap = r["early"] if d < 0 else r["late"]
                assert abs(abs(tap) - abs(r["peak"])) <= 1e-9 * abs(r["peak"]), (d, k)
            assert np.abs(prof[0, 0] - ref).max() <= 1e-5 * ref.max(), (d, k)
    trk.close()


@pytest.mark.parametrize("name", ["fs1", "fs8", "fs16", "fs16_long"])
def test_free_running_matches_reference_at_other_rates(engines, name):
    from gypsum_b200 import _native

    z, ch, x, n, fs, tt = load_tracker_case(name)
    init, rows = z["init"], z["rows"]
    n_ms = len(rows)
    eng = engines(n)
    trk = _native.Tracker(eng, [ch[0] - 1], [init[0]], [init[1]], [int(init[2])])
    eng.upload_iq(x)
    rec = trk.process(n_ms, tt[:n_ms, 0])[0]
    trk.close()
    assert_follows_reference(rec, rows, histories=True)
    assert np.array_equal(rec["doppler"] != rec["doppler_hist"], rows[:, 6] != rows[:, 12])
    if name == "fs16":  # sigma 0.01: the reference reaches is_locked(); the device decides the same milliseconds
        tr = t.TrackerOracle(ch[0], init[0], init[1], int(init[2]), fs, n)
        want = np.array([tr.step(x[k * n:(k + 1) * n], *tt[k])["locked"] for k in range(n_ms)])
        assert want.sum() > 0 and rec["locked"].sum() > 0
        assert np.count_nonzero(rec["locked"].astype(bool) != want) <= n_ms // 200
    if name == "fs16_long":  # sigma 0.02: never locked (I-pole variance ~ sigma^2 N / 2 > 2); the 6-s check passes
        assert n_ms > 6000 and rec["locked"].sum() == 0


def test_bank_and_profile_at_16368_ksps(engines):
    """Several channels over one stream == each channel alone; |prompt profile| matches the oracle."""
    from gypsum_b200 import _native

    chans = [(25, 1500.3, 0.0, 777, 0.3, 0.002), (7, -2212.7, 0.0, 100, 1.0, 0.002), (31, 3000.2, 0.0, 2045, 2.0, 0.002)]
    init = [(24, 1500.0, 0.0, 777), (6, -2210.0, 0.5, 100), (30, 3000.0, 0.0, 2045)]
    x = t.synth_tracking_iq(21, N16, 40, FS16, chans)
    eng = engines(N16)
    eng.upload_iq(x)
    bank = _native.Tracker(eng, *[list(v) for v in zip(*init)])
    rec, prof = bank.process(40, start_times(40, FS16, N16), want_profiles=True)
    bank.close()
    for c in range(3):
        one = _native.Tracker(eng, *[[v] for v in init[c]])
        r1 = one.process(40, start_times(40, FS16, N16))[0]
        one.close()
        for k in ("doppler", "carrier_phase", "peak_re", "code_phase", "symbol"):
            assert np.array_equal(rec[c][k], r1[k]), (c, k)
        assert (prof[c].argmax(axis=1) == rec[c]["peak_offset"]).all()
    tr = t.TrackerOracle(25, 1500.0, 0.0, 777, FS16, N16)
    y = x[:N16] * np.exp(-1j * (2 * np.pi * 1500.0 * (np.arange(N16) / FS16)))
    ref = np.abs(o.correlate_1ms(y, np.roll(tr.prn, 777)))
    assert np.abs(prof[0][0] - ref).max() <= 1e-5 * ref.max()


def test_drop_in_pool_with_undo_equals_bank_and_bits_at_16368_ksps(native_lib):
    """GpsSatelliteTracker, one call per millisecond through the channel pool: the second tracker is asked about a copy
    of the chunk the first one advanced it through, so the pool takes the step back (undo) and recomputes.  Same
    symbols as TrackerBank; integrate_bits gives the host NavigationBitIntegrator's events."""
    from gypsum_b200.antenna_sample_provider import AntennaSampleChunk, SampleProviderAttributes
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.navigation_bit_integrator import NavigationBitIntegrator
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import BitValue, GpsSatelliteTracker, GpsSatelliteTrackingParameters, TrackerBank

    n_ms = 400
    attrs = SampleProviderAttributes(FS16, N16)
    chans = [(25, 1500.3, 0.0, 777, 0.3, 0.002), (7, -2212.7, 0.0, 100, 1.0, 0.002)]
    seeds = [(25, 1500.0, 0.0, 777), (7, -2210.0, 0.5, 100)]
    x = t.synth_tracking_iq(33, N16, n_ms, FS16, chans)
    tt = np.array([t.chunk_times(k, FS16, N16) for k in range(n_ms)])
    codes = generate_replica_prn_signals()
    sats = {sv: GpsSatellite(GpsSatelliteId(sv), codes[GpsSatelliteId(sv)], 16) for sv in (25, 7)}
    bank = TrackerBank([(sats[sv], f, p, cp) for sv, f, p, cp in seeds], attrs)
    rec = bank.process(x, tt[:, 0])
    events = bank.integrate_bits(tt[:, 0], tt[:, 1])
    trks = [GpsSatelliteTracker(GpsSatelliteTrackingParameters(satellite=sats[sv], current_doppler_shift=f,
                                                               current_carrier_wave_phase_shift=p,
                                                               current_prn_code_phase_shift=cp, doppler_shifts=[]),
                                attrs, keep_correlation_profiles=False) for sv, f, p, cp in seeds]
    code = {BitValue.ONE: 1, BitValue.ZERO: 0, BitValue.UNKNOWN: -1}
    kept, got = [], [[], []]
    integ = [NavigationBitIntegrator(GpsSatelliteId(sv)) for sv, *_ in seeds]
    host_bits = [[], []]
    for k in range(n_ms):
        first = AntennaSampleChunk(tt[k, 0], tt[k, 1], x[k * N16:(k + 1) * N16])
        second = AntennaSampleChunk(tt[k, 0], tt[k, 1], x[k * N16:(k + 1) * N16].copy())
        kept += [first, second]  # keeps the two chunk keys distinct
        for c, chunk in enumerate((first, second)):
            ps = trks[c].process_samples(chunk)
            got[c].append(ps.pseudosymbol.as_val())
            host_bits[c] += [(k, e.receiver_timestamp, e.trailing_edge_receiver_timestamp, code[e.bit_value])
                             for e in integ[c].process_pseudosymbol(chunk.start_time, ps)]
    for c in range(2):
        assert got[c] == list(rec[c]["symbol"]), c
        assert trks[c].tracking_params.current_doppler_shift == rec[c, -1]["doppler"]
        dev = [(int(e["ms_index"]), float(e["receiver_timestamp"]), float(e["trailing_edge_receiver_timestamp"]),
                int(e["bit_value"])) for e in events[c]]
        assert dev == host_bits[c] and len(dev) >= 10, c
        trks[c].close()


def _receiver_flow(tmp_path, s, n_ms=60):
    """file provider -> DeviceSampleRing (10 ms) -> detector on the full window -> one drop-in tracker per detected
    satellite, each fed the newest ring slot from the first full window on (the first tracker call is at slot 9).
    Returns the IQ, {sv: acquisition result}, {sv: pseudosymbols} and the satellites."""
    from gypsum_b200.acquisition import GpsSatelliteDetector
    from gypsum_b200.antenna_sample_provider import (AntennaSampleProviderBackedByFile, DeviceSampleRing, InputFileInfo,
                                                     NoMoreSamplesError)
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import GpsSatelliteTracker, GpsSatelliteTrackingParameters

    n, fs = 1023 * s, 1023000 * s
    planted = [(25, 1500.3, 0.0, 777, 0.3, 0.004), (7, -2212.7, 0.0, 1900, 1.0, 0.004)]
    x = t.synth_tracking_iq(44, n, n_ms + 1, fs, planted)
    path = tmp_path / "recording"
    x.view(np.float32).tofile(path)
    provider = AntennaSampleProviderBackedByFile(InputFileInfo(path, fs))
    attrs = provider.get_attributes()
    codes = generate_replica_prn_signals()
    satellites = {sid: GpsSatellite(sid, code, attrs.samples_per_prn_transmission // 1023) for sid, code in codes.items()}
    detector = GpsSatelliteDetector(satellites)
    ring = DeviceSampleRing(attrs, 10)
    search_for = [GpsSatelliteId(i) for i in (3, 7, 25)]
    trackers, symbols, acq = {}, {}, {}
    k = 0
    while True:
        try:
            chunk = ring.append(provider.get_samples(attrs.samples_per_prn_transmission))
        except NoMoreSamplesError:
            break
        if ring.is_full() and not trackers:
            for r in detector.detect_satellites_in_antenna_data(search_for, ring.window(), attrs):
                params = GpsSatelliteTrackingParameters(
                    satellite=satellites[r.satellite_id], current_doppler_shift=r.doppler_shift,
                    current_carrier_wave_phase_shift=r.carrier_wave_phase_shift,
                    current_prn_code_phase_shift=r.prn_phase_shift, doppler_shifts=[])
                trackers[r.satellite_id.id] = GpsSatelliteTracker(params, attrs, keep_correlation_profiles=False)
                symbols[r.satellite_id.id], acq[r.satellite_id.id] = [], r
        for sv, trk in trackers.items():
            symbols[sv].append(trk.process_samples(chunk).pseudosymbol.as_val())
        k += 1
    assert k == n_ms and sorted(trackers) == [7, 25]  # detector first (acquisition), then the trackers
    for trk in trackers.values():
        trk.close()
    ring.native.close()
    return x, acq, symbols, satellites


def test_receiver_flow_at_16368_ksps(tmp_path, native_lib):
    """file provider -> DeviceSampleRing -> detector -> trackers -> pseudosymbols, step for step against the oracle
    flow (acquisition and tracking).  Planted code phases stay below 2046, the only ones the reference can keep."""
    n_ms = 60
    x, acq, symbols, _ = _receiver_flow(tmp_path, 16, n_ms)
    first = x[: 10 * N16]
    for sv in acq:
        ref = o.acquire_sv(sv, first, FS16, N16)
        assert (ref.doppler, ref.code_phase) == (acq[sv].doppler_shift, acq[sv].prn_phase_shift), sv
        tr = t.TrackerOracle(sv, ref.doppler, ref.carrier_phase, ref.code_phase, FS16, N16)
        want = [tr.step(x[ms * N16:(ms + 1) * N16], *t.chunk_times(ms, FS16, N16))["symbol"] for ms in range(9, n_ms)]
        assert symbols[sv] == want, sv


@pytest.mark.parametrize("s", [1, 3, 5])
def test_receiver_flow_reads_odd_ring_slots_at_odd_n(tmp_path, native_lib, s):
    """The flow above where N = 1023 S is odd: every other slot of the 10-ms ring starts 8 bytes past a 16-byte boundary,
    and the trackers read slots 9, 0, 1, ... in turn.  Each tracker's pseudosymbols and final Doppler == a TrackerBank
    seeded with the same acquisition and fed the same milliseconds by upload, bit for bit; and == the float64 oracle
    tracker from that acquisition, bar symbols where the oracle's in-phase prompt is float32 noise around zero.  The
    acquisition equals the oracle's in code phase; a different Doppler bin must be proved a near-tie (its non-coherent
    peak within 1e-5 of the oracle bin's on the oracle's own float64 profiles), as the acquisition tests do."""
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId
    from gypsum_b200.tracker import TrackerBank

    n_ms = 60
    n, fs = 1023 * s, 1023000 * s
    x, acq, symbols, satellites = _receiver_flow(tmp_path, s, n_ms)
    first = x[: 10 * n]
    tt = np.array([t.chunk_times(ms, fs, n) for ms in range(9, n_ms)])
    for sv, r in acq.items():
        ref = o.acquire_sv(sv, first, fs, n)
        assert r.prn_phase_shift == ref.code_phase, sv
        if r.doppler_shift != ref.doppler:
            prn = o.replica(sv, n)
            here = o.integrate(o.NON_COHERENT, first, fs, n, r.doppler_shift, prn).max()
            there = o.integrate(o.NON_COHERENT, first, fs, n, ref.doppler, prn).max()
            assert here >= there * (1 - 1e-5), (sv, r.doppler_shift, ref.doppler)
        seed = (r.doppler_shift, r.carrier_wave_phase_shift, r.prn_phase_shift)
        bank = TrackerBank([(satellites[GpsSatelliteId(sv)], *seed)], Attrs(fs, n))
        rec = bank.process(x[9 * n:n_ms * n], tt[:, 0])[0]
        assert symbols[sv] == list(rec["symbol"]), sv
        tr = t.TrackerOracle(sv, *seed, fs, n)
        got = [tr.step(x[ms * n:(ms + 1) * n], *tt[ms - 9]) for ms in range(9, n_ms)]
        scale = max(abs(g["peak"].real) for g in got)
        for k, g in enumerate(got):
            assert symbols[sv][k] == g["symbol"] or abs(g["peak"].real) <= 1e-4 * scale, (sv, k)
