"""The on-device satellite search (gb200_detect: k_refine_* and the correlate or fused launches of acquisition.py:70-152)
at every chunk, group and pass edge of its plan, against the float64 search oracle (o.acquire_sv).

The search has a schedule of its own (tests/acq_support.py `detect_plan`): the spectra of a pass run in chunks of
sv_per_chunk satellites, each satellite's 32 (satellite, bin) slots in groups of cpg cells with the slots past a pass's
bins switched off by NaN Dopplers, the refine kernels one thread per slot or per satellite in blocks of 128 or 64, and the
coherent pass over min(n_sv, SMs) CTAs.  Every case below asserts on the card's own SM count that it reaches the edge it
is named for, and every result is checked against the oracle with the tolerances of DESIGN.md section 6 (check_search):
Doppler and code phase exact, strength 1e-4 relative, carrier phase 1e-4 rad; a different answer only for a satellite
without a planted signal whose float64 search sits on a branch point.  Entries of one PRN in one call are
byte-identical."""
import math
import warnings

import numpy as np
import pytest

from acq_support import (budget_for, centre_crosses_zero, centre_outside, check_search,
                         detect_plan, kept_pass, oracle_searches_traced, rate, truncation_differs)
from gpu_support import Attrs, EngineCache, make_engine
from oracle import gypsum_oracle as o

pytestmark = pytest.mark.gpu
RATES = [1, 2, 3, 4, 5, 6, 8, 10, 12, 16]
RECEIVER_CHUNKS = {16: [6, 6, 6, 6, 6, 2], 12: [8, 8, 8, 8], 10: [10, 10, 10, 2], 8: [12, 12, 8]}
CHUNK_SVS = [17, 4, 29, 4, 11, 23, 8, 17, 2]  # 9 entries, unsorted, PRNs 4 and 17 twice in different chunks
CHUNK_EDGES = {"one": 1, "two": 2, "divides": 3, "last_chunk_one": 4, "n_sv_minus_1": 8}


@pytest.fixture(scope="module")
def engines(native_lib):
    cache = EngineCache()
    yield cache
    cache.close()


@pytest.fixture(scope="module")
def sms(native_lib):
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def check_detect(got, svs, refs, x, fs, n, planted, what):
    """Every entry of a detect call against its satellite's oracle search; entries of one PRN byte-identical.  A
    satellite that was not planted holds noise only, whichever side of the detection threshold its strength lands on: it
    may take another branch where its float64 search sits on one, and must then report a true cell of the search."""
    assert got.shape == (len(svs),)
    first = {}
    for i, sv in enumerate(svs):
        r, _, ambiguous = refs[sv]
        phase = float(np.angle(complex(got["probe_re"][i], got["probe_im"][i])))
        found = (int(got["doppler"][i]), int(got["code_phase"][i]), float(got["strength"][i]), phase)
        if sv not in planted and found[:2] != (r.doppler, r.code_phase):
            assert ambiguous, (what, i, sv)
            prof = o.integrate(o.NON_COHERENT, x, fs, n, found[0], o.replica(sv, n))
            assert abs(o.peak_strength(prof) - found[2]) <= 1e-4 * found[2], (what, i, sv)
        else:
            check_search(found, sv, (r.doppler, r.code_phase, r.strength, r.carrier_phase), ambiguous, x, fs, n,
                         (what, i, sv))
        assert got[i].tobytes() == got[first.setdefault(sv, i)].tobytes(), (what, i, sv)


def detect_with_budget(monkeypatch, fs, n, x, prn_idx, m, budget_mb):
    """detect on an engine made for this call, its spectra budget budget_mb MiB (read once, at gb200_create)."""
    monkeypatch.setenv("GB200_SPEC_BUDGET_MB", str(budget_mb))
    eng = make_engine(fs, n)
    monkeypatch.delenv("GB200_SPEC_BUDGET_MB")
    try:
        eng.upload_iq(x)
        return eng.detect(prn_idx, m)
    finally:
        eng.close()


def kept_before_last(refs, svs, x, fs, n):
    """The satellites whose kept pass is not pass 10 and whose kept Doppler is not the final centre, each with the
    carrier phase a coherent integration at the final centre would give instead (acquisition.py:120-136)."""
    out = {}
    for sv in svs:
        r, trace, _ = refs[sv]
        if kept_pass(trace) < 10 and r.doppler != trace[-1]["chosen"] and r.strength > o.DETECTION_THRESHOLD:
            coh = o.integrate(o.COHERENT, x, fs, n, trace[-1]["chosen"], o.replica(sv, n))
            out[sv] = float(np.angle(coh[r.code_phase]))
    return out


def phase_gap(a, b):
    d = abs(a - b) % (2 * np.pi)
    return min(d, 2 * np.pi - d)


# ---- 1. the receiver's call: 32 satellites over its 10-ms window --------------------------------------------------------
def receiver_planted(s):
    """(sv, Doppler, code phase, carrier phase, amplitude): code phase n - 1; beyond +7000 and below -7000 Hz, strong
    enough for pass 1's bins at +6300 and -7000 Hz to catch them on a sidelobe; near zero, where the centres cross zero;
    and one more."""
    n, _ = rate(s)
    return [(5, 2345.0, n - 1, 0.9, 0.15), (12, 7800.0, 1000 * s, 0.4, 0.4), (19, -9300.0, 77 * s + 1, 1.7, 0.5),
            (23, 15.0, 600 * s + s // 2, 2.9, 0.15), (30, -3725.0, 3, 0.1, 0.15)]


@pytest.mark.parametrize("s", [16, 12, 10, 8])
def test_receivers_call_over_every_chunk(native_lib, engines, sms, s):
    """At 16.368, 12.276, 10.23 and 8.184 Msps the receiver's own call (32 satellites, 10 ms, the default budget) runs in
    6, 4, 4 and 3 spectra chunks, two of them with a short last chunk.  The 32 satellites go in an unsorted order,
    through GpsSatelliteDetector on a DeviceSampleRing window and through Engine.detect on uploaded samples: the two
    bit for bit, both equal to o.detect / o.acquire_sv."""
    from gypsum_b200.acquisition import GpsSatelliteDetector
    from gypsum_b200.antenna_sample_provider import AntennaSampleChunk, DeviceSampleRing
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite

    n, fs = rate(s)
    plan = detect_plan(s, 10, 32, sms)
    assert [k for _, k in plan["chunks"]] == RECEIVER_CHUNKS[s] and not plan["fused"]
    svs = [int(v) for v in np.random.default_rng(s).permutation(np.arange(1, 33))]
    assert svs != sorted(svs)
    x = o.synth_iq(900 + s, n, 10, fs, receiver_planted(s))
    refs = oracle_searches_traced(svs, x, fs, n)
    # the edges the planted satellites are there for, on the oracle's own trace
    assert refs[5][0].code_phase == n - 1
    assert centre_outside(refs[12][1]) and max(c["chosen"] for c in refs[12][1]) > 7000
    assert centre_outside(refs[19][1]) and min(c["chosen"] for c in refs[19][1]) < -7000
    assert centre_crosses_zero(refs[23][1]) and truncation_differs(refs[23][1])
    assert all(refs[sv][0].strength > o.DETECTION_THRESHOLD for sv, *_ in receiver_planted(s))

    eng = engines(n)
    eng.upload_iq(x)
    got = eng.detect([sv - 1 for sv in svs], 10)
    check_detect(got, svs, refs, x, fs, n, {p[0] for p in receiver_planted(s)}, f"S={s} engine")
    late = kept_before_last(refs, svs, x, fs, n)
    assert late and all(phase_gap(late[sv], refs[sv][0].carrier_phase) > 1e-3 for sv in late), (s, late)

    attrs = Attrs(fs, n)
    det = GpsSatelliteDetector({sid: GpsSatellite(sid, code, s) for sid, code in generate_replica_prn_signals().items()})
    ring = DeviceSampleRing(attrs, 10)
    try:
        for k in range(10):
            ring.append(AntennaSampleChunk(k * 1e-3, (k + 1) * 1e-3, x[k * n:(k + 1) * n]))
        ids = [GpsSatelliteId(sv) for sv in svs]
        many = det._acquire_many(ids, ring.window(), attrs)
        found = det.detect_satellites_in_antenna_data(ids, ring.window(), attrs)
    finally:
        ring.native.close()
    for i, r in enumerate(many):
        phase = np.angle(np.float64(got["probe_re"][i]) + 1j * np.float64(got["probe_im"][i]))
        assert (r.satellite_id.id, r.doppler_shift, r.prn_phase_shift) == (svs[i], int(got["doppler"][i]),
                                                                          int(got["code_phase"][i])), (s, i)
        assert r.correlation_strength == float(got["strength"][i]) and r.carrier_wave_phase_shift == phase, (s, i)
    # o.detect: the searches above the threshold, in the order asked for
    assert [r.satellite_id.id for r in found] == [sv for sv in svs if refs[sv][0].strength > o.DETECTION_THRESHOLD]


# ---- 2. chunk edges under small spectra budgets -----------------------------------------------------------------------
@pytest.mark.parametrize("m", [1, 2])
@pytest.mark.parametrize("s", [1, 3, 5, 12])
def test_chunk_edges_under_small_budgets(native_lib, engines, monkeypatch, sms, s, m):
    """Nine unsorted entries (two PRNs twice, in different chunks) under the budgets that make sv_per_chunk 1, 2, 3
    (divides 9), 4 (last chunk one satellite) and 8 (n_sv - 1), where whole MiB reach them: every result byte for byte
    the default budget's (one chunk), which equals the oracle."""
    n, fs = rate(s)
    planted = [(4, 2345.0, n - 1, 0.9, 0.3), (29, -4150.0, 511 * s + s // 2, 2.2, 0.3), (23, 820.0, 7, 0.4, 0.3),
               (8, -1300.0, 100 * s + s - 1, 1.1, 0.3), (2, 6900.0, 0, 2.6, 0.3)]
    x = o.synth_iq(1000 + 10 * s + m, n, m, fs, planted)
    prn_idx = [sv - 1 for sv in CHUNK_SVS]
    assert len(detect_plan(s, m, 9, sms)["chunks"]) == 1
    eng = engines(n)
    eng.upload_iq(x)
    want = eng.detect(prn_idx, m)
    check_detect(want, CHUNK_SVS, oracle_searches_traced(CHUNK_SVS, x, fs, n), x, fs, n, {p[0] for p in planted},
                 f"S={s} M={m} default")
    reached = []
    for name, spc in CHUNK_EDGES.items():
        mb = budget_for(s, m, 9, spc, sms)
        if mb is None:
            continue
        chunks = [k for _, k in detect_plan(s, m, 9, sms, mb)["chunks"]]
        assert len(chunks) > 1 and all(k == spc for k in chunks[:-1]) and sum(chunks) == 9
        got = detect_with_budget(monkeypatch, fs, n, x, prn_idx, m, mb)
        assert got.tobytes() == want.tobytes(), (s, m, name, mb)
        reached.append(name)
    # whole MiB reach every edge at M = 2; at S = 1, M = 1 a satellite's spectra are half a MiB, so only even counts
    assert reached == list(CHUNK_EDGES) if (s, m) != (1, 1) else reached == ["two", "last_chunk_one", "n_sv_minus_1"]


# ---- 3. M = 1: the 12-warp kernel under the planner's gates -------------------------------------------------------------
M1_GROUPS = {1: [12, 12, 8], 3: [4] * 8, 5: [12, 12, 8], 6: [2] * 16, 8: [3] * 10 + [2], 10: [6] * 5 + [2],
             12: [1] * 32, 16: [3] * 10 + [2]}


@pytest.mark.parametrize("s", RATES)
def test_one_ms_search_at_every_rate(native_lib, engines, sms, s):
    """32 satellites at M = 1: the 12-warp kernel with the groups of 12 / 12 / 8, 3 ... 3 / 2, 6 ... 6 / 2 (and the exact
    splits of 4, 2 and 1 cells) whose last group is partial and whose slots past a pass's bins are switched off.  One
    satellite at +6300 Hz, pass 1's last live slot (19), in the group that straddles the first switched-off slot; one at
    +7000 Hz, where slot 20 would lie; the others at the code phase n - 1 and below -7000 Hz."""
    n, fs = rate(s)
    plan = detect_plan(s, 1, 32, sms)
    if plan["fused"]:
        assert s in (2, 4)
    else:
        assert plan["group_sizes"] == M1_GROUPS[s] and plan["slots"] == 12 and len(plan["chunks"]) == 1
    planted = [(7, 6300.0, 300 * s + 1, 0.5, 0.4), (14, 7000.0, n - 1, 1.5, 0.4), (21, -7600.0, 5, 2.5, 0.5),
               (28, -2650.0, 700 * s + s - 1, 0.2, 0.4)]
    x = o.synth_iq(1100 + s, n, 1, fs, planted)
    svs = [int(v) for v in np.random.default_rng(100 + s).permutation(np.arange(1, 33))]
    refs = oracle_searches_traced(svs, x, fs, n)
    assert refs[7][1][0]["chosen"] == 6300 and refs[14][1][0]["chosen"] == 6300  # pass 1: slot 19, slot 20 switched off
    assert refs[14][0].code_phase == n - 1
    eng = engines(n)
    eng.upload_iq(x)
    check_detect(eng.detect([sv - 1 for sv in svs], 1), svs, refs, x, fs, n, {p[0] for p in planted}, f"S={s} M=1")


# ---- 4. satellite-count edges -------------------------------------------------------------------------------------------
COUNT_RATES = [4, 3, 10]  # fused, split, split
COUNT_PLANTED = {3, 16, 27}


def count_edges(sms):
    """n_sv past one refine block of 64 satellites, past the SM count (the coherent pass's CTAs go round), and past
    the rsplit = 1 threshold at M = 2 (8 * SMs * 8 cells)."""
    return {"1": 1, "63": 63, "64": 64, "65": 65, "sms_plus_1": sms + 1, "rsplit_1": 2 * sms + 3}


@pytest.fixture(scope="module")
def count_cases():
    """S -> (IQ, {sv: oracle search}), made once per rate."""
    cache = {}

    def get(s):
        if s not in cache:
            n, fs = rate(s)
            planted = [(3, -3100.0, n - 1, 0.3, 0.3), (16, 4480.0, 250 * s, 1.9, 0.3), (27, -600.0, 2, 2.7, 0.3)]
            x = o.synth_iq(1200 + s, n, 2, fs, planted)
            cache[s] = (x, oracle_searches_traced(list(range(1, 33)), x, fs, n))
        return cache[s]

    return get


@pytest.mark.parametrize("edge", ["1", "63", "64", "65", "sms_plus_1", "rsplit_1"])
@pytest.mark.parametrize("s", COUNT_RATES)
def test_satellite_count_edges(native_lib, engines, sms, count_cases, s, edge):
    """Repeated, unsorted PRN lists of 1, 63, 64, 65, SMs + 1 and 2 SMs + 3 entries at M = 2: the refine kernels over one
    and more blocks, the coherent pass with more satellites than CTAs, and the whole-cell-per-warp correlate launches."""
    n, fs = rate(s)
    n_sv = count_edges(sms)[edge]
    plan = detect_plan(s, 2, n_sv, sms)
    if edge == "rsplit_1":
        assert plan["rsplit"] == 1 and detect_plan(s, 2, 2 * sms - 1, sms)["rsplit"] == math.gcd(s, 8)
    else:
        assert plan["rsplit"] == math.gcd(s, 8)
    assert plan["coherent_grid"] == min(n_sv, sms)
    rng = np.random.default_rng(1300 + 7 * s + n_sv)
    svs = [int(v) for v in rng.integers(1, 33, size=n_sv)]
    if n_sv > 32:
        assert len(set(svs)) < n_sv and svs != sorted(svs)
    x, refs = count_cases(s)
    eng = engines(n)
    eng.upload_iq(x)
    check_detect(eng.detect([sv - 1 for sv in svs], 2), svs, refs, x, fs, n, COUNT_PLANTED, f"S={s} n_sv={n_sv}")


# ---- 5. all-zero IQ ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", RATES)
def test_all_zero_input_keeps_pass_one(native_lib, engines, sms, s):
    """Every bin of every pass ties at peak 0 and every strength is NaN (0 / 0): the first bin wins each pass, no pass
    replaces pass 1, so the search keeps -7000 Hz at code phase 0 with strength NaN and a probe of exactly 0, as the
    oracle does.  70 repeated entries: the refine kernels over two blocks."""
    n, fs = rate(s)
    x = np.zeros(n, np.complex64)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        trace = []
        r = o.acquire_sv(9, x.astype(complex), fs, n, trace)
    assert (r.doppler, r.code_phase, r.carrier_phase) == (-7000, 0, 0.0) and math.isnan(r.strength)
    assert kept_pass(trace) == 1 and trace[-1]["chosen"] != -7000
    svs = [int(v) for v in np.random.default_rng(1400 + s).integers(1, 33, size=70)]
    eng = engines(n)
    eng.upload_iq(x)
    got = eng.detect([sv - 1 for sv in svs], 1)
    assert (got["doppler"] == -7000).all() and (got["code_phase"] == 0).all() and np.isnan(got["strength"]).all()
    assert (got["probe_re"] == 0).all() and (got["probe_im"] == 0).all()


# ---- 6. a kept pass before the last -----------------------------------------------------------------------------------
@pytest.mark.parametrize("s", [2, 3])
def test_kept_pass_before_the_last(native_lib, engines, s):
    """Satellites whose strongest pass is not the last and whose kept Doppler is not the final centre: the coherent
    pass must integrate at the kept Doppler (kept_doppler), which gives another carrier phase than the final centre
    would, by more than 10 times the tolerance.  S = 2 runs the fused kernel, S = 3 the split one."""
    n, fs = rate(s)
    planted = [(6, 1234.0, n - 1, 0.6, 0.2), (13, -2870.0, 400 * s, 1.6, 0.2), (24, 4321.0, 9, 2.6, 0.2),
               (31, -555.0, 800 * s + 1, 0.3, 0.2)]
    svs = [24, 6, 31, 13]
    x = o.synth_iq(1500 + s, n, 4, fs, planted)
    refs = oracle_searches_traced(svs, x, fs, n)
    late = kept_before_last(refs, svs, x, fs, n)
    assert late and all(phase_gap(late[sv], refs[sv][0].carrier_phase) > 1e-3 for sv in late), (s, late)
    eng = engines(n)
    eng.upload_iq(x)
    check_detect(eng.detect([sv - 1 for sv in svs], 4), svs, refs, x, fs, n, set(svs), f"S={s} M=4")
