"""gb200_detect's plan restated on the CPU (tests/acq_support.py `detect_plan`) and the helpers that read the search
oracle's trace: the bins of a pass fit the kernel's 32 slots at every centre the search can reach, every case of
tests/test_gpu_detect_edges.py reaches the edge it is named for on the plans of H100 SXM (132 SMs) and PCIe (114 SMs)
cards, and the trace helpers report the kept pass and the centres the search walks through."""
import math
import warnings

import numpy as np
import pytest

import test_gpu_detect_edges as edges
from acq_support import (REFINE_MAX_BINS, SPREADS, budget_for, centre_crosses_zero, centre_outside, detect_plan, kept_pass,
                         rate, refine_slots, trace_passes, truncation_differs)
from gypsum_b200.acquisition import doppler_search_bins
from oracle import gypsum_oracle as o

SM_COUNTS = [132, 114]


def test_spreads_are_the_ten_passes():
    spreads, s = [], 7000.0
    while s >= 10:  # acquisition.py:78-89
        spreads.append(s)
        s /= 2
    assert SPREADS == spreads and len(SPREADS) == 10


@pytest.mark.parametrize("spread", SPREADS)
def test_bin_counts_fit_the_slots_at_every_centre(spread):
    """20..28 bins (kernels.cuh) at every integer centre in +-60 kHz, so never more than kRefineMaxBins (32)."""
    counts = {len(doppler_search_bins(c, spread)) for c in range(-60000, 60001)}
    assert min(counts) >= 20 and max(counts) <= 28 <= REFINE_MAX_BINS, sorted(counts)


@pytest.mark.parametrize("spread", SPREADS)
def test_refine_slots_are_the_reference_bins(spread):
    """k_refine_plan's slots (truncation toward zero, NaN past the last bin) == range(int(c - s), int(c + s), int(s / 10))
    at centres on both sides of zero, where int() and floor differ, and far out."""
    for c in list(range(-40, 41)) + [-60000, -9451, -7000, -1, 7000, 8399, 60000]:
        want = list(doppler_search_bins(c, spread))
        got = refine_slots(float(c), spread)
        assert got[:len(want)] == want and all(math.isnan(v) for v in got[len(want):]), (c, spread)


# ---- the plan --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sms", SM_COUNTS)
def test_receivers_call_chunks(sms):
    """32 satellites over 10 ms with the default 512 MiB budget: 6 / 4 / 4 / 3 chunks at S = 16 / 12 / 10 / 8 (a last
    chunk of 2 at 16 and 10), 2 at S = 6 and 5, one at S <= 3 (S = 2 and 4 run fused)."""
    for s, chunks in edges.RECEIVER_CHUNKS.items():
        assert [k for _, k in detect_plan(s, 10, 32, sms)["chunks"]] == chunks
    assert [len(detect_plan(s, 10, 32, sms)["chunks"]) for s in (6, 5, 3, 1)] == [2, 2, 1, 1]
    assert detect_plan(2, 10, 32, sms)["fused"] and detect_plan(4, 10, 32, sms)["fused"]


@pytest.mark.parametrize("sms", SM_COUNTS)
@pytest.mark.parametrize("m", [1, 2])
@pytest.mark.parametrize("s", [1, 3, 5, 12])
def test_chunk_edge_budgets(sms, s, m):
    """The budgets the GPU file uses reach each chunk edge: the chunks of sv_per_chunk, the last holding the rest."""
    n_sv = len(edges.CHUNK_SVS)
    assert len(detect_plan(s, m, n_sv, sms)["chunks"]) == 1 and not detect_plan(s, m, n_sv, sms)["fused"]
    for name, spc in edges.CHUNK_EDGES.items():
        mb = budget_for(s, m, n_sv, spc, sms)
        if mb is None:
            assert (s, m) == (1, 1) and spc % 2, name  # half a MiB per satellite: odd counts need a budget below 1 MiB
            continue
        p = detect_plan(s, m, n_sv, sms, mb)
        assert p["sv_per_chunk"] == spc
        sizes = [k for _, k in p["chunks"]]
        assert sum(sizes) == n_sv and set(sizes[:-1]) == {spc}
        if name == "divides":
            assert sizes == [spc] * (n_sv // spc)
        if name in ("last_chunk_one", "n_sv_minus_1", "two"):
            assert sizes[-1] == 1


@pytest.mark.parametrize("sms", SM_COUNTS)
@pytest.mark.parametrize("s", [1, 2, 3, 4, 5, 6, 8, 10, 12, 16])
def test_one_ms_groups(sms, s):
    """32 satellites at M = 1: 12 slots, rsplit = gcd(S, 12) (far below the rsplit = 1 threshold), a partial last group
    at S = 1, 5 (12 / 12 / 8), 8, 16 (11 groups ending in 2) and 10 (6 ending in 2); pass 1's 20 bins leave slots
    20..31 switched off, so slot 19 (+6300 Hz) and slot 20 (+7000 Hz) share a group wherever cpg does not divide 20."""
    p = detect_plan(s, 1, 32, sms)
    assert p["slots"] == 12 and p["rsplit"] == math.gcd(s, 12) and p["cpg"] * p["rsplit"] == 12
    if p["fused"]:
        return
    assert p["group_sizes"] == edges.M1_GROUPS[s] and sum(p["group_sizes"]) == REFINE_MAX_BINS
    pass1 = refine_slots(0.0, 7000.0)
    assert pass1[19] == 6300 and math.isnan(pass1[20])
    assert (19 // p["cpg"] == 20 // p["cpg"]) == (20 % p["cpg"] != 0)


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_satellite_count_edges(sms):
    """The counts of the GPU file: one refine block of 64 and more, more satellites than SMs for the coherent pass, and
    the rsplit = 1 threshold at M = 2 (8 * SMs * 8 cells), at one fused and two split rates."""
    counts = edges.count_edges(sms)
    assert [counts[k] for k in ("1", "63", "64", "65")] == [1, 63, 64, 65]
    assert [math.ceil(c / 64) for c in (63, 64, 65)] == [1, 1, 2]
    assert [detect_plan(s, 2, 1, sms)["fused"] for s in edges.COUNT_RATES] == [True, False, False]
    for s in edges.COUNT_RATES:
        assert detect_plan(s, 2, counts["sms_plus_1"], sms)["coherent_grid"] == sms
        assert detect_plan(s, 2, counts["rsplit_1"], sms)["rsplit"] == 1
        assert detect_plan(s, 2, 2 * sms - 1, sms)["rsplit"] == math.gcd(s, 8)
    assert len(detect_plan(10, 2, counts["rsplit_1"], sms)["chunks"]) > 1


# ---- the trace helpers -----------------------------------------------------------------------------------------------
def _trace(chosen, strengths):
    return [dict(bins=[], peaks=[], gaps=[], chosen=c, strength=st) for c, st in zip(chosen, strengths)]


def test_trace_helpers_on_written_traces():
    t = _trace([-700, -350, -175, -88, 0, 5, 3, 2, 2, 1], [2, 3, 5, 5, 4, 6, 6, 5, 6, 1])
    assert [c for c, _, _, _ in trace_passes(t)] == [0, -700, -350, -175, -88, 0, 5, 3, 2, 2]
    assert kept_pass(t) == 6  # strictly greater only: passes 7 and 9 tie with it
    assert not centre_outside(t) and centre_crosses_zero(_trace([700, -350] + [1] * 8, [1] * 10))
    assert not centre_crosses_zero(t)  # 0 is no side
    assert truncation_differs(t)  # pass 5: -88 - 437.5
    assert not truncation_differs(_trace([7000] * 10, [1] * 10))
    assert kept_pass(_trace([0] * 10, [math.nan] * 10)) == 1
    assert kept_pass(_trace([0] * 10, [math.nan] + [9.0] * 9)) == 1  # nothing is greater than NaN
    assert centre_outside(_trace([-7000, -7350] + [0] * 8, [1] * 10)) and not centre_outside(_trace([-7000] * 10, [1] * 10))


def test_trace_helpers_on_oracle_searches():
    """On o.acquire_sv traces at 1.023 Msps over 10 ms: a satellite at +7600 Hz is centred past +7000 Hz; one at +15 Hz crosses
    zero with a lower edge where truncation and floor differ; all-zero input keeps pass 1 at -7000 Hz, code phase 0."""
    n, fs = rate(1)
    x = o.synth_iq(7, n, 10, fs, [(3, 7600.0, 100, 0.5, 0.5), (9, 15.0, 400, 1.0, 0.3)])
    t3, t9 = [], []
    r3, r9 = o.acquire_sv(3, x, fs, n, t3), o.acquire_sv(9, x, fs, n, t9)
    assert centre_outside(t3) and r3.doppler > 7000 and not centre_outside(t9)
    assert centre_crosses_zero(t9) and truncation_differs(t9) and abs(r9.doppler) < 100
    assert r3.strength == t3[kept_pass(t3) - 1]["strength"] and r3.doppler == t3[kept_pass(t3) - 1]["chosen"]
    tz = []
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        rz = o.acquire_sv(3, np.zeros(n, complex), fs, n, tz)
    assert kept_pass(tz) == 1 and (rz.doppler, rz.code_phase, rz.carrier_phase) == (-7000, 0, 0.0)
    assert np.isnan(rz.strength) and [p["chosen"] for p in tz][:2] == [-7000, -10500]
