"""Acquisition at every sample rate the engine accepts (S = 1, 2, 3, 4, 5, 6, 8, 10, 12, 16): every entry point against
the float64 oracle, and at 5.115 / 6.138 / 8.184 / 10.230 / 12.276 Msps against the live reference's outputs
(tests/golden/acquisition_rates.npz, tools/make_golden_rates.py).

These rates reach kernel builds and plans no other test does: k_doppler_spectra<5, 6, 8, 10, 12> (more than 16 samples per
thread, polyphase rows and transpose tiles in separate shared memory), correlate slot splits of 6, 8 and 12 slots per cell,
the multi-millisecond one-warp kernel above S = 4, and odd N (5115), where every other millisecond starts 8 but not 16 bytes
into an aligned buffer.

Tolerances (DESIGN.md section 6, checked by tests/acq_support.py): magnitudes and sums |gpu - ref| <= 1e-5 * max(ref); count
exact; argmax, Doppler bin and code phase exact unless the oracle's own float64 profile ties within the tolerance, proved per
mismatch; strength 1e-4 relative; carrier phase 1e-4 rad.  Oracle grids are spread over the host's cores (fork pool)."""
import os

import numpy as np
import pytest

from acq_support import (DOP41, MAG_TOL, assert_records_equal, check_detector_golden, check_grid, check_search,
                         mid_branch_lag, oracle_searches, rate)
from gpu_support import ROOT, Attrs, EngineCache, make_engine, run_child
from oracle import gypsum_oracle as o

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(ROOT, "tests", "golden", "acquisition_rates.npz")
RATES = [1, 2, 3, 4, 5, 6, 8, 10, 12, 16]
NEW_RATES = [5, 6, 8, 10, 12]

_FIRST_RUN_SCRIPT = r"""
import sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
from gpu_support import make_engine
from gypsum_b200 import _native
from oracle import gypsum_oracle as o

for s in (5, 6, 8, 10, 12):
    n, fs = 1023 * s, 1023000 * s
    x = o.synth_iq(s, n, 3, fs, [(25, 1500.0, n - 1, 0.3, 0.3)])
    eng = make_engine(fs, n)
    eng.upload_iq(x)
    dop = np.arange(-2000.0, 2001.0, 500.0)
    for m in (1, 3):
        g = eng.acquire_grid(1, m, [24, 3], dop)[0]
        assert int(g["argmax"][0, 7]) == n - 1 and int(np.argmax(g["peak"][0])) == 7, (s, m)
    c = eng.acquire_cells([24, 3], [1500.0, 0.0], 2, _native.COHERENT, probe_idx=[n - 1, 0])
    assert int(c["argmax"][0]) == n - 1, s
    p = eng.correlation_profile(24, 1500.0, 2, _native.NON_COHERENT)
    assert int(p.argmax()) == n - 1, s
    r = eng.detect([24], 3)[0]
    assert int(r["code_phase"]) == n - 1 and abs(float(r["doppler"]) - 1500.0) <= 100, s
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


# ---- 1. full grid, M = 1 --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", RATES)
def test_full_grid_one_ms_every_cell(engines, s):
    """32 PRN x 41 Doppler x 1 ms, every cell.  Planted code phases at 0, mid-code on branch s // 2 and at n - 1
    (branch s - 1); each planted satellite is found at its planted bin and phase."""
    n, fs = rate(s)
    planted = [(3, -3000.0, 0, 1.0, 0.3), (11, 4500.0, mid_branch_lag(s), 2.0, 0.3), (32, -9500.0, n - 1, 2.5, 0.3)]
    x = o.synth_iq(200 + s, n, 1, fs, planted)
    eng = engines(1023 * s)
    eng.upload_iq(x)
    rec = eng.acquire_grid(1, 1, np.arange(32), DOP41)[0]
    check_grid(rec, x, fs, n, list(range(1, 33)), DOP41, f"S={s}")
    for sv, f, tau, _, _ in planted:
        b = int(np.argmax(rec["peak"][sv - 1]))
        assert (DOP41[b], int(rec["argmax"][sv - 1, b])) == (f, tau), (s, sv)


# ---- 2. multi-millisecond grid, M = 3, two blocks -------------------------------------------------------------------
@pytest.mark.parametrize("s", RATES)
def test_three_ms_grid_two_blocks(engines, s):
    """8 PRNs x 9 Doppler, M = 3, two blocks in one call: the block stride M * N is odd at S = 5."""
    n, fs = rate(s)
    svs = [3, 7, 11, 14, 20, 25, 29, 32]
    dop = np.arange(-4000.0, 4001.0, 1000.0)
    planted = [(7, 2000.0, n - 1, 0.4, 0.15), (25, -3000.0, mid_branch_lag(s), 1.3, 0.15)]
    x = np.concatenate([o.synth_iq(300 + 10 * s + b, n, 3, fs, planted) for b in range(2)])
    eng = engines(1023 * s)
    eng.upload_iq(x)
    rec = eng.acquire_grid(2, 3, [sv - 1 for sv in svs], dop)
    for b in range(2):
        check_grid(rec[b], x[b * 3 * n:(b + 1) * 3 * n], fs, n, svs, dop, f"S={s} block {b}")
        for sv, f, tau, _, _ in planted:
            a, k = svs.index(sv), int(np.flatnonzero(dop == f)[0])
            assert int(np.argmax(rec[b]["peak"][a])) == k and int(rec[b]["argmax"][a, k]) == tau, (s, b, sv)


# ---- 3. coherent ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", RATES)
def test_coherent_grid_and_probes(engines, s):
    """A coherent grid at M = 2 (warp-pair kernel), and a coherent cell list whose probes sit at 0, at n - 1, on branch
    s - 1 and at the planted peak: each probe's complex value against the oracle's coherent profile."""
    from gypsum_b200 import _native

    n, fs = rate(s)
    svs = [2, 9, 17, 25, 31]
    dop = np.arange(-2000.0, 2001.0, 1000.0)
    planted = [(25, 1000.0, n - 1, 0.7, 0.3), (9, -2000.0, 300 * s + s - 1, 2.1, 0.3)]
    x = o.synth_iq(400 + s, n, 2, fs, planted)
    eng = engines(1023 * s)
    eng.upload_iq(x)
    rec = eng.acquire_grid(1, 2, [sv - 1 for sv in svs], dop, _native.COHERENT)[0]
    check_grid(rec, x, fs, n, svs, dop, f"S={s} coherent", o.COHERENT)
    cells = [(25, 1000.0, n - 1), (25, 1000.0, 0), (9, -2000.0, 300 * s + s - 1), (9, -2000.0, 700 * s + s - 1),
             (17, 500.0, n - 1), (2, -1250.0, 0), (31, 3333.0, 5 * s - 1)]
    got = eng.acquire_cells([c[0] - 1 for c in cells], [c[1] for c in cells], 2, _native.COHERENT,
                            probe_idx=[c[2] for c in cells])
    for i, (sv, f, p) in enumerate(cells):
        ref = o.integrate(o.COHERENT, x, fs, n, f, o.replica(sv, n))
        mag = np.abs(ref)
        assert abs(complex(got["probe_re"][i], got["probe_im"][i]) - ref[p]) <= MAG_TOL * mag.max(), (s, i)
        assert abs(got["peak"][i] - mag.max()) <= MAG_TOL * mag.max(), (s, i)
        assert abs(got["sum"][i] - mag.sum()) <= MAG_TOL * mag.sum(), (s, i)
        assert got["count"][i] == np.count_nonzero(mag == mag.max()), (s, i)
        if got["argmax"][i] != mag.argmax():
            assert mag.max() - mag[got["argmax"][i]] <= MAG_TOL * mag.max(), (s, i)
    assert int(got["argmax"][0]) == n - 1 and int(got["argmax"][2]) == 300 * s + s - 1


# ---- 4. full profiles -----------------------------------------------------------------------------------------------
# S -> (sv, Doppler) of the profiled cell; at the new rates the golden file's cells
PROFILE_CELLS = {1: (19, 700.0), 2: (25, 1500.0), 3: (11, -3500.0), 4: (32, 4875.0), 16: (6, -8250.0)}


@pytest.mark.parametrize("s", RATES)
def test_full_profiles(engines, s):
    """correlation_profile, non-coherent and coherent, M = 2, against the oracle and, at the five new rates, against the
    profiles recorded from the live reference.  The planted code phase is n - 1."""
    from gypsum_b200 import _native

    n, fs = rate(s)
    z = np.load(GOLDEN)
    key = f"cell_n{n}"
    if s in NEW_RATES:
        sv, f = int(z[f"{key}__sv"]), float(z[f"{key}__doppler"])
        planted = [(int(p[0]), p[1], int(p[2]), p[3], p[4]) for p in z[f"{key}__planted"]]
    else:
        sv, f = PROFILE_CELLS[s]
        planted = [(sv, f + 0.25, n - 1, 0.6, 0.3)]
    x = o.synth_iq(int(z["profile_seed"]), n, 2, fs, planted)
    eng = engines(1023 * s)
    eng.upload_iq(x)
    nc = eng.correlation_profile(sv - 1, f, 2, _native.NON_COHERENT)
    co = eng.correlation_profile(sv - 1, f, 2, _native.COHERENT)
    ref_nc = o.integrate(o.NON_COHERENT, x, fs, n, f, o.replica(sv, n))
    ref_co = o.integrate(o.COHERENT, x, fs, n, f, o.replica(sv, n))
    assert np.abs(nc - ref_nc).max() <= MAG_TOL * ref_nc.max()
    assert np.abs(co - ref_co).max() <= MAG_TOL * np.abs(ref_co).max()
    assert int(nc.argmax()) == int(ref_nc.argmax()) == n - 1
    if s in NEW_RATES:
        assert np.abs(nc - z[f"{key}__noncoherent"]).max() <= MAG_TOL * ref_nc.max()
        assert np.abs(co - z[f"{key}__coherent"]).max() <= MAG_TOL * np.abs(ref_co).max()
        golden_strength = float(z[f"{key}__strength"])
        assert abs(o.peak_strength(nc.astype(np.float64)) - golden_strength) <= 1e-4 * golden_strength


# ---- 5. large-batch path (rsplit = 1) -------------------------------------------------------------------------------
@pytest.mark.parametrize("s", [s for s in RATES if np.gcd(s, 12) > 1])
def test_large_batch_whole_cell_per_warp_path(engines, s):
    """Enough cells (more than 8 * SMs * 12) that every warp of the one-warp kernel keeps a whole cell: records
    identical to the split launches of single blocks (gcd(S, 12) warps per cell), and to the oracle on sampled cells.
    At S = 2 also on a large launch: records DMA'd straight into a pinned caller buffer, a wrong-shaped buffer refused,
    and a sub-block exact against the oracle."""
    import torch

    from gypsum_b200 import _native

    n, fs = rate(s)
    cells_per_block = 32 * DOP41.size
    nb = -(-8 * torch.cuda.get_device_properties(0).multi_processor_count * 12 // cells_per_block)
    assert nb * cells_per_block >= 8 * torch.cuda.get_device_properties(0).multi_processor_count * 12
    planted = [(25, 1500.0, n - 1, 0.3, 0.3), (4, -7000.0, mid_branch_lag(s), 0.0, 0.25)]
    x = o.synth_iq(500 + s, n, nb, fs, planted)
    eng = engines(1023 * s)
    eng.upload_iq(x)
    big = eng.acquire_grid(nb, 1, np.arange(32), DOP41)
    for b in (0, nb - 1):
        eng.upload_iq(x[b * n:(b + 1) * n])
        one = eng.acquire_grid(1, 1, np.arange(32), DOP41)[0]
        assert_records_equal(big[b], one, (s, b), sum_rtol=1e-9)
    b = nb // 2
    check_grid(big[b][[24, 3]][:, 15:26], x[b * n:(b + 1) * n], fs, n, [25, 4], DOP41[15:26], f"S={s} block {b}")
    assert int(big[b]["argmax"][24, 23]) == n - 1 and int(big[b]["argmax"][3, 6]) == mid_branch_lag(s)
    if s != 2:
        return
    # eight blocks of seed 8, repeated up to nb blocks; their sub-block below has no near-tie, so argmax and count are exact
    y = o.synth_iq(8, n, 8, fs, [(25, 1500.0, 777, 0.3, 0.3), (4, -7000.0, 2000, 0.0, 0.25)])
    eng.upload_iq(np.tile(y, -(-nb // 8))[:nb * n])
    want = eng.acquire_grid(nb, 1, np.arange(32), DOP41)
    pinned = torch.empty(nb * 32 * DOP41.size * 32, dtype=torch.uint8).pin_memory()
    view = pinned.numpy().view(_native.RECORD_DTYPE).reshape(nb, 32, DOP41.size)
    assert eng.acquire_grid(nb, 1, np.arange(32), DOP41, out=view) is view
    assert_records_equal(view, want, "pinned out")
    with pytest.raises(ValueError):
        eng.acquire_grid(nb, 1, np.arange(32), DOP41, out=view[:4])
    peak, arg, total, count = o.grid_cells(y[3 * n:4 * n], fs, n, [25, 4], list(DOP41[20:26]))
    sub = want[3][[24, 3]][:, 20:26]
    assert np.abs(sub["peak"] - peak).max() <= MAG_TOL * peak.max()
    assert np.array_equal(sub["argmax"], arg) and np.array_equal(sub["count"], count)
    assert np.abs(sub["sum"] - total).max() <= MAG_TOL * total.max()


# ---- 6. scratch batching --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", [2, 12])
def test_grid_split_into_scratch_sized_batches(engines, monkeypatch, s):
    """A grid whose spectra exceed the scratch budget runs as several (doppler_spectra, correlate) batches of blocks;
    records land exactly where a single batch puts them.  S = 2, M = 1: 33 bins x 32 KB ~ 1 MB per block and a 3 MB
    budget; S = 12, M = 2: 17 bins x 2 ms x 384 KB = 6.4 MB per block and 14 MB; batches of 2 blocks either way."""
    n, fs = rate(s)
    if s == 2:
        m, nb, budget_mb, lag, blocks = 1, 7, "3", 777, (0, 3, 6)
        x = o.synth_iq(12, n, nb, fs, [(25, 1500.0, lag, 0.3, 0.3), (2, 6500.0, 11, 0.0, 0.3)])
        dop = np.arange(-8000.0, 8001.0, 500.0)
    else:
        m, nb, budget_mb, lag, blocks = 2, 5, "14", n - 1, range(5)
        x = o.synth_iq(13, n, 2 * nb, fs, [(25, 1500.0, lag, 0.3, 0.3), (2, 6000.0, 11, 0.0, 0.3)])
        dop = np.arange(-8000.0, 8001.0, 1000.0)
    monkeypatch.setenv("GB200_SPEC_BUDGET_MB", budget_mb)
    small = make_engine(fs, n)
    monkeypatch.delenv("GB200_SPEC_BUDGET_MB")
    try:
        big = engines(n)
        for e in (small, big):
            e.upload_iq(x)
        a = small.acquire_grid(nb, m, np.arange(32), dop)
        b = big.acquire_grid(nb, m, np.arange(32), dop)
    finally:
        small.close()
    assert_records_equal(a, b, f"S={s}", sum_rtol=1e-9)
    for blk in blocks:
        assert a["argmax"][blk, 24, int(np.argmax(a["peak"][blk, 24]))] == lag
        assert a["argmax"][blk, 1, int(np.argmax(a["peak"][blk, 1]))] == 11


# ---- 7. on-device search --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", RATES)
def test_on_device_search_against_oracle(engines, s):
    """gb200_detect at M = 3 == acquire_sv (acquisition.py:70-152): two planted satellites, one at code phase n - 1, and
    one absent."""
    n, fs = rate(s)
    svs = [14, 27, 20]
    planted = [(14, 2345.0, n - 1, 0.9, 0.2), (27, -4150.0, mid_branch_lag(s), 2.2, 0.2)]
    x = o.synth_iq(600 + s, n, 3, fs, planted)
    eng = engines(1023 * s)
    eng.upload_iq(x)
    got = eng.detect([sv - 1 for sv in svs], 3)
    refs = oracle_searches(svs, x, fs, n)
    for i, (sv, (r, amb)) in enumerate(zip(svs, refs)):
        phase = float(np.angle(complex(got["probe_re"][i], got["probe_im"][i])))
        check_search((int(got["doppler"][i]), int(got["code_phase"][i]), float(got["strength"][i]), phase), sv,
                     (r.doppler, r.code_phase, r.strength, r.carrier_phase), amb, x, fs, n, (s, sv))
    assert refs[0][0].code_phase == n - 1 and min(refs[0][0].strength, refs[1][0].strength) > o.DETECTION_THRESHOLD
    # the best of ~220 noise-only cells can reach just above the threshold (3.1 - 3.4 at some rates): the absent satellite
    # is checked by the rules above whichever side of it it lands on
    assert refs[2][0].strength < min(refs[0][0].strength, refs[1][0].strength)


@pytest.mark.parametrize("s", [5, 12])
def test_detector_against_reference_golden_at_other_rates(native_lib, s):
    """GpsSatelliteDetector at M = 4 == the live reference's detector; the on-device search (_acquire_many) and the
    pass-by-pass search from the host (_acquire_many_stepwise) agree."""
    from gypsum_b200.acquisition import GpsSatelliteDetector
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite

    n, fs = rate(s)
    z = np.load(GOLDEN)
    key = f"detect_n{n}"
    planted = [(int(p[0]), p[1], int(p[2]), p[3], p[4]) for p in z[f"{key}__planted"]]
    x = o.synth_iq(int(z[f"{key}__seed"]), n, int(z[f"{key}__n_ms"]), fs, planted)
    codes = generate_replica_prn_signals()
    det = GpsSatelliteDetector({sid: GpsSatellite(sid, code, s) for sid, code in codes.items()})
    ids = [GpsSatelliteId(int(sv)) for sv in z[f"{key}__svs"]]
    check_detector_golden(det, ids, x, Attrs(fs, n), z[f"{key}__detected"], z[f"{key}__results"], fs, n, f"S={s}")


# ---- 8. generic replica ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", [5, 16])
def test_generic_replica_profiles(engines, s):
    """correlation_profile_replica with a random complex replica, M = 2, both kinds, against o.integrate."""
    from gypsum_b200 import _native

    n, fs = rate(s)
    x = o.synth_iq(700 + s, n, 2, fs, [(9, -1250.0, n - 1, 0.7, 0.3)])
    rep = (np.random.default_rng(s).standard_normal(n) + 1j * np.random.default_rng(100 + s).standard_normal(n))
    rep = rep.astype(np.complex64)
    eng = engines(1023 * s)
    eng.upload_iq(x)
    nc = eng.correlation_profile_replica(rep, 1500.0, 2, _native.NON_COHERENT)
    co = eng.correlation_profile_replica(rep, 1500.0, 2, _native.COHERENT)
    ref_nc = o.integrate(o.NON_COHERENT, x, fs, n, 1500.0, rep.astype(complex))
    ref_co = o.integrate(o.COHERENT, x, fs, n, 1500.0, rep.astype(complex))
    assert np.abs(nc - ref_nc).max() <= MAG_TOL * ref_nc.max()
    assert np.abs(co - ref_co).max() <= MAG_TOL * np.abs(ref_co).max()


# ---- 9. odd N: milliseconds that start 8 but not 16 bytes into a buffer ------------------------------------------------
def test_odd_n_ring_windows_and_graph_replayed_host_grid(engines):
    """At 5.115 Msps N is odd.  Grids and searches over a device-ring window bound at an odd slot and at an even slot,
    and acquire_grid_host (eager, captured, replayed), are bit-identical to upload_iq + acquire_grid / detect on the same
    samples."""
    from gypsum_b200 import _native

    n, fs = rate(5)
    svs = np.array([13, 24, 2], dtype=np.int32)
    dop = np.arange(-3000.0, 3001.0, 1000.0)
    x = o.synth_iq(800, n, 5, fs, [(14, 2000.0, n - 1, 0.9, 0.2), (25, -1000.0, 2557, 0.3, 0.2)])
    eng = engines(n)

    def run():
        return (eng.acquire_grid(3, 1, svs, dop), eng.acquire_grid(1, 3, svs, dop), eng.detect(svs, 3))

    def same(got, want, what):
        assert_records_equal(got[0], want[0], (what, "M=1"))
        assert_records_equal(got[1], want[1], (what, "M=3"))
        for k in ("doppler", "strength", "probe_re", "probe_im", "code_phase"):
            assert np.array_equal(got[2][k], want[2][k]), (what, k)

    ring = _native.Ring(eng, 4)
    try:
        ring.append(x[:4 * n])  # slots 0 .. 3
        ring.bind_newest(3)  # window at slot 1: starts N * 8 bytes (odd multiple of 8) into the ring
        odd = run()
        ring.append(x[4 * n:5 * n])
        ring.bind_newest(3)  # window at slot 2
        even = run()
    finally:
        ring.close()
    eng.upload_iq(x[n:4 * n])
    same(odd, run(), "odd slot")
    eng.upload_iq(x[2 * n:5 * n])
    want = run()
    same(even, want, "even slot")
    assert int(want[2]["code_phase"][0]) == n - 1 and int(want[1][0, 0, 5]["argmax"]) == n - 1
    eng.upload_iq(x[2 * n:5 * n])
    ref = eng.acquire_grid(3, 1, svs, dop)
    for call in ("eager", "captured", "replayed"):
        assert_records_equal(eng.acquire_grid_host(x[2 * n:5 * n], 3, 1, svs, dop), ref, call)


# ---- 10. all-zero input ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", RATES)
def test_all_zero_input(engines, s):
    """Every profile value ties at 0: peak 0, argmax 0, count N, sum 0 through the M = 1 grid, the M = 2 grid and a
    coherent list.  The fused kernel exists only at S = 2 and 4."""
    from gypsum_b200 import _native

    n, _ = rate(s)
    eng = engines(1023 * s)
    eng.upload_iq(np.zeros(2 * n, np.complex64))
    dop = np.array([-5000.0, 0.0, 2500.0])
    for rec in (eng.acquire_grid(1, 1, [0, 17, 31], dop), eng.acquire_grid(1, 2, [0, 17, 31], dop),
                eng.acquire_cells([0, 17, 31], [-5000.0, 0.0, 2500.0], 2, _native.COHERENT, probe_idx=[0, n - 1, 5])):
        assert (rec["peak"] == 0).all() and (rec["argmax"] == 0).all() and (rec["sum"] == 0).all()
        assert (rec["count"] == n).all()
    if s in (2, 4):
        eng.set_fused(True)
        eng.set_fused(None)
    else:
        with pytest.raises(ValueError):
            eng.set_fused(True)
