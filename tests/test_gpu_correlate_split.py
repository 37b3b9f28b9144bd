"""The correlate kernels' work split at every edge of its partition, and the best-bin reduction, against the float64 oracle.

Every record of a grid or cell list comes out of one schedule: cells are cut into groups of slots / rsplit
(`correlate_slots`, `pick_rsplit`), a PRN entry's cells into chunks of a group each, and the P * chunks groups go to
min(groups, SMs) CTAs, each walking a contiguous range and re-staging the replica when the PRN changes (`k_correlate_w2048`,
`k_correlate_cells`, `decode_group`).  Large non-coherent batches are walked in L2 windows whose extra groups go round the
CTAs, grids larger than the scratch budget run in batches of blocks (`run_grid`), and cell lists in chunks of the PRN-sorted
list (`run_cells`).  The shapes below are chosen from the card's SM count so that each case lands on the edge it is named
for, and each case asserts that it does.

Every record goes through check_grid (tolerances of DESIGN.md section 6) against vector_grid; grids are written into CUDA
buffers filled with 0xFF and one grid row longer than the output, so a skipped cell (its `reserved` word is not 0) and a write
past the end (the guard row is not 0xFF) fail whatever an earlier call left behind.  Cells with the same (PRN, Doppler) in one
launch must be byte-identical, and the best-bin rows (`k_best_bins`, acquisition.py:179-189) must be the oracle's."""
import math
import warnings

import numpy as np
import pytest

from acq_support import MAG_TOL, check_grid, mid_branch_lag, rate, vector_grid
from gpu_support import EngineCache, make_engine, run_child
from oracle import gypsum_oracle as o

SPLIT_RATES = [1, 2, 3, 5, 12, 16]  # rsplit 1, 2, 3, 1, 12, 4 on the one-warp kernel at M = 1
KINDS = [(o.NON_COHERENT, 1), (o.NON_COHERENT, 3), (o.COHERENT, 2)]
EDGES = ["one_group", "sms_minus_1", "sms", "sms_plus_1", "two_sms_plus_1"]
PRN_CYCLE = [4, 0, 4, 31, 0, 17, 9, 30, 17, 2, 4, 25]  # unsorted, repeats not adjacent: replicas are re-staged after others
SPEC_BUDGET = 512 << 20  # the engine's default scratch budget (GB200_SPEC_BUDGET_MB)


# ---- the host's split rules, restated only to choose shapes -----------------------------------------------------------
def split_plan(s, m, kind, n_cells, sms):
    """(slots, rsplit, cells per group) of a correlate launch of n_cells cells.  Coherent launches run on the warp-pair
    kernel (8 pairs), non-coherent ones on the one-warp kernel (12 warps at M = 1, 8 when the accumulators live across
    milliseconds); a cell takes rsplit = gcd(S, slots) slots below 8 * SMs * slots cells, else one."""
    slots = 8 if kind == o.COHERENT or m > 1 else 12
    rsplit = math.gcd(s, slots) if n_cells < 8 * sms * slots else 1
    return slots, rsplit, slots // rsplit


def grid_plan(s, m, kind, nb, P, D, sms):
    """The plan of a grid of nb blocks run in one scratch batch: each PRN entry's nb * D cells in chunks of a group."""
    _, rsplit, cpg = split_plan(s, m, kind, nb * P * D, sms)
    chunks = -(-nb * D // cpg)
    return dict(rsplit=rsplit, cpg=cpg, chunks=chunks, n_groups=P * chunks, grid=min(P * chunks, sms))


def unit_bytes(s, m):
    """Spectra of one (block, Doppler) unit."""
    return m * s * 2 * 1024 * 8


def window_plan(s, m, P, D, nb, sms, win_mb, min_groups):
    """(plan, chunks per L2 window or None) of a non-coherent grid batch, as run_grid chooses its windows."""
    p = grid_plan(s, m, o.NON_COHERENT, nb, P, D, sms)
    batch, win = nb * D * unit_bytes(s, m), win_mb << 20
    if batch <= win + win // 2:
        return p, None
    wc = -(-p["chunks"] // -(-batch // win))
    q = p["grid"] // math.gcd(P, p["grid"])
    even = ((wc + q // 2) // q) * q
    if even > 0 and 3 * wc <= 4 * even <= 5 * wc:
        wc = even
    return p, (wc if wc * P >= min_groups * p["grid"] and wc < p["chunks"] else None)


def prn_list(P):
    return [PRN_CYCLE[i % len(PRN_CYCLE)] for i in range(P)]


def doppler_list(D, fs, seed):
    """D bins, unsorted: 1500 Hz twice (the planted satellite's bin, an exact tie), -0.0 next to 0.0, fractional values,
    |f| up to 50 kHz and one bin near fs / 3, then random quarter-hertz bins, none within 1 kHz of 1500 Hz (so that 1500 Hz
    stays the planted satellite's best bin)."""
    head = [1500.0, -0.0, 0.0, -3000.25, 1500.0, 49999.5, -50000.0, fs / 3 + 0.375, 12.125]
    tail = np.round(np.random.default_rng(seed).uniform(-50000.0, 50000.0, 2 * D + 16) * 4) / 4
    tail = tail[np.abs(tail - 1500.0) > 1000.0][:max(0, D - len(head))]
    return np.array(head[:D] + list(tail))


def planted_iq(seed, s, n_ms):
    """PRN entry 4 (SV 5) at 1500 Hz and code phase n - 1, PRN entry 0 (SV 1) at -3000.25 Hz mid-code, in unit noise."""
    n, fs = rate(s)
    return o.synth_iq(seed, n, n_ms, fs, [(5, 1500.0, n - 1, 0.7, 0.3), (1, -3000.25, mid_branch_lag(s), 2.0, 0.3)])


def _divisor(g, lo):
    return next(p for p in range(lo, g + 1) if g % p == 0)


def edge_shape(edge, s, m, kind, sms):
    """(P, nb, D, groups) of the case named edge, for a card of sms SMs."""
    cpg = split_plan(s, m, kind, 0, sms)[2]
    if edge == "one_group":  # a single group with one slot switched off (a one-cell group when a cell takes every slot)
        return 1, 1, max(1, cpg - 1), 1
    if edge == "sms_minus_1":  # P = 1, D = 1: a group's cells span blocks; the last chunk holds one cell
        g = sms - 1
        return 1, (g - 1) * cpg + 1, 1, g
    if edge == "sms":  # one group per CTA, full last chunks, one block with a long Doppler list
        P = _divisor(sms, 3)
        return P, 1, sms // P * cpg, sms
    g = sms + 1 if edge == "sms_plus_1" else 2 * sms + 1  # P divides g, so it is coprime to the sms CTAs
    P = _divisor(g, 2)
    nc = (g // P - 1) * cpg + 1  # last chunk of one cell
    nb = next(k for k in (5, 4, 3, 2, 1) if nc % k == 0)
    return P, nb, nc // nb, g


# ---- running and checking -----------------------------------------------------------------------------------------------
def run_grid_guarded(eng, nb, m, prns, dop, kind):
    """acquire_grid_device and acquire_grid_best_device into CUDA buffers filled with 0xFF, each one grid row longer than its
    output.  Asserts that every record was written and the guard rows were not; returns (records [nb, P, D], best [nb, P])."""
    import torch

    from gypsum_b200 import _native

    prn, d = np.ascontiguousarray(prns, np.int32), np.ascontiguousarray(dop, np.float64)
    k = _native.COHERENT if kind == o.COHERENT else _native.NON_COHERENT
    n_rec, n_best = nb * prn.size * d.size, nb * prn.size
    rec_buf = torch.full(((n_rec + d.size) * 32,), 0xFF, dtype=torch.uint8, device="cuda")
    best_buf = torch.full(((n_best + prn.size) * 32,), 0xFF, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()  # the fills are done before the engine's own stream writes
    eng.acquire_grid_device(nb, m, prn, d, k, rec_buf.data_ptr())
    eng.acquire_grid_best_device(nb, m, prn, d, k, best_buf.data_ptr())
    torch.cuda.synchronize()
    raw, raw_best = rec_buf.cpu().numpy(), best_buf.cpu().numpy()
    assert (raw[n_rec * 32:] == 0xFF).all(), "a record was written past the end of the grid"
    assert (raw_best[n_best * 32:] == 0xFF).all(), "a best-bin row was written past the end"
    rec = raw[:n_rec * 32].view(_native.RECORD_DTYPE).reshape(nb, prn.size, d.size)
    best = raw_best[:n_best * 32].view(_native.BEST_DTYPE).reshape(nb, prn.size)
    assert (rec["reserved"] == 0).all(), f"{np.count_nonzero(rec['reserved'] != 0)} records never written"
    assert (best["reserved"] == 0).all(), "best-bin rows never written"
    host = eng.acquire_grid_best(nb, m, prn, d, k)
    assert host.tobytes() == best.tobytes(), "acquire_grid_best != acquire_grid_best_device"
    return rec, best


def check_best(best, rec, ref, dop, n, what):
    """One block's best-bin rows: the first bin with the largest float32 peak of the block's records (so exact ties go to
    the first), the oracle's first bin with the largest peak unless the two are a near-tie on the float64 peaks, and that
    bin's Doppler (bit for bit), code phase and peak; strength within 1e-4 of the oracle's at that bin."""
    peak, _, total, count = ref
    for a in range(best.size):
        b = int(best["bin"][a])
        assert b == int(np.argmax(rec["peak"][a])), (what, a)
        ob = int(np.argmax(peak[a]))
        assert b == ob or peak[a, ob] - peak[a, b] <= MAG_TOL * peak[a, ob], (what, a, b, ob)
        assert np.float64(best["doppler"][a]).tobytes() == np.float64(dop[b]).tobytes(), (what, a)
        assert (best["code_phase"][a], best["peak"][a]) == (rec["argmax"][a, b], rec["peak"][a, b]), (what, a)
        want = o.strength_from_record(peak[a, b], total[a, b], count[a, b], n)
        assert abs(best["strength"][a] - want) <= 1e-4 * want, (what, a)


def check_run(rec, best, x, s, m, prns, dop, kind, what):
    """Every block of a guarded run against vector_grid; cells with equal (PRN, Doppler) byte-identical."""
    n, fs = rate(s)
    svs = [p + 1 for p in prns]
    for b in range(rec.shape[0]):
        xb = x[b * m * n:(b + 1) * m * n]
        ref = vector_grid(xb, fs, n, svs, dop, kind)[:4]
        check_grid(rec[b], xb, fs, n, svs, dop, (what, b), kind, ref=ref)
        check_best(best[b], rec[b], ref, dop, n, (what, b))
    cells = {}
    for a, p in enumerate(prns):
        for b, f in enumerate(dop):
            cells.setdefault((p, np.float64(f).tobytes()), []).append((a, b))
    for same in cells.values():
        first = rec[:, same[0][0], same[0][1]].tobytes()
        assert all(rec[:, a, b].tobytes() == first for a, b in same[1:]), (what, same)


@pytest.fixture(scope="module")
def engines(native_lib):
    cache = EngineCache()
    yield cache
    cache.close()


@pytest.fixture(scope="module")
def sms(native_lib):
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- the CPU oracle, pinned -----------------------------------------------------------------------------------------------
def test_vector_oracle_matches_grid_cells():
    """vector_grid == o.grid_cells (count and argmax exact, magnitudes within 1e-12) and its probe values == o.integrate, at
    three rates, both kinds, M = 1 and 3, repeated SVs and a Doppler list with fractional, duplicated and signed-zero bins."""
    svs = [5, 1, 5, 32]
    dop = np.array([1500.0, -0.0, 0.0, -3000.25, 1500.0, 777.125, -49999.5])
    for s in (1, 2, 5):
        n, fs = rate(s)
        for m in (1, 3):
            x = planted_iq(40 + s, s, m)
            for kind in (o.NON_COHERENT, o.COHERENT):
                probe = np.random.default_rng(s + m).integers(0, n, (len(svs), dop.size))
                got = vector_grid(x, fs, n, svs, dop, kind, probe)
                want = o.grid_cells(x, fs, n, svs, list(dop), kind)
                what = (s, m, kind)
                assert np.array_equal(got[1], want[1]) and np.array_equal(got[3], want[3]), what
                for g, w in ((got[0], want[0]), (got[2], want[2])):
                    assert np.abs(g - w).max() <= 1e-12 * w.max(), what
                for a, sv in enumerate(svs):
                    for b, f in enumerate(dop):
                        prof = o.integrate(kind, x, fs, n, f, o.replica(sv, n))
                        assert abs(got[4][a, b] - prof[probe[a, b]]) <= 1e-12 * np.abs(prof).max(), what


# ---- 1. the edges of the group partition ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("edge", EDGES)
@pytest.mark.parametrize("kind, m", KINDS)
@pytest.mark.parametrize("s", SPLIT_RATES)
def test_grid_split_edges(engines, sms, s, kind, m, edge):
    """groups = 1 (one slot off), SMs - 1 (P = 1, D = 1 over many blocks, last chunk one cell), SMs (full chunks), SMs + 1
    and 2 SMs + 1 (P coprime to the CTAs, last chunk one cell), each against the oracle, through the guarded buffers."""
    n, fs = rate(s)
    P, nb, D, groups = edge_shape(edge, s, m, kind, sms)
    p = grid_plan(s, m, kind, nb, P, D, sms)
    assert p["n_groups"] == groups, p
    assert p["rsplit"] == split_plan(s, m, kind, 0, sms)[1]
    assert nb * D * unit_bytes(s, m) <= SPEC_BUDGET  # one scratch batch
    cells = nb * D  # per PRN entry
    if edge == "one_group":
        assert cells == max(1, p["cpg"] - 1)
    if edge in ("sms_minus_1", "sms_plus_1", "two_sms_plus_1"):
        assert cells % p["cpg"] == 1 % p["cpg"], p  # last chunk of exactly one cell
    if edge == "sms_minus_1":
        assert (P, D) == (1, 1) and nb == cells
    if edge in ("sms_plus_1", "two_sms_plus_1"):
        assert math.gcd(P, p["grid"]) == 1 and p["grid"] == sms
    seed = 1000 * s + 10 * EDGES.index(edge) + KINDS.index((kind, m))
    prns, dop = prn_list(P), doppler_list(D, fs, seed)
    x = planted_iq(seed, s, nb * m)
    eng = engines(n)
    eng.upload_iq(x)
    rec, best = run_grid_guarded(eng, nb, m, prns, dop, kind)
    check_run(rec, best, x, s, m, prns, dop, kind, (s, m, kind, edge))
    if D >= 5:  # bins 0 and 4 are both 1500 Hz: the planted satellite's rows tie exactly and take the first
        assert (best["bin"][:, [a for a, q in enumerate(prns) if q == 4]] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize("side", ["below", "at"])
def test_rsplit_threshold_sides(engines, sms, side):
    """S = 2, M = 1: one cell short of 8 * SMs * 12 cells (a cell on gcd(2, 12) = 2 warps; 1 block x 1 PRN x that many bins)
    and exactly that many (a whole cell per warp; SMs blocks x 32 PRN entries x 3 bins)."""
    s, m, limit = 2, 1, 8 * sms * 12
    n, fs = rate(s)
    P, nb, D = (1, 1, limit - 1) if side == "below" else (32, sms, 3)
    p = grid_plan(s, m, o.NON_COHERENT, nb, P, D, sms)
    assert nb * P * D == (limit - 1 if side == "below" else limit) and p["rsplit"] == (2 if side == "below" else 1)
    assert nb * D * unit_bytes(s, m) <= SPEC_BUDGET
    prns, dop = prn_list(P), doppler_list(D, fs, 7)
    x = planted_iq(9 if side == "below" else 10, s, nb)
    eng = engines(n)
    eng.upload_iq(x)
    rec, best = run_grid_guarded(eng, nb, m, prns, dop, o.NON_COHERENT)
    check_run(rec, best, x, s, m, prns, dop, o.NON_COHERENT, side)


# ---- 2. cell lists and grids under a small scratch budget ----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("budget_mb", [None, 1])
def test_cell_lists_and_grids_in_scratch_chunks(engines, monkeypatch, sms, budget_mb):
    """acquire_cells, coherent M = 2 with probes, on the split kernels: 74 unsorted cells with repeated (PRN, Doppler) pairs,
    in one chunk under the default budget and, under 1 MB, in chunks of 16 sorted cells with a cut inside one PRN's run.
    A non-coherent grid of 13 blocks x 5 bins runs in one batch, or in batches of 6, 6 and 1 blocks under 1 MB."""
    s, m = 2, 2
    n, fs = rate(s)
    rng = np.random.default_rng(74)
    prns = rng.permutation([4] * 40 + [0] * 15 + [31] * 10 + [17] * 9)
    dop = rng.choice([1500.0, -0.0, 0.0, -3000.25, 777.5], prns.size)
    probe = rng.integers(0, n, prns.size)
    probe[:3] = [0, n - 1, s - 1]
    x = planted_iq(74, s, 13)
    budget = SPEC_BUDGET if budget_mb is None else budget_mb << 20
    _, _, cpg = split_plan(s, m, o.COHERENT, prns.size, sms)
    max_cells = max(cpg, budget // unit_bytes(s, m) // cpg * cpg)
    order = np.argsort(prns, kind="stable")
    cuts = list(range(max_cells, prns.size, max_cells))
    if budget_mb is not None:
        monkeypatch.setenv("GB200_SPEC_BUDGET_MB", str(budget_mb))
        eng = make_engine(fs, n)
        monkeypatch.delenv("GB200_SPEC_BUDGET_MB")
        assert len(cuts) >= 3 and any(prns[order[c - 1]] == prns[order[c]] for c in cuts), cuts
    else:
        eng = engines(n)
        assert not cuts
    from gypsum_b200 import _native

    try:
        eng.upload_iq(x)
        # The records come back through the engine's buffer.  Fill every slot of it with other cells' records first (the fused
        # kernel writes each cell in one launch), so that a cell the split path skips cannot pass on what an earlier call left
        # there, of this engine or of one whose freed buffer this one reuses.
        eng.set_fused(True)
        eng.acquire_cells(prns, dop + 250.0, m, _native.COHERENT, probe_idx=probe)
        eng.set_fused(False)  # the split kernels, whatever the automatic choice would be
        got = eng.acquire_cells(prns, dop, m, _native.COHERENT, probe_idx=probe)
        for i, (pi, f, q) in enumerate(zip(prns, dop, probe)):
            ref = vector_grid(x[:m * n], fs, n, [pi + 1], [f], o.COHERENT, [[q]])
            check_grid(got[i:i + 1][None], x[:m * n], fs, n, [pi + 1], [f], ("cell", i), o.COHERENT, ref=ref[:4])
            assert abs(complex(got["probe_re"][i], got["probe_im"][i]) - ref[4][0, 0]) <= MAG_TOL * ref[0][0, 0], i
        nb, gdop = 13, np.array([1500.0, -0.0, 0.0, -3000.25, 250.5])
        per_batch = max(1, budget // (gdop.size * unit_bytes(s, 1)))
        assert (nb % per_batch != 0) if budget_mb is not None else per_batch >= nb
        gprns = prn_list(7)
        rec, best = run_grid_guarded(eng, nb, 1, gprns, gdop, o.NON_COHERENT)
        check_run(rec, best, x, s, 1, gprns, gdop, o.NON_COHERENT, ("grid", budget_mb))
    finally:
        eng.set_fused(None)
        if budget_mb is not None:
            eng.close()


# ---- 3. L2 windows against the oracle --------------------------------------------------------------------------------------
_WINDOW_CHILD = r"""
import os, sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
os.environ.update(GB200_L2_WINDOW_MB="1", GB200_L2_WINDOW_MIN_GROUPS="0")
from gpu_support import make_engine
from test_gpu_correlate_split import run_grid_guarded
z = np.load(sys.argv[2])
e = make_engine(int(z["fs"]), int(z["n"]))
e.upload_iq(z["x"])
rec, best = run_grid_guarded(e, int(z["nb"]), int(z["m"]), z["prn"], z["dop"], "non_coherent")
np.save(sys.argv[3], rec)
np.save(sys.argv[4], best)
e.close()
print("windows ok")
"""


def window_shape(s, m, sms, rotating):
    """(P, nb, D, chunks per window) of a grid walked in 1 MB windows where no window's groups divide evenly among the CTAs:
    rotating, every window gives each CTA at least one group and the extras go round the CTAs (at least three windows);
    else a full window has fewer groups than CTAs (per_cta = 0) and the last window is ragged."""
    D = 7
    for P in ((37, 41, 43, 47, 53, 59) if rotating else (5, 7, 11)):
        for nb in range(1, 200):
            p, wc = window_plan(s, m, P, D, nb, sms, 1, 0)
            if wc is None or (P * wc) % p["grid"] == 0:
                continue
            n_win = -(-p["chunks"] // wc)
            if rotating and P * wc > p["grid"] and n_win >= 3:
                return P, nb, D, wc
            if not rotating and P * wc < p["grid"] and p["chunks"] % wc != 0:
                return P, nb, D, wc
    raise AssertionError("no such shape")


@pytest.mark.gpu
@pytest.mark.parametrize("rotating", [False, True], ids=["few_groups", "rotating_extras"])
@pytest.mark.parametrize("m", [1, 3])
def test_l2_windows_against_oracle(native_lib, sms, tmp_path, m, rotating):
    """GB200_L2_WINDOW_MB = 1 and GB200_L2_WINDOW_MIN_GROUPS = 0 for an engine created in a child process, S = 2: every
    record of the windowed walk against the oracle and the guard rows, not only against the unwindowed launch."""
    s = 2
    n, fs = rate(s)
    P, nb, D, wc = window_shape(s, m, sms, rotating)
    prns, dop = prn_list(P), doppler_list(D, fs, 5 + m)
    x = planted_iq(20 + m, s, nb * m)
    np.savez(tmp_path / "case.npz", x=x, n=n, fs=fs, nb=nb, m=m, prn=np.array(prns, np.int32), dop=dop)
    run_child(_WINDOW_CHILD, tmp_path / "case.npz", tmp_path / "rec.npy", tmp_path / "best.npy", ok="windows ok")
    rec, best = np.load(tmp_path / "rec.npy"), np.load(tmp_path / "best.npy")
    check_run(rec, best, x, s, m, prns, dop, o.NON_COHERENT, ("windows", m, rotating, P, nb, wc))


# ---- 4. the best-bin reduction on all-zero input ----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("s", [1, 16])
def test_best_bin_of_all_zero_input(engines, s):
    """Every profile value is 0, so every bin ties: bin 0, its Doppler, code phase 0 and peak 0.  The strength, max over the
    mean of the values not equal to the max, is the mean of an empty selection: NaN on the device, as o.peak_strength's
    np.mean gives."""
    from gypsum_b200 import _native

    n, _ = rate(s)
    eng = engines(n)
    eng.upload_iq(np.zeros(2 * 3 * n, np.complex64))
    dop = np.array([-0.0, 0.0, 1500.0, -2500.5])
    for kind, m in ((_native.NON_COHERENT, 1), (_native.NON_COHERENT, 3), (_native.COHERENT, 2)):
        best = eng.acquire_grid_best(2, m, prn_list(3), dop, kind)
        assert (best["bin"] == 0).all() and (best["code_phase"] == 0).all() and (best["peak"] == 0).all(), (s, m)
        assert all(np.float64(d).tobytes() == np.float64(-0.0).tobytes() for d in best["doppler"].ravel()), (s, m)
        assert np.isnan(best["strength"]).all(), (s, m)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        assert np.isnan(o.peak_strength(np.zeros(n)))
