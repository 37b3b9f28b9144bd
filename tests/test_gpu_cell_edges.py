"""The block-per-cell acquisition kernel and the per-cell entry points at every edge, against the float64 oracle.

`k_acquire_fused` (fused.cu) evaluates one (PRN, Doppler) cell per CTA at 2.046 and 4.092 Msps: its own wipe-off into the
polyphase rows, a TMA double buffer of IQ whose mbarrier phase alternates per millisecond, coherent sums in registers and
its own probe match.  It runs every pass of gb200_detect there, and gb200_acquire_cells picks it automatically for lists of
mostly distinct Dopplers or few cell-milliseconds (`run_cells`).  Here it is forced on for lists of 1 cell, one resident
wave of CTAs and one wave + 1, at M = 1, 2, 3, 10 and 20, with code phases at 0, n - 1 and on every polyphase branch,
coherent probes at both ends of the code and on every branch, -0.0 next to 0.0, fractional, +-50 kHz and non-kHz
Dopplers (where the carrier's millisecond term matters), and repeated cells that must be byte-identical.  The same cells
run through the split kernels, the automatic choice at its thresholds, the kernel reading a device ring at every slot,
both profile entry points at all ten rates, and the drop-in helpers' roll undo.  Before every call under test the other
kernels fill the engine's record buffer with other cells, so a record the kernel skips cannot pass.

Every record is checked through acq_support.check_cells against vector_cells (tolerances of DESIGN.md section 6, each cell
against its own profile's maximum).  A non-finite Doppler is refused by every entry point that takes one (EINVAL,
ValueError), and the engine goes on as a fresh one would."""
import math

import numpy as np
import pytest

from acq_support import (FUSED_RATES, MAG_TOL, check_cells, choice_list, fused_choice, mid_branch_lag, rate,
                         vector_cells)
from gpu_support import Attrs, EngineCache, make_engine
from oracle import gypsum_oracle as o

ALL_RATES = [1, 2, 3, 4, 5, 6, 8, 10, 12, 16]
MS = [1, 2, 3, 10, 20]
SIZES = ["one", "wave", "wave_plus_1"]
SPEC_BUDGET = 512 << 20  # the engine's default scratch budget (GB200_SPEC_BUDGET_MB)
OTHER = 250.0  # Hz between the cells of the call that fills the record buffer and the cells of the call under test
EXTRA = [(4, -0.0), (4, 0.0), (31, 12.125), (17, -777.75), (2, 50000.0), (2, -50000.0), (9, 49999.5), (30, 1234.5),
         (31, -0.0)]  # (PRN entry, Doppler) cells beside the planted ones


def planted(s):
    """(SV, Doppler, code phase) of the planted satellites: n - 1, 0 and lag 511 S + r on every branch r.  No Doppler is a
    multiple of 1 kHz, so each millisecond's carrier differs from the first's by a phase a coherent sum sees."""
    n, _ = rate(s)
    return [(5, 1500.0, n - 1), (1, -3000.25, 0)] + [(10 + r, 700.5 + 1000.0 * r, 511 * s + r) for r in range(s)]


def planted_iq(seed, s, m):
    n, fs = rate(s)
    return o.synth_iq(seed, n, m, fs, [(sv, f, cp, 0.3 + sv, 0.7) for sv, f, cp in planted(s)])


def probe_lags(s):
    """0, 1, S - 1, N - S, N - 1 and one lag on every branch."""
    n, _ = rate(s)
    return [0, 1, s - 1, n - s, n - 1] + [511 * s + r for r in range(s)]


def wave(s, sms):
    """CTAs of one resident wave of the fused kernel: three per SM at S = 2, one at S = 4 (__launch_bounds__)."""
    return (3 if s == 2 else 1) * sms


def cell_list(s, size, sms, seed):
    """(PRN entries, Dopplers, probe lags, {index: planted code phase}) of an unsorted list: the planted cells (probed at
    their code phase), EXTRA, the first two planted cells again (same probes), then random quarter-hertz cells up to the
    size.  size "one" is the planted n - 1 cell alone."""
    n, _ = rate(s)
    cells = [(sv - 1, f, cp, cp) for sv, f, cp in planted(s)]
    if size == "one":
        cells = cells[:1]
    else:
        lags = probe_lags(s)
        cells += [(p, f, lags[i % len(lags)], None) for i, (p, f) in enumerate(EXTRA)] + cells[:2]
        target = wave(s, sms) + (size == "wave_plus_1")
        rng = np.random.default_rng(seed)
        while len(cells) < target:
            cells.append((int(rng.integers(0, 32)), float(np.round(rng.uniform(-50000, 50000) * 4) / 4),
                          lags[len(cells) % len(lags)], None))
        cells = [cells[i] for i in rng.permutation(len(cells))]
    prns = np.array([c[0] for c in cells], np.int32)
    dop = np.array([c[1] for c in cells])
    probe = np.array([c[2] for c in cells], np.int32)
    return prns, dop, probe, {i: c[3] for i, c in enumerate(cells) if c[3] is not None}


def split_chunks(s, m, n_cells, sms):
    """Scratch chunks of a non-coherent list on the split kernels (run_cells), two launches each: cells per group from
    correlate_slots (12 warps at M = 1, else 8) and pick_rsplit, chunks of whole groups whose spectra fit the budget."""
    slots = 12 if m == 1 else 8
    cpg = slots // (1 if n_cells >= 8 * sms * slots else math.gcd(s, slots))
    max_cells = max(cpg, SPEC_BUDGET // (m * s * 2 * 1024 * 8) // cpg * cpg)
    return -(-n_cells // max_cells)


def kind_of(kind):
    from gypsum_b200 import _native

    return _native.COHERENT if kind == o.COHERENT else _native.NON_COHERENT


def run_cells(eng, fused, prns, dop, m, kind, probe=None):
    """acquire_cells on the fused (True) or split (False) kernels after the other kernels filled the engine's record buffer
    with the same PRNs OTHER Hz away.  Returns (records, launches)."""
    eng.set_fused(not fused)
    eng.acquire_cells(prns, np.asarray(dop) + OTHER, m, kind_of(kind), probe_idx=probe)
    eng.set_fused(fused)
    n0 = eng.launch_count
    rec = eng.acquire_cells(prns, dop, m, kind_of(kind), probe_idx=probe)
    return rec, eng.launch_count - n0


def assert_repeats_identical(rec, prns, dop, probe, what):
    """Cells of equal (PRN, Doppler bits, probe) are byte-identical."""
    same = {}
    for i, key in enumerate(zip(prns.tolist(), [f.tobytes() for f in np.asarray(dop)], probe.tolist())):
        same.setdefault(key, []).append(i)
    repeated = [ix for ix in same.values() if len(ix) > 1]
    for ix in repeated:
        assert all(rec[i].tobytes() == rec[ix[0]].tobytes() for i in ix[1:]), (what, ix)
    return len(repeated)


@pytest.fixture(scope="module")
def engines(native_lib):
    cache = EngineCache()
    yield cache
    cache.close()


@pytest.fixture(scope="module")
def sms(native_lib):
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- 1. the fused kernel forced on, and the same cells on the split kernels ------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("m", MS)
@pytest.mark.parametrize("kind", [o.NON_COHERENT, o.COHERENT])
@pytest.mark.parametrize("s", FUSED_RATES)
def test_fused_and_split_cells(engines, sms, s, kind, m, size):
    """Every record of the fused kernel (one launch) against the oracle; planted cells at their code phase, repeated cells
    byte-identical; coherent without probes: the same records with probe exactly 0.  The same list on the split kernels
    (one doppler_spectra and one correlate launch) against the oracle, and within float32 rounding of the fused records."""
    n, fs = rate(s)
    seed = 100 * s + 10 * MS.index(m) + SIZES.index(size) + (5 if kind == o.COHERENT else 0)
    prns, dop, probe, plant = cell_list(s, size, sms, seed)
    assert prns.size == (1 if size == "one" else wave(s, sms) + (size == "wave_plus_1"))
    x = planted_iq(seed, s, m)
    pr = probe if kind == o.COHERENT else None
    svs = [int(p) + 1 for p in prns]
    ref = vector_cells(x, fs, n, svs, dop, kind, pr)
    assert all(ref[1][i] == cp for i, cp in plant.items()), "a planted cell is not at its code phase in the oracle"
    eng = engines(n)
    eng.upload_iq(x)
    what = (s, kind, m, size)
    try:
        fused, launches = run_cells(eng, True, prns, dop, m, kind, pr)
        assert launches == 1, (what, launches)
        check_cells(fused, ref, x, fs, n, svs, dop, ("fused",) + what, kind, pr)
        assert all(fused["argmax"][i] == cp for i, cp in plant.items()), what
        if size != "one":
            assert assert_repeats_identical(fused, prns, dop, probe, what) >= 2
        if kind == o.COHERENT:
            bare, _ = run_cells(eng, True, prns, dop, m, kind, None)
            assert (bare["probe_re"] == 0).all() and (bare["probe_im"] == 0).all(), what
            for k in ("peak", "argmax", "sum", "count"):
                assert np.array_equal(bare[k], fused[k]), (what, k)
        split, launches = run_cells(eng, False, prns, dop, m, kind, pr)
        assert launches == 2, (what, launches)
        check_cells(split, ref, x, fs, n, svs, dop, ("split",) + what, kind, pr)
        assert (np.abs(fused["peak"] - split["peak"]) <= 2e-6 * split["peak"]).all(), what
        assert (np.abs(fused["sum"] - split["sum"]) <= 2e-6 * split["sum"]).all(), what
        assert np.array_equal(fused["count"], split["count"]), what
        if kind == o.COHERENT:
            d = np.abs((fused["probe_re"] - split["probe_re"]) + 1j * (fused["probe_im"] - split["probe_im"]))
            assert (d <= 2e-6 * split["peak"]).all(), what
    finally:
        eng.set_fused(None)


@pytest.mark.gpu
@pytest.mark.parametrize("s", FUSED_RATES)
def test_all_zero_iq_cells(engines, s):
    """All-zero IQ on both kernels, both kinds, M = 1, 2 and 3: argmax 0, peak 0, sum 0, count N, probe 0 and a NaN
    strength, as numpy gives; the record buffer was filled from noise first."""
    from gypsum_b200 import _native

    n, fs = rate(s)
    prns = np.array([4, 0, 31, 4], np.int32)
    dop = np.array([-0.0, 0.0, 1500.0, -2500.5])
    probe = np.array([0, n - 1, s - 1, 511 * s + 1], np.int32)
    noise = planted_iq(3, s, 3)
    zero = np.zeros(3 * n, np.complex64)
    eng = engines(n)
    try:
        for kind, m in ((o.NON_COHERENT, 1), (o.NON_COHERENT, 2), (o.COHERENT, 1), (o.COHERENT, 3)):
            for fused in (True, False):
                pr = probe if kind == o.COHERENT else None
                eng.upload_iq(noise)
                eng.set_fused(not fused)
                eng.acquire_cells(prns, dop, m, kind_of(kind), probe_idx=pr)
                eng.upload_iq(zero)
                eng.set_fused(fused)
                rec = eng.acquire_cells(prns, dop, m, kind_of(kind), probe_idx=pr)
                what = (s, kind, m, fused)
                assert (rec["argmax"] == 0).all() and (rec["peak"] == 0).all() and (rec["sum"] == 0).all(), what
                assert (rec["count"] == n).all() and (rec["probe_re"] == 0).all() and (rec["probe_im"] == 0).all(), what
                with np.errstate(invalid="ignore", divide="ignore"):
                    assert np.isnan(_native.strength_from_records(rec, n)).all(), what
    finally:
        eng.set_fused(None)


# ---- 2. the automatic choice at its thresholds --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["unique_at", "unique_past", "size_at", "size_past"])
@pytest.mark.parametrize("s", [2, 3, 4])
def test_automatic_choice_at_thresholds(engines, sms, s, case):
    """Lists exactly at and one past each threshold of run_cells' choice (acq_support.choice_list; -0.0 and 0.0 in each):
    the kernel that ran, told by the launch count (1 fused, 2 per scratch chunk split), is the one fused_choice names, and
    every record is the oracle's, written over the records of the same list OTHER Hz away.  At S = 3 the split kernels run
    whatever the list; at S = 4 the split lists fill the scratch budget twice, the second chunk holding a few cells."""
    n, fs = rate(s)
    prns, dop, m = choice_list(case, s, 20 + s)
    want_fused = fused_choice(s, dop, m)
    assert want_fused == (s != 3 and case in ("unique_past", "size_at"))
    x = planted_iq(30 + s, s, m)
    eng = engines(n)
    eng.upload_iq(x)
    try:
        eng.acquire_cells(prns, dop + OTHER, m, kind_of(o.NON_COHERENT))  # the same choice: OTHER keeps the distinct count
        n0 = eng.launch_count
        rec = eng.acquire_cells(prns, dop, m, kind_of(o.NON_COHERENT))
        launches = eng.launch_count - n0
        chunks = split_chunks(s, m, prns.size, sms)
        assert launches == (1 if want_fused else 2 * chunks), (s, case, launches, chunks)
        svs = [int(p) + 1 for p in prns]
        check_cells(rec, vector_cells(x, fs, n, svs, dop), x, fs, n, svs, dop, (s, case))
    finally:
        eng.set_fused(None)


# ---- 3. the fused kernel reading a device ring -----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("s", FUSED_RATES)
def test_fused_from_device_ring(native_lib, sms, s):
    """A 7-ms ring fed one millisecond at a time up to 12: after 8 to 12 appends, the newest 1, 3 and 7 ms (windows starting
    at every slot, odd and even, crossing the mirror boundary) through the fused kernel == upload_iq of the same samples +
    acquire_cells, both kinds, byte for byte; one window of each size against the oracle."""
    from gypsum_b200 import _native

    n, fs = rate(s)
    x = planted_iq(40 + s, s, 12)
    prns, dop, probe, _ = cell_list(s, "wave", 12, 7)  # the planted and EXTRA cells and a few random ones
    eng = make_engine(fs, n)
    ring = _native.Ring(eng, 7)
    starts, crossing, checked = set(), False, set()
    try:
        for k in range(12):
            ring.append(x[k * n:(k + 1) * n])
            a = k + 1
            if a < 8:
                continue
            for w in (1, 3, 7):
                first = (a - w) % 7
                starts.add(first)
                crossing |= first + w > 7
                for kind in (o.NON_COHERENT, o.COHERENT):
                    pr = probe if kind == o.COHERENT else None
                    ring.bind_newest(w)
                    got, launches = run_cells(eng, True, prns, dop, w, kind, pr)
                    assert launches == 1
                    eng.upload_iq(x[(a - w) * n:a * n])
                    want, _ = run_cells(eng, True, prns, dop, w, kind, pr)
                    assert got.tobytes() == want.tobytes(), (s, a, w, kind)
                    if (w, kind) not in checked:
                        checked.add((w, kind))
                        xw = x[(a - w) * n:a * n]
                        svs = [int(p) + 1 for p in prns]
                        check_cells(got, vector_cells(xw, fs, n, svs, dop, kind, pr), xw, fs, n, svs, dop, (s, a, w), kind, pr)
        assert starts == set(range(7)) and crossing
    finally:
        eng.set_fused(None)
        eng.close()


# ---- 4. the profile entry points at all ten rates -------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("s", ALL_RATES)
def test_correlation_profile_every_lag(engines, s):
    """correlation_profile, non-coherent M = 1 and 3 and coherent M = 2, every lag against o.integrate; the satellite is
    planted at lags 0, N - 1 and the last lag of every branch, each of which is checked by name."""
    from gypsum_b200 import _native

    n, fs = rate(s)
    lags = sorted({0, n - 1} | {1022 * s + r for r in range(s)})
    x = o.synth_iq(50 + s, n, 3, fs, [(5, 1500.25, lag, 0.3, 0.5) for lag in lags])
    eng = engines(n)
    eng.upload_iq(x)
    for kind, m in ((o.NON_COHERENT, 1), (o.NON_COHERENT, 3), (o.COHERENT, 2)):
        got = eng.correlation_profile(4, 1500.25, m, kind_of(kind)).astype(np.complex128 if kind == o.COHERENT else np.float64)
        want = o.integrate(kind, x[:m * n], fs, n, 1500.25, o.replica(5, n))
        tol = MAG_TOL * np.abs(want).max()
        assert np.abs(got - want).max() <= tol, (s, kind, m)
        for lag in lags:
            assert abs(got[lag] - want[lag]) <= tol and abs(want[lag]) > 0.5 * np.abs(want).max(), (s, kind, m, lag)
        mag, wmag = np.abs(got), np.abs(want)
        assert wmag.max() - wmag[int(mag.argmax())] <= tol, (s, kind, m)


@pytest.mark.gpu
@pytest.mark.parametrize("s", ALL_RATES)
def test_generic_replica_profile_every_lag(engines, s):
    """correlation_profile_replica with a random complex replica and a +-1 sequence that is not chip-repeated (planted at
    lag N - 1), M = 1 and 3, both kinds: every lag against o.integrate (N = 1023 ends on a partial 1024-sample chunk)."""
    n, fs = rate(s)
    rng = np.random.default_rng(60 + s)
    cplx = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    pm1 = rng.choice([-1.0, 1.0], n).astype(np.complex64)
    if s > 1:
        assert not all(np.array_equal(np.repeat(np.roll(pm1.real, -p)[::s], s), np.roll(pm1.real, -p)) for p in range(s))
    t = np.arange(3 * n) / fs
    x = (o.synth_iq(70 + s, n, 3, fs, []) + 0.5 * np.tile(np.roll(pm1, n - 1), 3) * np.exp(1j * math.tau * 1500.25 * t))
    x = x.astype(np.complex64)
    eng = engines(n)
    eng.upload_iq(x)
    for name, rep in (("complex", cplx), ("pm1", pm1)):
        for kind in (o.NON_COHERENT, o.COHERENT):
            for m in (1, 3):
                got = eng.correlation_profile_replica(rep, 1500.25, m, kind_of(kind))
                want = o.integrate(kind, x[:m * n], fs, n, 1500.25, rep.astype(np.complex128))
                assert np.abs(got - want).max() <= MAG_TOL * np.abs(want).max(), (s, name, kind, m)
                if name == "pm1":
                    assert int(np.abs(got).argmax()) == n - 1, (s, kind, m)


@pytest.mark.gpu
@pytest.mark.parametrize("s", [2, 3, 4, 16])
def test_drop_in_utils_rolled_replicas(native_lib, s):
    """integrate_correlation_with_doppler_shifted_prn and frequency_domain_correlation with the replica rolled by 0, 1,
    S - 1, S, S + 1, N - S and N - 1 == o.integrate / o.correlate_1ms with the same rolled replica, every lag, both kinds,
    over 2 ms and a trailing partial chunk."""
    from gypsum_b200 import utils

    n, fs = rate(s)
    x = o.synth_iq(80 + s, n, 2, fs, [(5, 1500.25, mid_branch_lag(s), 0.3, 0.6)])
    data = np.concatenate([x, x[:n // 3]])
    for k in sorted({0, 1, s - 1, s, s + 1, n - s, n - 1}):
        rep = np.roll(o.replica(5, n), k)
        for it, kind in ((utils.IntegrationType.NonCoherent, o.NON_COHERENT), (utils.IntegrationType.Coherent, o.COHERENT)):
            got = utils.integrate_correlation_with_doppler_shifted_prn(it, data, Attrs(fs, n), 1500.25, rep)
            want = o.integrate(kind, data, fs, n, 1500.25, rep)
            assert got.dtype == want.dtype and np.abs(got - want).max() <= MAG_TOL * np.abs(want).max(), (s, k, kind)
            assert int(np.abs(got).argmax()) == (mid_branch_lag(s) - k) % n, (s, k, kind)
        got = utils.frequency_domain_correlation(x[:n], rep)
        want = o.correlate_1ms(x[:n].astype(np.complex128), rep)
        assert np.abs(got - want).max() <= MAG_TOL * np.abs(want).max(), (s, k)


# ---- 5. non-finite Dopplers ----------------------------------------------------------------------------------------------
def valid_calls(eng, x, n, gdop, prns, cdop, probe):
    """Every entry point that takes a Doppler, on valid arguments: their outputs as bytes, in call order."""
    from gypsum_b200 import _native

    nc, co = kind_of(o.NON_COHERENT), kind_of(o.COHERENT)
    eng.upload_iq(x)
    out = [eng.acquire_grid(1, 2, prns[:3], gdop).tobytes(), eng.acquire_grid_best(1, 2, prns[:3], gdop, co).tobytes()]
    for mode in (True, False, None):
        eng.set_fused(mode)
        out.append(eng.acquire_cells(prns, cdop, 2, co, probe_idx=probe).tobytes())
    eng.set_fused(None)
    out += [eng.correlation_profile(4, 1500.0, 2, nc).tobytes(), eng.correlation_profile(4, 1500.0, 2, co).tobytes(),
            eng.correlation_profile_replica(o.replica(5, n), 1500.0, 2, co).tobytes()]
    out.append(eng.acquire_grid_host(x[:2 * n], 1, 2, prns[:3], gdop).tobytes())
    gs = _native.GridStream(eng, 1, 2, prns[:3], gdop)
    gs.submit(x[:2 * n])
    out.append(gs.collect().tobytes())
    gs.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("bad", [math.nan, math.inf, -math.inf], ids=["nan", "inf", "minus_inf"])
def test_non_finite_doppler_refused(native_lib, bad):
    """NaN, +inf and -inf as one bin of a grid (acquire_grid, _best, _device, _best_device, _host, GridStream), one cell of
    a list (fused, split and automatic) and the Doppler of both profile calls: ValueError naming the first bad index.
    Afterwards every entry point gives what a fresh engine gives, byte for byte."""
    import torch

    from gypsum_b200 import _native

    s = 2
    n, fs = rate(s)
    x = planted_iq(90, s, 2)
    prns = np.array([4, 0, 17, 4, 31, 9, 0, 2, 4], np.int32)
    gdop = np.array([1500.0, -0.0, 0.0, bad, 250.5])
    cdop = np.array([1500.0, -3000.25, 0.0, -0.0, 49999.5, bad, 1500.0, bad, 12.125])
    probe = np.array([n - 1, 0, 1, s - 1, n - s, 511 * s, n - 1, 0, 511 * s + 1], np.int32)
    nc, co = kind_of(o.NON_COHERENT), kind_of(o.COHERENT)
    eng = make_engine(fs, n)
    fresh = None
    try:
        eng.upload_iq(x)
        p3 = prns[:3].copy()
        rec_buf = torch.zeros(3 * gdop.size * 32, dtype=torch.uint8, device="cuda")
        best_buf = torch.zeros(3 * 32, dtype=torch.uint8, device="cuda")
        grid_calls = [
            lambda: eng.acquire_grid(1, 2, p3, gdop),
            lambda: eng.acquire_grid_best(1, 2, p3, gdop, co),
            lambda: eng.acquire_grid_device(1, 2, p3, gdop, nc, rec_buf.data_ptr()),
            lambda: eng.acquire_grid_best_device(1, 2, p3, gdop, nc, best_buf.data_ptr()),
            lambda: eng.acquire_grid_host(x, 1, 2, p3, gdop),
            lambda: _native.GridStream(eng, 1, 2, p3, gdop),
        ]
        for i, call in enumerate(grid_calls):
            with pytest.raises(ValueError, match="Doppler 3 is not finite"):
                call()
        torch.cuda.synchronize()
        assert not rec_buf.any() and not best_buf.any(), "a refused grid call wrote records"
        for mode in (True, False, None):
            eng.set_fused(mode)
            for kind, pr in ((nc, None), (co, probe)):
                with pytest.raises(ValueError, match="Doppler 5 is not finite"):
                    eng.acquire_cells(prns, cdop, 2, kind, probe_idx=pr)
        eng.set_fused(None)
        for kind in (nc, co):
            with pytest.raises(ValueError, match="Doppler 0 is not finite"):
                eng.correlation_profile(4, bad, 2, kind)
            with pytest.raises(ValueError, match="Doppler 0 is not finite"):
                eng.correlation_profile_replica(o.replica(5, n), bad, 2, kind)
        good_g, good_c = np.where(np.isfinite(gdop), gdop, 3000.5), np.where(np.isfinite(cdop), cdop, -1234.5)
        got = valid_calls(eng, x, n, good_g, prns, good_c, probe)
        fresh = make_engine(fs, n)
        want = valid_calls(fresh, x, n, good_g, prns, good_c, probe)
        assert [g == w for g, w in zip(got, want)] == [True] * len(want)
        # the records are the oracle's, so equality is not two engines agreeing on something stale
        rec = np.frombuffer(got[2], _native.RECORD_DTYPE)
        svs = [int(p) + 1 for p in prns]
        check_cells(rec, vector_cells(x, fs, n, svs, good_c, o.COHERENT, probe), x, fs, n, svs, good_c, bad, o.COHERENT,
                    probe)
    finally:
        eng.close()
        if fresh is not None:
            fresh.close()
