"""What the acquisition test modules share: the tolerances of DESIGN.md section 6, the float64 oracle's grids and searches
spread over the host's cores (fork pool), and the rules that hold the device's records and searches to them."""
import functools
import math
import multiprocessing as mp
import os
import warnings

import numpy as np

from oracle import gypsum_oracle as o

MAG_TOL = 1e-5
DOP41 = np.arange(-10000.0, 10001.0, 500.0)


def rate(s):
    """(n, fs) at S = s samples per chip."""
    return 1023 * s, 1023000 * s


def mid_branch_lag(s):
    """A lag in the middle of the code on the middle polyphase branch (branch s // 2)."""
    return 511 * s + s // 2


def _pool(jobs):
    return mp.get_context("fork").Pool(max(1, min(jobs, os.cpu_count() or 1)))


def _cells_worker(args):
    x, fs, n, svs, dop, kind = args
    return o.grid_cells(x, fs, n, svs, dop, kind)


def oracle_grid(x, fs, n, svs, dop, kind=o.NON_COHERENT):
    """o.grid_cells over all SVs, one process per SV group."""
    procs = max(1, min(len(svs), os.cpu_count() or 1))
    parts = [svs[i::procs] for i in range(procs)]
    with _pool(procs) as pool:
        res = pool.map(_cells_worker, [(x, fs, n, p, list(dop), kind) for p in parts])
    shape = (len(svs), len(dop))
    peak, arg, total, count = (np.zeros(shape), np.zeros(shape, np.int64), np.zeros(shape), np.zeros(shape, np.int64))
    for i, (pk, ag, tt, ct) in enumerate(res):
        rows = list(range(i, len(svs), procs))
        peak[rows], arg[rows], total[rows], count[rows] = pk, ag, tt, ct
    return peak, arg, total, count


@functools.lru_cache(maxsize=None)
def _replica_spectrum(sv, n):
    return np.conj(np.fft.fft(o.replica(sv, n)))


def _vector_cols(x, fs, n, svs, dop, kind, probe):
    uniq = sorted(set(svs))
    rows = [uniq.index(sv) for sv in svs]
    rep = np.stack([_replica_spectrum(sv, n) for sv in uniq])
    shape = (len(svs), len(dop))
    peak, arg, total, count = (np.zeros(shape), np.zeros(shape, np.int64), np.zeros(shape), np.zeros(shape, np.int64))
    val = np.zeros(shape, complex)
    cols = {}  # equal Doppler entries (bit for bit) share one profile
    for b, f in enumerate(dop):
        cols.setdefault(np.float64(f).tobytes(), []).append(b)
    for bs in cols.values():
        f = dop[bs[0]]
        acc = np.zeros((len(uniq), n), dtype=complex if kind == o.COHERENT else np.float64)
        for i in range(len(x) // n):  # o.integrate's arithmetic, every SV of the column at once
            t = (np.arange(n) / fs) + ((i * n) / fs)
            carrier = np.exp(-1j * math.tau * f * t)
            c = np.fft.ifft(np.fft.fft(x[i * n:(i + 1) * n] * carrier)[None, :] * rep, axis=-1)
            if kind == o.COHERENT:
                acc += c
            else:
                acc += np.abs(c)
        mag = np.abs(acc) if kind == o.COHERENT else acc
        mx = mag.max(axis=1)
        for b in bs:
            peak[:, b], arg[:, b], total[:, b] = mx[rows], mag.argmax(axis=1)[rows], mag.sum(axis=1)[rows]
            count[:, b] = np.count_nonzero(mag == mx[:, None], axis=1)[rows]
            if probe is not None:
                val[:, b] = acc[rows, np.asarray(probe)[:, b]]
    return peak, arg, total, count, val


def _apply(args):
    fn, fn_args = args
    return fn(*fn_args)


def by_doppler_column(cols, n_dop, work, part_args):
    """cols(*part_args(p)) over the Doppler columns p of an n_dop-column grid, each result an array whose last axis is the
    Doppler.  Large grids (work: distinct SVs x columns x samples, times the bit phases of a weak grid) are spread over the
    host's cores (fork pool) by Doppler column and put back together."""
    procs = max(1, min(n_dop, os.cpu_count() or 1, work // (1 << 24)))
    if procs == 1:
        return cols(*part_args(slice(None)))
    parts = [np.arange(i, n_dop, procs) for i in range(procs)]
    with _pool(procs) as pool:
        res = pool.map(_apply, [(cols, part_args(p)) for p in parts])
    out = [np.zeros(a.shape[:-1] + (n_dop,), a.dtype) for a in res[0]]
    for p, r in zip(parts, res):
        for o_, a in zip(out, r):
            o_[..., p] = a
    return tuple(out)


def vector_grid(x, fs, n, svs, dop, kind=o.NON_COHERENT, probe=None):
    """o.grid_cells restated for speed, same float64 arithmetic: per (Doppler, ms) one wiped-off forward FFT, its products
    with conj(FFT(replica)) of every SV at once and one batched inverse FFT; repeated SVs and bit-equal Doppler entries are
    computed once.  Returns (peak, argmax, sum, count, probe values), each [len(svs), len(dop)]: probe values are the
    coherent (complex) or non-coherent profile at the lag probe[a, b], zeros without probe.  Large grids are spread over
    the host's cores by Doppler column (by_doppler_column)."""
    dop = np.asarray(dop, dtype=np.float64)
    return by_doppler_column(_vector_cols, dop.size, len(set(svs)) * dop.size * len(x), lambda p: (
        x, fs, n, list(svs), dop[p], kind, None if probe is None else np.asarray(probe)[:, p]))


def check_records(rec, ref, n, profile, what):
    """The tolerances of DESIGN.md section 6 on a grid's records against the oracle's ref = (peak, argmax, sum, count), of
    the same shape: peak and sum within MAG_TOL of the largest, count exact, argmax exact bar near-ties proved on the
    float64 profile(idx) of the cell at index idx, strength within 1e-4.  Returns the number of near-tie proofs."""
    peak, arg, total, count = ref
    assert rec.shape == peak.shape, what
    assert np.abs(rec["peak"] - peak).max() <= MAG_TOL * peak.max(), what
    assert np.abs(rec["sum"] - total).max() <= MAG_TOL * total.max(), what
    assert np.array_equal(rec["count"], count), what
    bad = np.argwhere(rec["argmax"] != arg)
    for idx in map(tuple, bad):  # a different index is only acceptable where the float64 profile itself ties within the tolerance
        prof = profile(idx)
        assert prof.max() - prof[rec["argmax"][idx]] <= MAG_TOL * prof.max(), (what, *idx)
    strength = o.strength_from_record(rec["peak"].astype(np.float64), rec["sum"], rec["count"], n)
    ref_strength = o.strength_from_record(peak, total, count, n)
    assert np.abs(strength - ref_strength).max() <= 1e-4 * ref_strength.max(), what
    return len(bad)


def check_grid(rec, x, fs, n, svs, dop, what, kind=o.NON_COHERENT, ref=None):
    """check_records on a (SV x Doppler) grid.  ref: the oracle's (peak, argmax, sum, count) of the grid when the caller
    has them (vector_grid), else o.grid_cells runs here.  Returns the number of near-tie proofs."""
    ref = ref if ref is not None else oracle_grid(x, fs, n, svs, dop, kind)
    return check_records(rec, ref, n, lambda i: np.abs(o.integrate(kind, x, fs, n, dop[i[1]], o.replica(svs[i[0]], n))),
                         what)


def _cells_cols(x, fs, n, svs, dop, kind, probe, cols):
    """vector_cells over the Doppler columns cols ([cell indices] of one bit-equal Doppler each)."""
    out = []
    for idx in cols:
        pr = None if probe is None else np.asarray(probe)[idx][:, None]
        out.append(_vector_cols(x, fs, n, [svs[i] for i in idx], dop[idx[:1]], kind, pr))
    return out


def _cell_list_worker(args):
    return _cells_cols(*args)


def vector_cells(x, fs, n, svs, dop, kind=o.NON_COHERENT, probe=None):
    """vector_grid for a cell list: cell i is (svs[i], dop[i]), and with probe its profile value at lag probe[i].  Returns
    (peak, argmax, sum, count, probe values), each [len(svs)].  Cells of bit-equal Dopplers share one wiped-off forward FFT
    per millisecond; long lists are spread over the host's cores by Doppler."""
    dop = np.asarray(dop, dtype=np.float64)
    by_dop = {}
    for i, f in enumerate(dop):
        by_dop.setdefault(f.tobytes(), []).append(i)
    cols = list(by_dop.values())
    procs = max(1, min(len(cols), os.cpu_count() or 1, len(cols) * len(x) // (1 << 22)))
    parts = [cols[i::procs] for i in range(procs)]
    if procs == 1:
        res = [_cells_cols(x, fs, n, list(svs), dop, kind, probe, cols)]
    else:
        with _pool(procs) as pool:
            res = pool.map(_cell_list_worker, [(x, fs, n, list(svs), dop, kind, probe, p) for p in parts])
    out = [np.zeros(dop.size, np.float64), np.zeros(dop.size, np.int64), np.zeros(dop.size, np.float64),
           np.zeros(dop.size, np.int64), np.zeros(dop.size, complex)]
    for p, r in zip(parts, res):
        for idx, col in zip(p, r):
            for o_, a in zip(out, col):
                o_[idx] = a[:, 0]
    return tuple(out)


def check_cells(rec, ref, x, fs, n, svs, dop, what, kind=o.NON_COHERENT, probe=None):
    """Every record of a cell list against vector_cells' ref, each against its own profile's maximum: peak and sum within
    MAG_TOL of the oracle's, strength within 1e-4 (NaN where the oracle's is, as for all-zero input), count exact, argmax
    exact bar near-ties proved on the float64 profile; coherent probes within MAG_TOL * peak of the oracle's complex value
    at the probe lag, and exactly 0 without a probe or for non-coherent cells.  Returns the number of near-tie proofs."""
    peak, arg, total, count, val = ref
    assert rec.shape == peak.shape, what
    assert (np.abs(rec["peak"] - peak) <= MAG_TOL * peak).all(), (what, np.flatnonzero(np.abs(rec["peak"] - peak) > MAG_TOL * peak)[:8])
    assert (np.abs(rec["sum"] - total) <= MAG_TOL * total).all(), (what, np.flatnonzero(np.abs(rec["sum"] - total) > MAG_TOL * total)[:8])
    assert np.array_equal(rec["count"], count), (what, np.flatnonzero(rec["count"] != count)[:8])
    bad = np.flatnonzero(rec["argmax"] != arg)
    for i in bad:
        prof = np.abs(o.integrate(kind, x, fs, n, dop[i], o.replica(svs[i], n)))
        assert prof.max() - prof[rec["argmax"][i]] <= MAG_TOL * prof.max(), (what, i, rec["argmax"][i], arg[i])
    with np.errstate(invalid="ignore", divide="ignore"):
        got_s = o.strength_from_record(rec["peak"].astype(np.float64), rec["sum"], rec["count"], n)
        want_s = o.strength_from_record(peak, total, count, n)
    assert np.array_equal(np.isnan(got_s), np.isnan(want_s)), what
    ok = ~np.isnan(want_s)
    assert (np.abs(got_s[ok] - want_s[ok]) <= 1e-4 * want_s[ok]).all(), what
    got_p = rec["probe_re"].astype(np.float64) + 1j * rec["probe_im"]
    if probe is None or kind != o.COHERENT:
        assert (got_p == 0).all(), (what, np.flatnonzero(got_p != 0)[:8])
    else:
        assert (np.abs(got_p - val) <= MAG_TOL * peak).all(), (what, np.flatnonzero(np.abs(got_p - val) > MAG_TOL * peak)[:8])
    return len(bad)


# ---- gb200_acquire_cells' kernel choice (run_cells) -------------------------------------------------------------------
FUSED_CELL_LIMIT = 8192  # lists of at most this many cell-milliseconds always take the fused kernel


def fused_choice(s, dop, m, profile=False):
    """run_cells' automatic choice restated: True for the fused block-per-cell kernel, False for doppler_spectra +
    correlate_cells.  Fused only where it covers the rate (S = 2, 4) and no profile is wanted, and then when more than a
    quarter of the cells have distinct Dopplers or n_cells * M <= 8192.  Distinct as std::sort + std::unique count them:
    -0.0 and 0.0 are one value."""
    n_cells, n_unique = len(dop), len({float(f) for f in dop})
    return s in FUSED_RATES and not profile and (n_unique * 4 > n_cells or n_cells * m <= FUSED_CELL_LIMIT)


def choice_list(case, s, seed):
    """(PRN entries, Dopplers, M) of a list on one side of one of fused_choice's thresholds, unsorted, with -0.0 and 0.0
    both in it (one distinct value; counted as two, "unique_at" would cross its threshold):
      unique_at    4k cells, k distinct Dopplers, n_cells * M > 8192    split
      unique_past  4k cells, k + 1 distinct                             fused
      size_at      n_cells * M == 8192, few distinct                    fused
      size_past    n_cells * M == 8193, few distinct                    split"""
    rng = np.random.default_rng(seed)
    n_cells, m, n_unique = {"unique_at": (2732, 3, 683), "unique_past": (2732, 3, 684), "size_at": (8192, 1, 5),
                            "size_past": (8193, 1, 5)}[case]
    others = rng.permutation(np.arange(1, 4 * n_unique) * 37.25 - 50000.0)[:n_unique - 1]
    values = np.concatenate([[-0.0, 0.0], others])
    dop = np.concatenate([values, rng.choice(values, n_cells - values.size)])[rng.permutation(n_cells)]
    prns = rng.integers(0, 32, n_cells)
    return prns, dop, m


def assert_records_equal(a, b, what, sum_rtol=0):
    """peak, argmax and count exact; sum exact, or within sum_rtol * max(b's sums) where the two launches add a cell's
    values in a different order."""
    for k in ("peak", "argmax", "count"):
        assert np.array_equal(a[k], b[k]), (what, k)
    if sum_rtol:
        assert np.abs(a["sum"] - b["sum"]).max() <= sum_rtol * b["sum"].max(), (what, "sum")
    else:
        assert np.array_equal(a["sum"], b["sum"]), (what, "sum")


def _search_worker(args):
    sv, x, fs, n = args
    trace = []
    r = o.acquire_sv(sv, x, fs, n, trace)
    return r, o.search_is_ambiguous(trace, MAG_TOL)


def oracle_searches(svs, x, fs, n):
    """[(o.acquire_sv result, whether its search sits on a branch point)] per SV, one process each."""
    with _pool(len(svs)) as pool:
        return pool.map(_search_worker, [(sv, x, fs, n) for sv in svs])


def check_search(got, sv, ref, ambiguous, x, fs, n, what):
    """got: (doppler, code_phase, strength, carrier phase) of a search; ref: the same of the float64 search, which is
    ambiguous if it sits on a branch point (two bins' maxima, two profile values or two passes' strengths within the
    tolerance of each other, proved with the oracle's trace)."""
    doppler, code_phase, strength, phase = got
    if ref[2] > o.DETECTION_THRESHOLD:  # detected satellites: everything must agree
        assert (doppler, code_phase) == (ref[0], ref[1]), what
        assert abs(strength - ref[2]) <= 1e-4 * ref[2], what
        d = abs(phase - ref[3])
        assert min(d, 2 * np.pi - d) <= 1e-4, what
    elif (doppler, code_phase) == (ref[0], ref[1]):
        assert abs(strength - ref[2]) <= 1e-4 * ref[2], what
    else:  # noise only: another answer only on a branch point, and then a true cell of the search
        assert ambiguous, what
        prof = o.integrate(o.NON_COHERENT, x, fs, n, doppler, o.replica(sv, n))
        assert abs(o.peak_strength(prof) - strength) <= 1e-4 * strength, what


def _traced_worker(args):
    sv, x, fs, n = args
    trace = []
    with warnings.catch_warnings():  # all-zero input: numpy's mean of an empty slice, the strength NaN (utils.py:111-116)
        warnings.simplefilter("ignore", RuntimeWarning)
        r = o.acquire_sv(sv, x, fs, n, trace)
    return r, trace, o.search_is_ambiguous(trace, MAG_TOL)


def oracle_searches_traced(svs, x, fs, n):
    """{sv: (o.acquire_sv result, its trace, whether it sits on a branch point)}, each distinct SV searched once, one
    process each."""
    uniq = sorted(set(int(sv) for sv in svs))
    with _pool(len(uniq)) as pool:
        return dict(zip(uniq, pool.map(_traced_worker, [(sv, x, fs, n) for sv in uniq])))


# ---- the on-device search's plan (gb200_detect) and the oracle's trace ------------------------------------------------
REFINE_MAX_BINS = 32  # kRefineMaxBins: (satellite, bin) slots per satellite and pass
SPREADS = [7000.0 / 2 ** k for k in range(10)]  # acquisition.py:78-89: 7000 halved while >= 10
DEFAULT_SPEC_BUDGET_MB = 512  # GB200_SPEC_BUDGET_MB when unset
FUSED_RATES = (2, 4)  # fused_supports: the block-per-cell kernel, no spectra scratch and no groups


def refine_slots(center, spread):
    """k_refine_plan restated: Dopplers of a satellite's kRefineMaxBins slots, NaN past the bins of
    range(int(c - s), int(c + s), int(s / 10)) (int() truncates toward zero)."""
    lo, hi, step = int(center - spread), int(center + spread), int(spread / 10)
    return [float(lo + b * step) if lo + b * step < hi else math.nan for b in range(REFINE_MAX_BINS)]


def detect_plan(s, m, n_sv, sms, budget_mb=DEFAULT_SPEC_BUDGET_MB):
    """gb200_detect's schedule at S = s, M = m for n_sv satellites on a card of `sms` SMs with a budget_mb MiB spectra
    budget: the refinement passes' correlate slots per CTA, rsplit, cells per group (cpg), groups per satellite (gps),
    satellites per spectra chunk, the chunks (first satellite, satellites) and each chunk's CTA count; the coherent pass's
    rsplit and CTA count.  The fused kernel (S = 2, 4) runs every pass as one launch of a CTA per slot instead."""
    slots = 12 if m == 1 else 8  # correlate_slots, non-coherent: one-warp kernel
    n_cells = n_sv * REFINE_MAX_BINS
    rsplit = 1 if n_cells >= 8 * sms * slots else math.gcd(s, slots)  # pick_rsplit
    cpg = slots // rsplit
    gps = -(-REFINE_MAX_BINS // cpg)
    unit_bytes = m * s * 2 * 1024 * 8  # unit_floats2 float2s: one (block, Doppler) spectra unit
    spc = min(max(1, (budget_mb << 20) // (unit_bytes * REFINE_MAX_BINS)), n_sv)
    chunks = [(sv0, min(spc, n_sv - sv0)) for sv0 in range(0, n_sv, spc)]
    crsplit = 1 if n_sv >= 8 * sms * 8 else math.gcd(s, 8)  # coherent pass: warp-pair kernel, 8 pairs
    return dict(slots=slots, rsplit=rsplit, cpg=cpg, gps=gps, group_sizes=[min(cpg, REFINE_MAX_BINS - g * cpg)
                for g in range(gps)], sv_per_chunk=spc, chunks=chunks, grids=[min(k * gps, sms) for _, k in chunks],
                crsplit=crsplit, coherent_grid=min(n_sv, sms), fused=s in FUSED_RATES)


def budget_for(s, m, n_sv, spc, sms, limit_mb=4096):
    """The smallest whole-MiB budget (>= 1) whose plan has spc satellites per chunk, or None."""
    for mb in range(1, limit_mb + 1):
        got = detect_plan(s, m, n_sv, sms, mb)["sv_per_chunk"]
        if got == spc:
            return mb
        if got > spc:
            return None
    return None


def trace_passes(trace):
    """[(centre, spread, chosen Doppler, strength)] of each pass of an o.acquire_sv trace."""
    out, centre = [], 0.0
    for spread, p in zip(SPREADS, trace):
        out.append((centre, spread, p["chosen"], p["strength"]))
        centre = p["chosen"]
    return out


def kept_pass(trace):
    """1-based pass whose result the search keeps: the first pass, replaced only by a strictly greater strength (NaN
    never replaces and is never replaced)."""
    kept, best = 1, trace[0]["strength"]
    for k, p in enumerate(trace[1:], 2):
        if p["strength"] > best:
            kept, best = k, p["strength"]
    return kept


def centre_outside(trace, limit=7000.0):
    """Whether a pass of the search is centred beyond +-limit Hz."""
    return any(abs(c) > limit for c, _, _, _ in trace_passes(trace))


def truncation_differs(trace):
    """Whether a pass's lower edge c - spread is a negative non-integer, where int() (toward zero) and floor differ."""
    return any(c - s < 0 and c - s != math.floor(c - s) for c, s, _, _ in trace_passes(trace))


def centre_crosses_zero(trace):
    """Whether consecutive pass centres (pass 1's 0 excluded) lie on both sides of zero."""
    cs = [c for c, _, _, _ in trace_passes(trace)[1:]] + [trace[-1]["chosen"]]
    return any(a * b < 0 for a, b in zip(cs, cs[1:]))


def _is_ambiguous(sv, x, fs, n):
    trace = []
    o.acquire_sv(sv, x, fs, n, trace)
    return o.search_is_ambiguous(trace, MAG_TOL)


def check_detector_golden(det, ids, x, attrs, detected, rows, fs, n, what):
    """GpsSatelliteDetector against the live reference's detector: the satellites found, each recorded result row (sv,
    doppler, carrier phase, code phase, strength) by check_search, and the on-device search (_acquire_many) against the
    pass-by-pass search from the host (_acquire_many_stepwise), the same algorithm on other kernels.  Returns the
    on-device results by SV."""
    found = det.detect_satellites_in_antenna_data(ids, x, attrs)
    assert [r.satellite_id.id for r in found] == [int(sv) for sv in detected], what
    many = det._acquire_many(ids, x, attrs)
    results = {r.satellite_id.id: r for r in many}
    for row in rows:
        sv = int(row[0])
        r = results[sv]
        ambiguous = (r.doppler_shift, r.prn_phase_shift) != (int(row[1]), int(row[3])) and _is_ambiguous(sv, x, fs, n)
        check_search((r.doppler_shift, r.prn_phase_shift, r.correlation_strength, r.carrier_wave_phase_shift), sv,
                     (int(row[1]), int(row[3]), row[4], row[2]), ambiguous, x, fs, n, (what, sv))
    # identical decisions for the detected satellites, values equal to float32 rounding
    for a, b in zip(many, det._acquire_many_stepwise(ids, x, attrs)):
        if (a.doppler_shift, a.prn_phase_shift) != (b.doppler_shift, b.prn_phase_shift):
            sv = a.satellite_id.id
            assert b.correlation_strength <= o.DETECTION_THRESHOLD, (what, sv)  # detected satellites: never
            assert _is_ambiguous(sv, x, fs, n), (what, sv)
            continue
        assert abs(a.correlation_strength - b.correlation_strength) <= 1e-5 * b.correlation_strength, what
        d = abs(a.carrier_wave_phase_shift - b.carrier_wave_phase_shift)
        assert min(d, 2 * np.pi - d) <= 1e-4 or b.correlation_strength <= o.DETECTION_THRESHOLD, what
    return results
