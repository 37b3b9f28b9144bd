"""Weak grids (gb200_acquire_grid_weak*, GpsSatelliteDetector.search_weak_satellites) against the float64 oracle of
tests/weak_support.py, with the tolerances of DESIGN.md section 6: magnitudes and sums within 1e-5 of the grid's largest,
count exact, strength 1e-4 relative, argmax and best bin exact unless the oracle's own float64 profile ties within the
tolerance (proved per mismatch).

The bit phases' segment sums and the code-Doppler realignment run in k_aligned_segment_spectra<S>, one instantiation per
rate, whose first launches happen in a child process; the correlate launch is the non-coherent one over the K segment
spectra of each folded (bit phase, Doppler) unit."""
import numpy as np
import pytest

import weak_support as ws
from acq_support import MAG_TOL, mid_branch_lag, rate
from gpu_support import Attrs, EngineCache, run_child
from oracle import gypsum_oracle as o

pytestmark = pytest.mark.gpu
RATES = [1, 2, 3, 4, 5, 6, 8, 10, 12, 16]

_FIRST_RUN_SCRIPT = r"""
import sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
from gpu_support import make_engine
from oracle import gypsum_oracle as o

for s in (1, 2, 3, 4, 5, 6, 8, 10, 12, 16):
    n, fs = 1023 * s, 1023000 * s
    x = o.synth_iq(s, n, 5, fs, [(25, 1500.0, n - 1, 0.3, 0.3)])
    eng = make_engine(fs, n)
    eng.upload_iq(x)
    dop = np.arange(-2000.0, 2001.0, 250.0)
    for t, b, m in ((2, 2, 5), (1, 1, 4), (4, 1, 4)):
        g = eng.acquire_grid_weak(1, m, t, b, [24, 3], dop)[0]
        assert all(int(g["argmax"][0, j, 14]) == n - 1 and int(np.argmax(g["peak"][0, j])) == 14 for j in range(b)), (s, t, b)
    eng.close()
print("aligned segments ok")
"""


def test_first_run_of_the_aligned_segment_kernels_in_a_child_process(native_lib):
    """Runs first, in its own process, so that a fault in a never-exercised kernel cannot disturb the CUDA context of
    the tests below."""
    run_child(_FIRST_RUN_SCRIPT, ok="aligned segments ok")


@pytest.fixture(scope="module")
def engines(native_lib):
    cache = EngineCache()
    yield cache
    cache.close()


def _prn(svs):
    return [sv - 1 for sv in svs]


def _check_found(rec, svs, dop, planted, what):
    """Each planted satellite's best folded bin has its Doppler (within 125 Hz) and its code phase exactly."""
    for sv, f, tau, *_ in planted:
        a = svs.index(sv)
        _, j, d = ws.best_folded(rec["peak"][a])
        assert abs(dop[d] - f) <= 125.0 and int(rec["argmax"][a, j, d]) == tau, (what, sv)


# ---- every rate ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", RATES)
def test_every_rate(engines, s):
    """T = 2, B = 2, M = 33 (K = 16) at every rate, on a grid with fractional, -0.0 and +-50 kHz Dopplers whose shifts
    reach 1 (S = 1) to 17 (S = 16) samples; satellites planted with code Doppler at +50 kHz and two small Dopplers.  The
    best records are the oracle's first folded bin with the largest peak, and agree with the full records."""
    n, fs = rate(s)
    svs = [3, 11, 19, 32]
    dop = np.array([-50000.0, -1250.0, -0.0, 500.0, 1737.5, 50000.0])
    planted = [(3, 50000.0, 0, 1.0, 0.12, 0, None), (11, 1737.5, mid_branch_lag(s), 2.0, 0.12, 7, None),
               (32, -1250.0, n - 1, 2.5, 0.12, 3, None)]
    assert ws.shift(32, n, 50000.0) >= 1
    x = ws.synth_weak_iq(900 + s, n, 33, fs, planted)
    eng = engines(n)
    eng.upload_iq(x)
    rec = eng.acquire_grid_weak(1, 33, 2, 2, _prn(svs), dop)[0]
    ref = ws.vector_weak(x, fs, n, svs, dop, 2, 2)
    ws.check_weak(rec, x, fs, n, svs, dop, 2, 2, f"S={s}", ref)
    _check_found(rec, svs, dop, planted, f"S={s}")
    best = eng.acquire_grid_weak_best(1, 33, 2, 2, _prn(svs), dop)[0]
    want, _, _ = ws.best_folded(ref[0])
    for a in range(len(svs)):
        b = int(best["bin"][a])
        j, d = divmod(b, dop.size)
        if b != want[a]:
            assert ref[0][a].max() - ref[0][a, j, d] <= MAG_TOL * ref[0][a].max(), (s, a)
        r = rec[a, j, d]
        assert (best["peak"][a], best["code_phase"][a], best["doppler"][a]) == (r["peak"], r["argmax"], dop[d]), (s, a)
        assert best["strength"][a] == pytest.approx(o.strength_from_record(float(r["peak"]), r["sum"], r["count"], n), rel=1e-6)


# ---- coherent lengths, bit phases and segment counts -----------------------------------------------------------------
SHAPES = [(t, b, k) for t, b in ((2, 1), (2, 2), (10, 2), (20, 4), (20, 20), (1, 1)) for k in (1, 3)]


@pytest.mark.parametrize("t,b,k", SHAPES)
def test_shapes(engines, t, b, k):
    n, fs = rate(2)
    svs = [3, 11, 32]
    dop = np.array([-40000.0, -1250.0, 480.0, 500.0, 40000.0])
    planted = [(3, -1250.0, 0, 1.0, 0.1, 5, None), (11, 40000.0, 1023, 2.0, 0.1, 13, None),
               (32, 500.0, n - 1, 2.5, 0.1, 0, None)]
    m = (b - 1) * (t // b) + k * t
    x = ws.synth_weak_iq(950 + 10 * t + b + k, n, m, fs, planted)
    eng = engines(n)
    eng.upload_iq(x)
    rec = eng.acquire_grid_weak(1, m, t, b, _prn(svs), dop)[0]
    ws.check_weak(rec, x, fs, n, svs, dop, t, b, f"T={t} B={b} K={k}")
    if t * k >= 4:  # enough integration for every planted satellite to win its row
        _check_found(rec, svs, dop, planted, f"T={t} B={b} K={k}")


@pytest.mark.parametrize("s", [1, 2, 5, 16])
def test_one_phase_without_shifts_is_the_semicoherent_grid_byte_for_byte(engines, s):
    """B = 1 with every shift 0 (|f| * M * N well below f_L1 / 2), at T = 1, 2 and 3."""
    n, fs = rate(s)
    dop = np.array([-2000.0, -0.0, 733.25, 1500.0])
    x = o.synth_iq(960 + s, n, 6, fs, [(25, 1500.0, n - 1, 0.3, 0.2)])
    eng = engines(n)
    eng.upload_iq(x)
    for t, m in ((1, 3), (2, 6), (3, 6)):
        assert all(ws.shift(i, n, f) == 0 for i in range(m) for f in dop)
        weak = eng.acquire_grid_weak(2 if m == 3 else 1, m, t, 1, [24, 3, 0], dop)
        semi = eng.acquire_grid_semicoherent(2 if m == 3 else 1, m, t, [24, 3, 0], dop)
        assert weak.tobytes() == semi.tobytes(), (s, t)
        best = eng.acquire_grid_weak_best(1, m, t, 1, [24, 3, 0], dop)
        assert best.tobytes() == eng.acquire_grid_semicoherent_best(1, m, t, [24, 3, 0], dop).tobytes(), (s, t)


@pytest.mark.parametrize("s,m", [(2, 11), (5, 7)])
def test_three_blocks(engines, s, m):
    """Three blocks in one call, each its own window (the block stride is odd at S = 5, M = 7); T = 4, B = 4."""
    n, fs = rate(s)
    svs = [3, 7, 25]
    dop = np.array([-30000.0, -0.0, 1000.0])
    planted = [(7, 1000.0, 0, 0.4, 0.15, 2, None), (25, -30000.0, n - 1, 1.3, 0.15, 9, None)]
    x = np.concatenate([ws.synth_weak_iq(970 + 10 * s + b, n, m, fs, planted) for b in range(3)])
    eng = engines(n)
    eng.upload_iq(x)
    rec = eng.acquire_grid_weak(3, m, 4, 4, _prn(svs), dop)
    assert rec.shape == (3, 3, 4, 3)
    for b in range(3):
        xb = x[b * m * n:(b + 1) * m * n]
        ws.check_weak(rec[b], xb, fs, n, svs, dop, 4, 4, f"S={s} block {b}")


# ---- device calls and arguments --------------------------------------------------------------------------------------
def test_device_calls_write_every_record_and_nothing_else(engines):
    import torch

    n, fs = rate(2)
    prn, dop = np.array([24, 3, 0], np.int32), np.array([-1000.0, 0.0, 1500.0, 1750.0])
    x = o.synth_iq(88, n, 14, fs, [(25, 1500.0, 1234, 0.3, 0.1)])
    eng = engines(n)
    eng.upload_iq(x)
    host = eng.acquire_grid_weak(2, 7, 4, 4, prn, dop)
    host_best = eng.acquire_grid_weak_best(2, 7, 4, 4, prn, dop)
    for rows, want, call in ((2 * 3 * 4 * 4, host, eng.acquire_grid_weak_device),
                             (2 * 3, host_best, eng.acquire_grid_weak_best_device)):
        buf = torch.full(((rows + 1) * 32,), 0xFF, dtype=torch.uint8, device="cuda")
        call(2, 7, 4, 4, prn, dop, buf.data_ptr())
        torch.cuda.synchronize()
        got = buf.cpu().numpy()
        assert got[:rows * 32].tobytes() == want.tobytes()
        assert (got[rows * 32:] == 0xFF).all(), "guard row written"


def test_existing_grids_unchanged_around_a_weak_call(engines):
    n, fs = rate(2)
    dop = np.arange(-2000.0, 2001.0, 500.0)
    x = o.synth_iq(99, n, 10, fs, [(25, 1500.0, 777, 0.3, 0.1)])
    eng = engines(n)
    eng.upload_iq(x)
    before = eng.acquire_grid(1, 10, [24, 3], dop).tobytes()
    semi = eng.acquire_grid_semicoherent(1, 10, 5, [24, 3], dop).tobytes()
    eng.acquire_grid_weak(1, 9, 2, 2, [24, 3, 7], np.arange(-2000.0, 2001.0, 100.0))
    assert eng.acquire_grid(1, 10, [24, 3], dop).tobytes() == before
    assert eng.acquire_grid_semicoherent(1, 10, 5, [24, 3], dop).tobytes() == semi


@pytest.mark.parametrize("case", ["t0", "tneg", "b0", "bneg", "b_divides_not", "short", "partial", "partial_b1", "nan", "inf",
                                  "blocks0", "prn0", "dop0", "samples", "prn_range"])
def test_argument_errors_launch_nothing(engines, case):
    n, fs = rate(2)
    eng = engines(n)
    eng.upload_iq(o.synth_iq(3, n, 14, fs, []))
    args = dict(nb=1, m=14, t=8, b=4, prn=np.array([0, 3], np.int32), dop=np.array([0.0, 500.0]))  # K = 1
    args.update({"t0": dict(t=0, b=1), "tneg": dict(t=-4, b=1), "b0": dict(b=0), "bneg": dict(b=-2),
                 "b_divides_not": dict(b=3), "short": dict(m=13), "partial": dict(m=12, t=4), "partial_b1": dict(m=14, b=1),
                 "nan": dict(dop=np.array([0.0, np.nan])), "inf": dict(dop=np.array([-np.inf, 0.0])),
                 "blocks0": dict(nb=0), "prn0": dict(prn=np.zeros(0, np.int32)), "dop0": dict(dop=np.zeros(0)),
                 "samples": dict(nb=2), "prn_range": dict(prn=np.array([0, 32], np.int32))}[case])
    a = (args["nb"], args["m"], args["t"], args["b"], args["prn"], args["dop"])
    before = eng.launch_count
    for call in (eng.acquire_grid_weak, eng.acquire_grid_weak_best):
        with pytest.raises(ValueError) as err:
            call(*a)
        if case == "nan":
            assert "Doppler 1" in str(err.value)
    for call in (eng.acquire_grid_weak_device, eng.acquire_grid_weak_best_device):
        with pytest.raises(ValueError):
            call(*a, 1 << 40)
    assert eng.launch_count == before, case


# ---- bit edges and code Doppler on the device ------------------------------------------------------------------------
def test_bit_phase_case_on_the_device(engines):
    """The oracle's bit-phase case (tests/test_weak_cpu.py): B = 1 loses the satellite, B = 2 and 4 find its code phase
    and Doppler on the phase that starts at a bit edge, and the records match the oracle."""
    x = ws.bit_phase_iq()
    eng = engines(ws.BIT_N)
    eng.upload_iq(x)
    prn = _prn(ws.BIT_SVS)
    for b, m, want in ((1, 100, None), (2, 90, 1), (4, 95, 2)):
        rec = eng.acquire_grid_weak(1, m, 20, b, prn, ws.BIT_BINS)[0]
        ref = ws.vector_weak(x[:m * ws.BIT_N], ws.BIT_FS, ws.BIT_N, ws.BIT_SVS, ws.BIT_BINS, 20, b)
        ws.check_weak(rec, x[:m * ws.BIT_N], ws.BIT_FS, ws.BIT_N, ws.BIT_SVS, ws.BIT_BINS, 20, b, f"B={b}", ref)
        got = ws.search_decision(rec["peak"], rec["argmax"], ws.BIT_BINS)
        assert got == ws.search_decision(ref[0], ref[1], ws.BIT_BINS), b
        if want is None:
            assert got[0][1] != ws.BIT_DOPPLER
        else:
            assert got == ((want, ws.BIT_DOPPLER), ws.BIT_CODE_PHASE, True), b


def test_code_doppler_case_on_the_device(engines):
    """The oracle's code-Doppler case: 1 s at 2.046 Msps and 6 kHz.  The weak grid at T = 1 peaks on the planted code
    phase with at least 0.95 of the zero-Doppler control's peak; the non-coherent grid without realignment is at least
    2.4x lower and misses the code phase."""
    n, fs = rate(2)
    x = ws.synth_weak_iq(3, n, 1000, fs, [(9, 6000.0, 700, 0.2, 0.1, 0, [1.0] * 60)])
    c = ws.synth_weak_iq(3, n, 1000, fs, [(9, 0.0, 700, 0.2, 0.1, 0, [1.0] * 60)])
    eng = engines(n)
    eng.upload_iq(x)
    aligned = eng.acquire_grid_weak(1, 1000, 1, 1, [8], [6000.0])[0, 0, 0, 0]
    unaligned = eng.acquire_grid(1, 1000, [8], [6000.0])[0, 0, 0]
    eng.upload_iq(c)
    control = eng.acquire_grid_weak(1, 1000, 1, 1, [8], [0.0])[0, 0, 0, 0]
    ref = ws.integrate_weak(x, fs, n, 6000.0, o.replica(9, n), 1, 1)[0]
    assert abs(float(aligned["peak"]) - ref.max()) <= MAG_TOL * ref.max()
    assert int(aligned["argmax"]) == 700 == int(control["argmax"])
    assert aligned["peak"] >= 0.95 * control["peak"]
    assert unaligned["peak"] * 2.4 <= aligned["peak"] and int(unaligned["argmax"]) != 700


# ---- the detector ----------------------------------------------------------------------------------------------------
def _detector():
    from gypsum_b200.acquisition import GpsSatelliteDetector
    from gypsum_b200.gps_ca_prn_codes import generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite

    return GpsSatelliteDetector({sid: GpsSatellite(sid, code, 2) for sid, code in generate_replica_prn_signals().items()})


def test_search_weak_satellites_uploaded_and_ring_window(native_lib):
    """A strong satellite at 4500 Hz (on the default 25-Hz grid of T = 20) with random bits whose edges fall 6.6 ms into
    every 20: over a 100-ms window trimmed to 95 ms, its Doppler and code phase exactly, the bit phase starting at 5 ms,
    and the carrier phase of the probe over that phase's first segment, referred back to the window's first sample,
    within 0.02 rad of the planted one modulo pi.  Uploaded samples and a DeviceSampleRing window give the same results
    byte for byte, with the strength of the oracle's best folded bin."""
    from gypsum_b200.antenna_sample_provider import AntennaSampleChunk, DeviceSampleRing
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId

    n, fs = rate(2)
    f, tau, phi = 4500.0, 1234, 0.9
    x = ws.synth_weak_iq(123, n, 100, fs, [(14, f, tau, phi, 0.5, 6, None)])
    attrs = Attrs(fs, n)
    det = _detector()
    ids = [GpsSatelliteId(14), GpsSatelliteId(3)]
    up = det.search_weak_satellites(ids, x, attrs)
    ring = DeviceSampleRing(attrs, 100)
    try:
        for k in range(100):
            ring.append(AntennaSampleChunk(k * 1e-3, (k + 1) * 1e-3, x[k * n:(k + 1) * n]))
        dev = det.search_weak_satellites(ids, ring.window(), attrs)
    finally:
        ring.native.close()
    assert up == dev
    r = up[0]
    assert (r.doppler_shift, r.prn_phase_shift) == (f, tau)
    assert abs(np.angle(np.exp(2j * (r.carrier_wave_phase_shift - phi)))) / 2 <= 0.02
    assert len(up) == 2 and up[1].satellite_id == ids[1]
    bins = np.arange(-7000.0, 7012.5, 25.0)
    near = np.flatnonzero(np.abs(bins - f) <= 100.0)  # the oracle over the bins around the planted one
    ref = ws.vector_weak(x[:95 * n], fs, n, [14], bins[near], 20, 4)
    _, j, d = ws.best_folded(ref[0][0])
    assert j == 1 and bins[near][d] == f
    assert r.correlation_strength == pytest.approx(
        o.strength_from_record(ref[0][0, j, d], ref[2][0, j, d], ref[3][0, j, d], n), rel=1e-4)


def test_search_weak_satellites_argument_errors(native_lib):
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId

    n, fs = rate(2)
    attrs = Attrs(fs, n)
    det = _detector()
    x = o.synth_iq(5, n, 40, fs, [])
    for kw in (dict(coherent_ms=0), dict(coherent_ms=-1), dict(coherent_ms=2.5), dict(bit_phases=0), dict(bit_phases=3),
               dict(bit_phases=True), dict(doppler_step=0.0), dict(doppler_spread=np.nan), dict(doppler_spread=-1.0)):
        with pytest.raises(ValueError):
            det.search_weak_satellites([GpsSatelliteId(1)], x, attrs, **kw)
    with pytest.raises(ValueError, match="needs 35 ms"):
        det.search_weak_satellites([GpsSatelliteId(1)], x[:34 * n], attrs)
    assert len(det.search_weak_satellites([GpsSatelliteId(1)], x[:35 * n], attrs)) == 1
    assert det.search_weak_satellites([], x, attrs) == []
