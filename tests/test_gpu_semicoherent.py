"""Semi-coherent grids (gb200_acquire_grid_semicoherent*, GpsSatelliteDetector.acquire_weak_satellites) against the float64
oracle of tests/semicoherent_support.py, with the tolerances of DESIGN.md section 6: magnitudes and sums within 1e-5 of the
grid's largest, count exact, strength 1e-4 relative, argmax and best bin exact unless the oracle's own float64 profile ties
within the tolerance (proved per mismatch).

The segment sums run in k_segment_spectra<S>, one instantiation per rate, whose first launches happen in a child process;
the correlate launch is the non-coherent one over K = M / T segment spectra per unit."""
import numpy as np
import pytest

import semicoherent_support as ss
from acq_support import MAG_TOL, mid_branch_lag, rate, vector_grid
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
    x = o.synth_iq(s, n, 4, fs, [(25, 1500.0, n - 1, 0.3, 0.3)])
    eng = make_engine(fs, n)
    eng.upload_iq(x)
    dop = np.arange(-2000.0, 2001.0, 250.0)
    for t in (2, 4):
        g = eng.acquire_grid_semicoherent(1, 4, t, [24, 3], dop)[0]
        assert int(g["argmax"][0, 14]) == n - 1 and int(np.argmax(g["peak"][0])) == 14, (s, t)
    eng.close()
print("segments ok")
"""


def test_first_run_of_the_segment_kernels_in_a_child_process(native_lib):
    """Runs first, in its own process, so that a fault in a never-exercised kernel cannot disturb the CUDA context of
    the tests below."""
    run_child(_FIRST_RUN_SCRIPT, ok="segments ok")


@pytest.fixture(scope="module")
def engines(native_lib):
    cache = EngineCache()
    yield cache
    cache.close()


def _planted(s, n):
    """Code phases 0, n - 1 and mid-code on branch s // 2, at a fractional and two whole Dopplers."""
    return [(3, -1250.0, 0, 1.0, 0.12), (11, 1737.5, mid_branch_lag(s), 2.0, 0.12), (32, 500.0, n - 1, 2.5, 0.12)]


def _check_found(rec, svs, dop, planted, what):
    for sv, f, tau, _, _ in planted:
        a = svs.index(sv)
        b = int(np.argmax(rec["peak"][a]))
        assert abs(dop[b] - f) <= 125.0 and int(rec["argmax"][a, b]) == tau, (what, sv)


# ---- every rate ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s", RATES)
def test_every_rate(engines, s):
    """T = 2, K = 2 at every rate, on a grid with fractional, -0.0 and +-50 kHz Dopplers; the best records equal the
    oracle's first bin with the largest peak."""
    n, fs = rate(s)
    svs = [3, 11, 19, 32]
    dop = np.array([-50000.0, -1250.0, -0.0, 500.0, 1737.5, 1862.5, 50000.0])
    planted = _planted(s, n)
    x = o.synth_iq(500 + s, n, 4, fs, planted)
    eng = engines(n)
    eng.upload_iq(x)
    rec = eng.acquire_grid_semicoherent(1, 4, 2, [sv - 1 for sv in svs], dop)[0]
    ref = ss.vector_semicoherent(x, fs, n, svs, dop, 2)
    ss.check_semicoherent(rec, x, fs, n, svs, dop, 2, f"S={s}", ref)
    _check_found(rec, svs, dop, planted, f"S={s}")
    best = eng.acquire_grid_semicoherent_best(1, 4, 2, [sv - 1 for sv in svs], dop)[0]
    want = ss.best_bins(ref[0])
    for a in range(len(svs)):
        b = int(best["bin"][a])
        if b != want[a]:
            assert ref[0][a].max() - ref[0][a, b] <= MAG_TOL * ref[0][a].max(), (s, a)
        r = rec[a, b]
        assert (best["peak"][a], best["code_phase"][a], best["doppler"][a]) == (r["peak"], r["argmax"], dop[b]), (s, a)
        assert best["strength"][a] == pytest.approx(o.strength_from_record(float(r["peak"]), r["sum"], r["count"], n), rel=1e-6)


# ---- segment lengths and counts --------------------------------------------------------------------------------------
SHAPES = [(t, k) for t in (2, 5, 10, 20) for k in (1, 2, 3)]


@pytest.mark.parametrize("t,k", SHAPES)
def test_segment_shapes(engines, t, k):
    n, fs = rate(2)
    svs = [3, 11, 32]
    dop = np.array([-1250.0, 480.0, 500.0, 1737.5])
    planted = [(3, -1250.0, 0, 1.0, 0.1), (11, 1737.5, 1023, 2.0, 0.1), (32, 500.0, n - 1, 2.5, 0.1)]
    x = o.synth_iq(600 + 10 * t + k, n, t * k, fs, planted)
    eng = engines(n)
    eng.upload_iq(x)
    rec = eng.acquire_grid_semicoherent(1, t * k, t, [sv - 1 for sv in svs], dop)[0]
    ss.check_semicoherent(rec, x, fs, n, svs, dop, t, f"T={t} K={k}")
    _check_found(rec, svs, dop, planted, f"T={t} K={k}")


@pytest.mark.parametrize("s", [2, 5])
def test_one_segment_is_the_coherent_grid(engines, s):
    """T = M: the records' peaks, sums and code phases agree with the coherent grid's magnitudes."""
    from gypsum_b200 import _native

    n, fs = rate(s)
    svs, dop = [3, 11, 32], np.array([-1250.0, 500.0, 1737.5])
    x = o.synth_iq(650 + s, n, 6, fs, _planted(s, n))
    eng = engines(n)
    eng.upload_iq(x)
    semi = eng.acquire_grid_semicoherent(1, 6, 6, [sv - 1 for sv in svs], dop)[0]
    coh = eng.acquire_grid(1, 6, [sv - 1 for sv in svs], dop, _native.COHERENT)[0]
    ss.check_semicoherent(semi, x, fs, n, svs, dop, 6, f"S={s} T=M")
    assert np.abs(semi["peak"] - coh["peak"]).max() <= MAG_TOL * coh["peak"].max()
    assert np.abs(semi["sum"] - coh["sum"]).max() <= MAG_TOL * coh["sum"].max()
    assert np.array_equal(semi["argmax"], coh["argmax"])


@pytest.mark.parametrize("s", [1, 2, 5, 16])
def test_one_ms_segments_are_the_non_coherent_grid_byte_for_byte(engines, s):
    n, fs = rate(s)
    dop = np.array([-2000.0, -0.0, 733.25, 1500.0])
    x = o.synth_iq(700 + s, n, 3, fs, [(25, 1500.0, n - 1, 0.3, 0.2)])
    eng = engines(n)
    eng.upload_iq(x)
    for m in (1, 3):
        semi = eng.acquire_grid_semicoherent(1, m, 1, [24, 3, 0], dop)
        assert semi.tobytes() == eng.acquire_grid(1, m, [24, 3, 0], dop).tobytes(), (s, m)


# ---- blocks ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("s,m,t", [(2, 4, 2), (5, 3, 3), (5, 9, 3), (4, 6, 2)])
def test_three_blocks(engines, s, m, t):
    """Three blocks in one call, each its own window; the block stride M * N is odd at S = 5 with M = 3 and 9.  At S = 4
    the planted code phases sit on every polyphase branch."""
    n, fs = rate(s)
    svs = [3, 7, 11, 19, 25, 32]
    dop = np.array([-2000.0, -0.0, 1000.0, 1500.0])
    planted = [(7, 1000.0, 0, 0.4, 0.12), (25, -2000.0, n - 1, 1.3, 0.12)]
    planted += [(sv, 1500.0, 100 * s * (r + 1) + r, 0.2 * r, 0.12) for r, sv in zip(range(s), (3, 11, 32, 19))]
    x = np.concatenate([o.synth_iq(800 + 10 * s + b, n, m, fs, planted) for b in range(3)])
    eng = engines(n)
    eng.upload_iq(x)
    rec = eng.acquire_grid_semicoherent(3, m, t, [sv - 1 for sv in svs], dop)
    for b in range(3):
        xb = x[b * m * n:(b + 1) * m * n]
        ss.check_semicoherent(rec[b], xb, fs, n, svs, dop, t, f"S={s} block {b}")
        _check_found(rec[b], svs, dop, planted, f"S={s} block {b}")


def test_bit_edge_inside_a_segment(engines):
    """Data bits every 20 ms and 15-ms segments: the second segment holds a bit edge.  The device still equals the
    oracle, which loses part of that segment the same way."""
    n, fs = rate(2)
    svs, dop = [9, 14], np.arange(-300.0, 301.0, 50.0)
    x = o.synth_iq(41, n, 30, fs, [(9, 100.0, 777, 0.7, 0.05)], nav_bits=True)
    eng = engines(n)
    eng.upload_iq(x)
    rec = eng.acquire_grid_semicoherent(1, 30, 15, [8, 13], dop)[0]
    ss.check_semicoherent(rec, x, fs, n, svs, dop, 15, "bit edge")


# ---- plan edges ------------------------------------------------------------------------------------------------------
_BUDGET_SCRIPT = r"""
import os, sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
from gpu_support import make_engine
from oracle import gypsum_oracle as o

n, fs = 1023, 1023000
x = o.synth_iq(5, n, 5 * 4, fs, [(25, 1500.0, 1000, 0.3, 0.2)])
dop = np.arange(-6375.0, 6376.0, 50.0)  # 256 bins: 8 MB of spectra per block at K = 2, S = 1
prn = list(range(32))
ref = make_engine(fs, n)
ref.upload_iq(x)
want = ref.acquire_grid_semicoherent(5, 4, 2, prn, dop)
want_best = ref.acquire_grid_semicoherent_best(5, 4, 2, prn, dop)
ref.close()
os.environ["GB200_SPEC_BUDGET_MB"] = "17"  # two blocks per batch: 2, 2, 1
os.environ["GB200_L2_WINDOW_MB"] = "4"     # four L2 windows in a full batch
eng = make_engine(fs, n)
eng.upload_iq(x)
eng.enable_kernel_timing(True)
got = eng.acquire_grid_semicoherent(5, 4, 2, prn, dop)
assert eng.kernel_timing(0)[1] == 3 and eng.kernel_timing(1)[1] == 3, "three batches"
assert got.tobytes() == want.tobytes(), "ragged batches changed the records"
assert eng.acquire_grid_semicoherent_best(5, 4, 2, prn, dop).tobytes() == want_best.tobytes()
eng.close()
print("budget ok")
"""


def test_ragged_batches_and_l2_windows_in_a_child_process(native_lib):
    """A scratch budget of two blocks and 4-MB L2 windows (read by gb200_create, so in a child): five blocks run in
    batches of 2, 2 and 1 and give the same bytes as one batch.  At S = 1 every launch keeps one warp per cell."""
    run_child(_BUDGET_SCRIPT, ok="budget ok")


@pytest.mark.parametrize("below", [False, True])
def test_at_the_rsplit_threshold(engines, below):
    """pick_rsplit keeps one warp per cell from 8 * SMs * 8 cells on; one cell fewer splits each cell's two polyphase
    branches over two warps (S = 2).  Both sides against the oracle."""
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n, fs = rate(2)
    d = 2 * sms - (1 if below else 0)  # 32 PRNs x d bins = 8 * sms * 8 cells, or 32 fewer
    dop = -3000.0 + 25.0 * np.arange(d)
    x = o.synth_iq(77, n, 4, fs, [(5, 100.0, 1500, 0.3, 0.1)])
    eng = engines(n)
    eng.upload_iq(x)
    svs = list(range(1, 33))
    rec = eng.acquire_grid_semicoherent(1, 4, 2, [sv - 1 for sv in svs], dop)[0]
    ss.check_semicoherent(rec, x, fs, n, svs, dop, 2, f"rsplit below={below}")


# ---- device calls, neighbours and degenerate input -------------------------------------------------------------------
def test_device_calls_write_every_record_and_nothing_else(engines):
    import torch

    from gypsum_b200 import _native

    n, fs = rate(2)
    prn, dop = np.array([24, 3, 0], np.int32), np.array([-1000.0, 0.0, 1500.0, 1750.0])
    x = o.synth_iq(88, n, 8, fs, [(25, 1500.0, 1234, 0.3, 0.1)])
    eng = engines(n)
    eng.upload_iq(x)
    host = eng.acquire_grid_semicoherent(2, 4, 2, prn, dop)
    host_best = eng.acquire_grid_semicoherent_best(2, 4, 2, prn, dop)
    for rows, want, call, itemsize in ((2 * 3 * 4, host, eng.acquire_grid_semicoherent_device, 32),
                                        (2 * 3, host_best, eng.acquire_grid_semicoherent_best_device, 32)):
        buf = torch.full(((rows + 1) * itemsize,), 0xFF, dtype=torch.uint8, device="cuda")
        call(2, 4, 2, prn, dop, buf.data_ptr())
        torch.cuda.synchronize()
        got = buf.cpu().numpy()
        assert got[:rows * itemsize].tobytes() == want.tobytes()
        assert (got[rows * itemsize:] == 0xFF).all(), "guard row written"
    assert _native.BEST_DTYPE.itemsize == _native.RECORD_DTYPE.itemsize == 32


def test_existing_grid_unchanged_around_a_semicoherent_call(engines):
    n, fs = rate(2)
    dop = np.arange(-2000.0, 2001.0, 500.0)
    x = o.synth_iq(99, n, 10, fs, [(25, 1500.0, 777, 0.3, 0.1)])
    eng = engines(n)
    eng.upload_iq(x)
    before = eng.acquire_grid(1, 10, [24, 3], dop).tobytes()
    eng.acquire_grid_semicoherent(1, 10, 5, [24, 3, 7], np.arange(-2000.0, 2001.0, 100.0))
    assert eng.acquire_grid(1, 10, [24, 3], dop).tobytes() == before


def test_all_zero_input(engines):
    n, fs = rate(2)
    eng = engines(n)
    eng.upload_iq(np.zeros(4 * n, np.complex64))
    best = eng.acquire_grid_semicoherent_best(1, 4, 2, [0, 5], np.array([-500.0, 0.0, 500.0]))[0]
    assert (best["bin"] == 0).all() and (best["code_phase"] == 0).all() and np.isnan(best["strength"]).all()


@pytest.mark.parametrize("case", ["t0", "tneg", "partial", "partial_big", "nan", "inf", "blocks0", "prn0", "dop0",
                                  "samples", "prn_range"])
def test_argument_errors_launch_nothing(engines, case):
    n, fs = rate(2)
    eng = engines(n)
    eng.upload_iq(o.synth_iq(3, n, 6, fs, []))
    args = dict(nb=1, m=6, t=2, prn=np.array([0, 3], np.int32), dop=np.array([0.0, 500.0]))
    args.update({"t0": dict(t=0), "tneg": dict(t=-2), "partial": dict(t=4), "partial_big": dict(t=7),
                 "nan": dict(dop=np.array([0.0, np.nan])), "inf": dict(dop=np.array([-np.inf, 0.0])), "blocks0": dict(nb=0),
                 "prn0": dict(prn=np.zeros(0, np.int32)), "dop0": dict(dop=np.zeros(0)), "samples": dict(nb=2),
                 "prn_range": dict(prn=np.array([0, 32], np.int32))}[case])
    before = eng.launch_count
    for call in (eng.acquire_grid_semicoherent, eng.acquire_grid_semicoherent_best):
        with pytest.raises(ValueError) as err:
            call(args["nb"], args["m"], args["t"], args["prn"], args["dop"])
        if case == "nan":
            assert "Doppler 1" in str(err.value)
    for call in (eng.acquire_grid_semicoherent_device, eng.acquire_grid_semicoherent_best_device):
        with pytest.raises(ValueError):
            call(args["nb"], args["m"], args["t"], args["prn"], args["dop"], 1 << 40)
    assert eng.launch_count == before, case


# ---- sensitivity and the detector ------------------------------------------------------------------------------------
def test_sensitivity_on_the_device(engines):
    """The satellite of the oracle's sensitivity case: the device's 20-ms non-coherent grid misses it as the oracle's
    does, and its T = 10, K = 2 grid finds the planted code phase within one bin of the Doppler, as the oracle's does."""
    x = ss.sensitivity_iq()
    eng = engines(ss.SENS_N)
    eng.upload_iq(x)
    prn = [sv - 1 for sv in ss.SENS_SVS]
    nc = eng.acquire_grid(1, 20, prn, ss.SENS_BINS)[0]
    nc_ref = vector_grid(x, ss.SENS_FS, ss.SENS_N, ss.SENS_SVS, ss.SENS_BINS)
    assert ss.search_decision(nc["peak"], nc["argmax"]) == ss.search_decision(nc_ref[0], nc_ref[1])
    semi = eng.acquire_grid_semicoherent(1, 20, 10, prn, ss.SENS_BINS)[0]
    ref = ss.vector_semicoherent(x, ss.SENS_FS, ss.SENS_N, ss.SENS_SVS, ss.SENS_BINS, 10)
    ss.check_semicoherent(semi, x, ss.SENS_FS, ss.SENS_N, ss.SENS_SVS, ss.SENS_BINS, 10, "sensitivity", ref)
    b, tau, above = ss.search_decision(semi["peak"], semi["argmax"])
    assert (b, tau, above) == ss.search_decision(ref[0], ref[1])
    assert tau == ss.SENS_CODE_PHASE and above and abs(ss.SENS_BINS[b] - ss.SENS_DOPPLER) <= 50.0


def _detector():
    from gypsum_b200.acquisition import GpsSatelliteDetector
    from gypsum_b200.gps_ca_prn_codes import generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite

    return GpsSatelliteDetector({sid: GpsSatellite(sid, code, 2) for sid, code in generate_replica_prn_signals().items()})


def test_acquire_weak_satellites_uploaded_and_ring_window(native_lib):
    """A strong satellite on a bin of the default 100-Hz grid (T = 5): its Doppler and code phase exactly, and the
    carrier phase of the coherent probe within 1e-3 rad of the planted one; uploaded samples and a DeviceSampleRing
    window give the same results byte for byte, with the strength of the oracle's best bin."""
    from gypsum_b200.antenna_sample_provider import AntennaSampleChunk, DeviceSampleRing
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId

    n, fs = rate(2)
    f, tau, phi = 1300.0, 1234, 0.9
    x = o.synth_iq(123, n, 10, fs, [(14, f, tau, phi, 20.0)])
    attrs = Attrs(fs, n)
    det = _detector()
    ids = [GpsSatelliteId(14), GpsSatelliteId(3)]
    up = det.acquire_weak_satellites(ids, x, attrs, 5)
    ring = DeviceSampleRing(attrs, 10)
    try:
        for k in range(10):
            ring.append(AntennaSampleChunk(k * 1e-3, (k + 1) * 1e-3, x[k * n:(k + 1) * n]))
        dev = det.acquire_weak_satellites(ids, ring.window(), attrs, 5)
    finally:
        ring.native.close()
    assert up == dev
    r = up[0]
    assert (r.doppler_shift, r.prn_phase_shift) == (f, tau)
    assert abs(np.angle(np.exp(1j * (r.carrier_wave_phase_shift - phi)))) <= 1e-3
    assert len(up) == 2 and up[1].satellite_id == ids[1]
    ref = ss.vector_semicoherent(x, fs, n, [14, 3], np.arange(-7000.0, 7050.0, 100.0), 5)
    assert r.correlation_strength == pytest.approx(o.strength_from_record(ref[0][0].max(), ref[2][0][ref[0][0].argmax()],
                                                                         ref[3][0][ref[0][0].argmax()], n), rel=1e-4)


def test_acquire_weak_satellites_argument_errors(native_lib):
    n, fs = rate(2)
    attrs = Attrs(fs, n)
    det = _detector()
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId

    x = o.synth_iq(5, n, 10, fs, [])
    for kw in (dict(coherent_ms=0), dict(coherent_ms=-1), dict(coherent_ms=3), dict(coherent_ms=2.5),
               dict(coherent_ms=5, doppler_step=0.0), dict(coherent_ms=5, doppler_spread=np.nan),
               dict(coherent_ms=5, doppler_spread=-1.0)):
        with pytest.raises(ValueError):
            det.acquire_weak_satellites([GpsSatelliteId(1)], x, attrs, **kw)
    assert det.acquire_weak_satellites([], x, attrs, 5) == []
