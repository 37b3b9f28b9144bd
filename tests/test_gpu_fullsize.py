"""Every BASELINE.json configuration compared with the oracle CELL FOR CELL at its full size, through the C ABI.

Tolerances (DESIGN.md section 6): magnitudes / sums |gpu - ref| <= 1e-5 * max(ref); count exact; code phase exact unless the
ORACLE's own profile shows a near-tie at the two indices (proved per mismatch, never as a percentage).  The oracle grids
are spread over the host's cores (fork pool) so the file runs in well under a minute on the GPU box."""
import multiprocessing as mp

import numpy as np
import pytest

from acq_support import assert_records_equal, check_grid
from gpu_support import Attrs, EngineCache, all_chips, run_child
from oracle import gypsum_oracle as o
from oracle import tracker_oracle as t
from tracker_support import assert_follows_reference, oracle_row

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines(native_lib):
    cache = EngineCache()
    yield cache
    cache.close()


PLANTED = [(3, -3000.0, 5, 1.0, 0.3), (11, 4500.0, 1234, 2.0, 0.3), (25, 1500.0, 777, 0.3, 0.3), (32, -9500.0, 2045, 2.5, 0.3)]
SVS = list(range(1, 33))


def test_config2_all_1312_cells(engines):
    """32 PRN x 41 Doppler x 1 ms @ 2.046 Msps: every record of the grid, by every entry point that produces it."""
    n, fs = 2046, 2046000
    dop = np.arange(-10000.0, 10001.0, 500.0)
    x = o.synth_iq(2, n, 1, fs, PLANTED)
    eng = engines(n)
    eng.upload_iq(x)
    rec = eng.acquire_grid(1, 1, np.arange(32), dop)[0]
    check_grid(rec, x, fs, n, SVS, dop, "acquire_grid")
    rec_h = eng.acquire_grid_host(x, 1, 1, np.arange(32), dop)[0]  # eager call of the shape ...
    rec_g = eng.acquire_grid_host(x, 1, 1, np.arange(32), dop)[0]  # ... captured into a graph ...
    rec_r = eng.acquire_grid_host(x, 1, 1, np.arange(32), dop)[0]  # ... replayed
    for call, other in zip(("eager", "captured", "replayed"), (rec_h, rec_g, rec_r)):
        assert_records_equal(other, rec, call)
    # the replayed graph reads the grid's axes and the replica spectra from device buffers other calls reuse: a list-mode call
    # with other Dopplers, a different grid, and a re-loaded replica table in between must not leak into the next replay
    eng.acquire_cells([3, 4], [123.0, -456.0], 1)
    eng.acquire_grid(1, 1, [5], [777.0])
    assert_records_equal(eng.acquire_grid_host(x, 1, 1, np.arange(32), dop)[0], rec, "again")
    chips = all_chips()
    eng.set_replicas(chips[::-1].copy())  # row a now holds SV 32 - a
    assert_records_equal(eng.acquire_grid_host(x, 1, 1, np.arange(32), dop)[0], rec[::-1], "flipped")
    eng.set_replicas(chips)
    eng.upload_iq(x)
    best = eng.acquire_grid_best(1, 1, np.arange(32), dop)[0]
    for a in range(32):  # acquisition.py:179-189 per PRN row
        b = int(np.argmax(rec["peak"][a]))
        assert (best["bin"][a], best["doppler"][a], best["code_phase"][a], best["peak"][a]) == (b, dop[b], rec["argmax"][a, b], rec["peak"][a, b])
    for sv, f, tau, _, _ in PLANTED:
        assert (best["doppler"][sv - 1], best["code_phase"][sv - 1]) == (f, tau) and best["strength"][sv - 1] > 8


def test_config3_all_cells_10ms_4092(engines):
    """32 PRN x 41 Doppler x 10 ms non-coherent @ 4.092 Msps."""
    n, fs = 4092, 4092000
    dop = np.arange(-10000.0, 10001.0, 500.0)
    planted = [(3, -3000.0, 5, 1.0, 0.1), (11, 4500.0, 2500, 2.0, 0.1), (25, 1500.0, 4091, 0.3, 0.08), (32, -9500.0, 2045, 2.5, 0.1)]
    x = o.synth_iq(3, n, 10, fs, planted)
    eng = engines(n)
    eng.upload_iq(x)
    rec = eng.acquire_grid(1, 10, np.arange(32), dop)[0]
    check_grid(rec, x, fs, n, SVS, dop, "config 3")
    for sv, f, tau, _, _ in planted:
        b = int(np.argmax(rec["peak"][sv - 1]))
        assert dop[b] == f and rec["argmax"][sv - 1, b] == tau


def test_config5_all_cells_two_blocks_16368(engines):
    """32 PRN x 81 Doppler @ 16.368 Msps, two independent 1-ms blocks in one call (the shape the 8-GPU job shards)."""
    n, fs = 16368, 16368000
    dop = np.arange(-10000.0, 10001.0, 250.0)
    assert len(dop) == 81
    planted = [(3, -3000.0, 5, 1.0, 0.12), (11, 4500.0, 12345, 2.0, 0.12), (25, 1500.0, 16367, 0.3, 0.1)]
    x = np.concatenate([o.synth_iq(50 + b, n, 1, fs, planted) for b in range(2)])
    eng = engines(n)
    eng.upload_iq(x)
    rec = eng.acquire_grid(2, 1, np.arange(32), dop)
    for b in range(2):
        check_grid(rec[b], x[b * n:(b + 1) * n], fs, n, SVS, dop, f"config 5 block {b}")


def test_config4_four_channels_ten_seconds_with_bits(engines):
    """Config 4 on a stated subset the CPU can afford: 4 channels x 10 s of ONE shared stream through TrackerBank (one
    launch) + the device bit integrator, against TrackerOracle per channel + the host integrator restatement (itself
    pinned to events recorded from the live reference).  Symbols / code phase exact bar per-millisecond proofs."""
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.navigation_bit_integrator import NavigationBitIntegrator
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import BitValue, EmittedPseudosymbol, NavigationBitPseudosymbol, TrackerBank

    n, fs, n_ms = 2046, 2046000, 10000
    chans = [(25, 1500.3, 0.0, 777, 0.3, 0.004), (7, -2212.7, 0.2, 100, 1.0, 0.005), (31, 3000.2, -0.3, 2045, 2.0, 0.004),
             (12, 640.4, 0.0, 1501, 0.7, 0.006)]
    inits = [(1500.0, 0.0, 777), (-2210.0, 0.5, 100), (3000.0, 0.0, 2045), (640.0, 0.0, 1501)]
    # every channel tracks its own satellite inside the SAME stream (sum of the four signals + one noise realisation)
    x = t.synth_tracking_iq(77, n, n_ms, fs, chans)
    codes = generate_replica_prn_signals()
    sats = {c[0]: GpsSatellite(GpsSatelliteId(c[0]), codes[GpsSatelliteId(c[0])], 2) for c in chans}
    bank = TrackerBank([(sats[c[0]], i[0], i[1], i[2]) for c, i in zip(chans, inits)], Attrs(fs, n))
    tt = np.array([t.chunk_times(k, fs, n) for k in range(n_ms)])
    rec = bank.process(x, tt[:, 0])
    bits = bank.integrate_bits(tt[:, 0], tt[:, 1])

    # oracle: one process per channel, each on the same stream
    with mp.get_context("fork").Pool(4) as pool:
        want = pool.map(oracle_channel_entry, [(x, chans[ci], inits[ci], n_ms) for ci in range(4)])
    for ci in range(4):
        w, g = want[ci], rec[ci]
        assert_follows_reference(g, w)
        # bits: the host integrator on the ORACLE's pseudosymbols vs the device integrator on the device's records
        integ = NavigationBitIntegrator(chans[ci][0])
        code = {BitValue.ONE: 1, BitValue.ZERO: 0, BitValue.UNKNOWN: -1}
        ref_bits = []
        for k in range(n_ms):
            ps = EmittedPseudosymbol(w[k, 9], w[k, 10], NavigationBitPseudosymbol.from_val(int(w[k, 3])), 0)
            ref_bits += [(k, e.receiver_timestamp, e.trailing_edge_receiver_timestamp, code[e.bit_value])
                         for e in integ.process_pseudosymbol(tt[k, 0], ps)]
        got_bits = [(int(e["ms_index"]), float(e["receiver_timestamp"]), float(e["trailing_edge_receiver_timestamp"]),
                     int(e["bit_value"])) for e in bits[ci]]
        if np.array_equal(g["symbol"], w[:, 3].astype(int)) and np.array_equal(g["code_phase"], w[:, 8].astype(int)):
            assert got_bits == ref_bits, ci  # same symbols and code phases in => same bits and edges out, event for event
        assert len(got_bits) >= 480  # 10 s at 50 bit/s minus the synchronisation backlog


def oracle_channel_entry(args):
    x, ch, init, n_ms = args
    n, fs = 2046, 2046000
    tr = t.TrackerOracle(ch[0], init[0], init[1], init[2], fs, n)
    rows = []
    for k in range(n_ms):
        a, b = t.chunk_times(k, fs, n)
        rows.append(oracle_row(tr, tr.step(x[k * n:(k + 1) * n], a, b)))
    return np.array(rows)


_WINDOW_CHILD = r"""
import os, sys
import numpy as np
sys.path[:0] = [sys.argv[1], sys.argv[1] + "/tests"]
os.environ.update(GB200_L2_WINDOW_MB=sys.argv[2], GB200_L2_WINDOW_MIN_GROUPS="0")
from gpu_support import make_engine
n, nb = int(sys.argv[3]), int(sys.argv[4])
e = make_engine(n * 1000, n)
e.upload_iq(np.load(sys.argv[5]))
rec = e.acquire_grid(nb, 1, np.arange(32, dtype=np.int32), np.arange(-10000.0, 10001.0, 500.0))
np.save(sys.argv[6], rec.view(np.uint8))
e.close()
"""


@pytest.mark.parametrize("n, nb", [(2046, 20), (16368, 3)])
def test_l2_windows_leave_every_record_unchanged(engines, tmp_path, n, nb):
    """The one-warp kernel walks batches larger than L2 in windows of units (group order window / PRN / chunk, extra groups going
    round the CTAs).  That only reorders independent cells: with windows forced onto a small batch (an engine
    created in a child process) every record is byte-identical to the single-window launch's, also with a ragged last window."""
    rng = np.random.default_rng(n + nb)
    x = (rng.standard_normal(2 * n * nb).astype(np.float32)).view(np.complex64)
    x[:n] += o.synth_iq(0, n, 1, n * 1000, [(25, 1500.0, 777, 0.3, 0.3)], sigma=0.0)
    e = engines(n)
    e.upload_iq(x)
    ref = e.acquire_grid(nb, 1, np.arange(32, dtype=np.int32), np.arange(-10000.0, 10001.0, 500.0))
    assert int(ref["argmax"][0, 24, 23]) == 777
    np.save(tmp_path / "x.npy", x)
    for mb in ("1", "3"):
        run_child(_WINDOW_CHILD, mb, n, nb, tmp_path / "x.npy", tmp_path / f"r{mb}.npy")
        got = np.load(tmp_path / f"r{mb}.npy")
        assert np.array_equal(got, ref.view(np.uint8)), mb
