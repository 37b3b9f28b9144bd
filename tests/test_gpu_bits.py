"""GPU parity of the navigation-bit integration kernel (bits.cu through gb200_tracker_integrate_bits) against event
streams recorded from the live reference integrator (tests/golden/bit_integrator.npz), and end to end behind the
tracking kernel against the host mirror fed with the same records."""
import os

import numpy as np
import pytest

from gpu_support import make_engine
from oracle import tracker_oracle as t

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
N, FS = 2046, 2046000


@pytest.fixture(scope="module")
def engine(native_lib):
    e = make_engine(FS, N)
    yield e
    e.close()


def _records_on_device(symbols_by_channel):
    """TRACK_DTYPE records carrying the given symbols (code phase 0) in device memory."""
    import torch

    from gypsum_b200._native import TRACK_DTYPE

    rec = np.zeros((len(symbols_by_channel), len(symbols_by_channel[0])), dtype=TRACK_DTYPE)
    for c, s in enumerate(symbols_by_channel):
        rec["symbol"][c] = s
    return torch.from_numpy(rec.view(np.uint8).reshape(rec.shape[0], -1)).cuda()


@pytest.mark.parametrize("case,chunk", [("long", 6300), ("long", 997), ("synth", 45000), ("synth", 4001)])
def test_bit_stream_identical_to_reference(engine, case, chunk):
    from gypsum_b200 import _native

    z = np.load(os.path.join(GOLDEN, "bit_integrator.npz"))
    sym, t0, t1 = z[f"{case}_symbols"].astype(np.int32), z[f"{case}_starts"], z[f"{case}_ends"]
    # channel 0: the recorded stream; channel 1: the same stream negated (same timing, complemented bits);
    # channel 2: loses lock 1234 ms in
    trk = _native.Tracker(engine, [0, 1, 2], [0.0] * 3, [0.0] * 3, [0] * 3)
    rows = [[], [], []]
    for a in range(0, sym.size, chunk):
        b = min(sym.size, a + chunk)
        dev = _records_on_device([sym[a:b], -sym[a:b], sym[a:b]])
        if a <= 1234 < b:
            import torch

            from gypsum_b200._native import TRACK_DTYPE
            host = np.zeros((3, b - a), dtype=TRACK_DTYPE)
            host[:] = dev.cpu().numpy().view(TRACK_DTYPE).reshape(3, b - a)
            host["lost"][2, 1234 - a] = 1
            host["lost"][2, 1234 - a + 1:] = 2
            dev = torch.from_numpy(host.view(np.uint8).reshape(3, -1)).cuda()
        ev = trk.integrate_bits(b - a, t0[a:b], t1[a:b], dev.data_ptr())
        for c in range(3):
            rows[c] += [[a + e["ms_index"], e["receiver_timestamp"], e["trailing_edge_receiver_timestamp"], e["bit_value"]]
                        for e in ev[c]]
    want = z[f"{case}_events"]
    got = np.array(rows[0], dtype=np.float64)
    assert np.array_equal(got, want)
    neg = np.array(rows[1], dtype=np.float64)
    flipped = want.copy()
    known = want[:, 3] >= 0
    flipped[known, 3] = 1 - want[known, 3]
    # a sum of exactly 0 is ZERO-then-UNKNOWN either way (:149-161), so only resolved bits complement
    assert np.array_equal(neg, flipped)
    lost = np.array(rows[2], dtype=np.float64)
    assert np.array_equal(lost, want[want[:, 0] < 1234])
    st = trk.bit_state(0)
    final = z[f"{case}_final"]
    assert [st["emitted_bit_count"], st["failed_bit_count"], st["processed_pseudosymbol_count"], st["slide"],
            -1 if st["determined_bit_phase"] is None else st["determined_bit_phase"],
            -1 if st["previous_bit_phase_decision"] is None else st["previous_bit_phase_decision"],
            st["pseudosymbol_cursor_within_queue"]] == list(final)
    assert trk.bit_state(2)["stopped"] == 1 and trk.bit_state(2)["processed_pseudosymbol_count"] == 1234
    trk.close()


def test_bits_behind_the_tracking_kernel(engine):
    """Track the recorded 6.3 s signal, integrate its records where the tracking kernel left them, and compare with
    the host mirror of the reference integrator fed from the same records (timestamps include the code-phase delay of
    tracker.py:319)."""
    from gypsum_b200 import _native
    from gypsum_b200.navigation_bit_integrator import NavigationBitIntegrator
    from gypsum_b200.tracker import BitValue, _pseudosymbol

    z = np.load(os.path.join(GOLDEN, "tracker_long.npz"))
    ch = z["channel"]
    ch = (int(ch[0]), ch[1], ch[2], int(ch[3]), ch[4], ch[5])
    n_ms = int(z["n_ms"])
    x = t.synth_tracking_iq(int(z["seed"]), N, n_ms, FS, [ch], float(z["sigma"]))
    init = z["init"]
    trk = _native.Tracker(engine, [ch[0] - 1], [init[0]], [init[1]], [int(init[2])])
    engine.upload_iq(x)
    tt = np.array([t.chunk_times(k, FS, N) for k in range(n_ms)])
    rec = trk.process(n_ms, tt[:, 0])
    ev = trk.integrate_bits(n_ms, tt[:, 0], tt[:, 1])[0]
    integ = NavigationBitIntegrator(ch[0])
    code = {BitValue.ONE: 1, BitValue.ZERO: 0, BitValue.UNKNOWN: -1}
    want = []
    for k in range(n_ms):
        for e in integ.process_pseudosymbol(tt[k, 0], _pseudosymbol(rec[0, k], tt[k, 0], tt[k, 1])):
            want.append((k, e.receiver_timestamp, e.trailing_edge_receiver_timestamp, code[e.bit_value]))
    got = [(int(e["ms_index"]), float(e["receiver_timestamp"]), float(e["trailing_edge_receiver_timestamp"]), int(e["bit_value"]))
           for e in ev]
    assert got == want and len(got) > 300
    # the planted data bits come back (up to the BPSK sign ambiguity) once the loop has pulled in
    bits = np.array([g[3] for g in got[60:]])
    assert (bits >= 0).mean() > 0.98
    with pytest.raises(RuntimeError):
        trk.integrate_bits(n_ms - 1, tt[:-1, 0], tt[:-1, 1])  # no records of that length on the device
    trk.close()
