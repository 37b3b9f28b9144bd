"""GPU parity of the subframe decoding kernel (nav.cu through gb200_tracker_decode_subframes) against event streams
recorded from the live reference decoder (tests/golden/nav_decoder.npz), and end to end behind the tracking and bit
integration kernels on IQ that carries LNAV data, against the planted subframes and the oracle decoder."""
import os

import numpy as np
import pytest

from gpu_support import make_engine
from oracle import nav_oracle as nav
from oracle import tracker_oracle as t

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "nav_decoder.npz")
STREAMS = ["clean", "negated", "unknown", "bad_tlm_how", "false_pair", "no_preamble", "raise", "parity"]
N, FS = 2046, 2046000


@pytest.fixture(scope="module")
def engine(native_lib):
    e = make_engine(FS, N)
    yield e
    e.close()


def _negate(bits):
    b = np.asarray(bits, dtype=np.int8)
    return np.where(b < 0, b, 1 - b).astype(np.int8)


def _rows(events, offset):
    rows = np.array([[offset + e["bit_index"], e["kind"], e["subframe_id"], e["tow"], e["phase"], e["polarity"],
                      e["parity_ok"], e["receiver_timestamp"], e["trailing_edge_receiver_timestamp"]] for e in events],
                    dtype=np.float64).reshape(-1, 9)
    return rows, np.array([e["words"] for e in events], dtype=np.int64).reshape(-1, 10)


def _decode_streams(trk, streams, chunk):
    """Feeds per-channel (bits, t0, t1) streams as device bit events, `chunk` bits per call; rows and words per channel."""
    import torch

    from gypsum_b200._native import BIT_DTYPE

    n_ch = len(streams)
    longest = max(s[0].size for s in streams)
    rows = [[] for _ in range(n_ch)]
    words = [[] for _ in range(n_ch)]
    for a in range(0, longest, chunk):
        host = np.zeros((n_ch, chunk), dtype=BIT_DTYPE)
        counts = np.zeros(n_ch, dtype=np.int32)
        for c, (bits, t0, t1) in enumerate(streams):
            m = max(0, min(chunk, bits.size - a))
            counts[c] = m
            host["bit_value"][c, :m] = bits[a:a + m]
            host["receiver_timestamp"][c, :m] = t0[a:a + m]
            host["trailing_edge_receiver_timestamp"][c, :m] = t1[a:a + m]
        dev = torch.from_numpy(host.view(np.uint8).reshape(n_ch, -1)).cuda()
        ev = trk.decode_subframes(dev.data_ptr(), counts, chunk)
        for c in range(n_ch):
            r, w = _rows(ev[c], a)
            rows[c].append(r)
            words[c].append(w)
    return [np.concatenate(r) for r in rows], [np.concatenate(w) for w in words]


def _state_list(st):
    return [-1 if st["determined_subframe_phase"] is None else st["determined_subframe_phase"], st["emitted_subframe_count"],
            st["polarity"], st["queued_bit_count"], st["stopped"], st["processed_bit_count"]]


@pytest.mark.parametrize("chunk", [997, 4001])
def test_golden_streams_on_the_device(engine, chunk):
    """Every golden stream and a negated copy of it, 16 channels in each call."""
    from gypsum_b200 import _native

    z = np.load(GOLDEN)
    streams = []
    for s in STREAMS:
        bits, t0, t1 = z[f"{s}_bits"], z[f"{s}_t0"], z[f"{s}_t1"]
        streams += [(bits, t0, t1), (_negate(bits), t0, t1)]
    trk = _native.Tracker(engine, list(range(len(streams))), [0.0] * len(streams), [0.0] * len(streams), [0] * len(streams))
    rows, words = _decode_streams(trk, streams, chunk)
    for i, s in enumerate(STREAMS):
        assert np.array_equal(rows[2 * i], z[f"{s}_events"]), s
        assert np.array_equal(words[2 * i], z[f"{s}_words"]), s
        assert _state_list(trk.subframe_state(2 * i)) == list(z[f"{s}_final"]), s
        bits, t0, t1 = streams[2 * i + 1]
        ev, final = nav.decode(bits, t0, t1)
        want_rows, want_words = nav.events_to_arrays(ev)
        assert np.array_equal(rows[2 * i + 1], want_rows) and np.array_equal(words[2 * i + 1], want_words), s
        assert _state_list(trk.subframe_state(2 * i + 1)) == final, s
    trk.close()


def test_queue_overflow_latches_at_the_documented_bit(engine):
    from gypsum_b200 import _native

    bits = nav.no_preamble_noise(11, 4300)
    bits[1000:1003] = -1
    t0, t1 = nav.bit_times(bits.size)
    trk = _native.Tracker(engine, [0], [0.0], [0.0], [0])
    rows, _ = _decode_streams(trk, [(bits, t0, t1)], 1500)
    st = trk.subframe_state(0)
    assert _state_list(st) == [-1, 0, 0, 4096, _native.STOP_OVERFLOW, 4096]
    assert np.array_equal(rows[0][:, 0], np.arange(3599, 4096)) and (rows[0][:, 1] == nav.KIND_CANNOT).all()
    trk.close()


def _lnav_end_to_end(n, fs, chans, seconds, seed, block_ms=1000):
    """Tracks `chans` (sv, doppler, code_phase, carrier_phase, amplitude, subframes, first_bit_ms) over `seconds` of IQ
    through TrackerBank in blocks, integrating bits and decoding subframes after every block.  Returns the subframe
    events per channel (bit_index made global) and the bit events the decoder was fed, per channel and call."""
    from gypsum_b200.antenna_sample_provider import SampleProviderAttributes
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import TrackerBank

    attrs = SampleProviderAttributes(fs, n)
    codes = generate_replica_prn_signals()
    s = n // 1023
    seeds = [(GpsSatellite(GpsSatelliteId(c[0]), codes[GpsSatelliteId(c[0])], s), round(c[1]), c[3], c[2]) for c in chans]
    bank = TrackerBank(seeds, attrs)
    iq_chans = [(c[0], c[1], c[2], c[3], c[4], np.concatenate([np.asarray(sf, np.int8) for sf in c[5]]), c[6]) for c in chans]
    events = [[] for _ in chans]
    fed = [[] for _ in chans]
    n_bits = [0] * len(chans)
    for k0 in range(0, seconds * 1000, block_ms):
        x = nav.synth_lnav_iq(seed, n, fs, k0, block_ms, iq_chans, sigma=0.01)
        tt = np.array([t.chunk_times(k, fs, n) for k in range(k0, k0 + block_ms)])
        bank.process(x, tt[:, 0])
        bits = bank.integrate_bits(tt[:, 0], tt[:, 1])
        sub = bank.decode_subframes()
        for c in range(len(chans)):
            fed[c].append(bits[c])
            for e in sub[c]:
                e = e.copy()
                e["bit_index"] += n_bits[c]
                events[c].append(e)
            n_bits[c] += len(bits[c])
    return bank, events, fed


def _check_channel(events, fed, planted, tow0, first_id):
    from gypsum_b200._native import subframe_bits

    sub = [e for e in events if e["kind"] == 0]
    assert len(sub) >= 3
    assert all(e["kind"] in (0, 1) for e in events)
    for e in sub:
        k = int(e["tow"]) - tow0
        assert 0 <= k < len(planted) and subframe_bits(e) == list(planted[k])
        assert int(e["subframe_id"]) == (first_id - 1 + k) % 5 + 1 and int(e["parity_ok"]) == 0x3FF
    assert all(int(b["tow"]) == int(a["tow"]) + 1 and int(b["subframe_id"]) == int(a["subframe_id"]) % 5 + 1
               for a, b in zip(sub, sub[1:]))
    # the oracle decoder fed the device's own bit events, call by call
    dec = nav.NavDecoderOracle()
    want = []
    base = 0
    for call in fed:
        for j, b in enumerate(call):
            want += [(base + ev[0], *ev[1:]) for ev in dec.push(int(b["bit_value"]), float(b["receiver_timestamp"]),
                                                                float(b["trailing_edge_receiver_timestamp"]), j)]
        base += len(call)
    got_rows, got_words = _rows(events, 0)
    want_rows, want_words = nav.events_to_arrays(want)
    assert np.array_equal(got_rows, want_rows) and np.array_equal(got_words, want_words)
    return dec


def test_subframes_behind_the_tracking_kernel():
    """4 channels x 40 s of IQ carrying LNAV at 2.046 Msps: TrackerBank.process in 1-s blocks, integrate_bits,
    decode_subframes; every subframe comes back upright and intact."""
    chans = []
    planted = []
    rng = np.random.default_rng(3)
    for i, sv in enumerate((5, 12, 19, 27)):
        sfs = nav.lnav_frames(40 + i, 9, first_id=i + 1, tow0=5000 + 100 * i)
        planted.append(sfs)
        chans.append((sv, float(rng.integers(-4000, 4000)) + 0.3, int(rng.integers(0, N)), float(rng.uniform(0, 6)), 0.004,
                      sfs, int(rng.integers(0, 20))))
    bank, events, fed = _lnav_end_to_end(N, FS, chans, 40, seed=9)
    for c in range(len(chans)):
        dec = _check_channel(events[c], fed[c], planted[c], 5000 + 100 * c, c + 1)
        st = bank.native.subframe_state(c)
        assert _state_list(st) == dec.state() and st["stopped"] == 0
    bank.native.close()


def test_subframes_behind_the_tracking_kernel_4092():
    n, fs = 4092, 4092000
    sfs = nav.lnav_frames(77, 9, first_id=3, tow0=12345)
    chans = [(14, -1733.3, 1501, 2.0, 0.004, sfs, 11)]
    bank, events, fed = _lnav_end_to_end(n, fs, chans, 40, seed=10)
    dec = _check_channel(events[0], fed[0], sfs, 12345, 3)
    assert _state_list(bank.native.subframe_state(0)) == dec.state()
    bank.native.close()


def test_decode_errors(engine):
    import ctypes as C

    import torch

    from gypsum_b200 import _native

    trk = _native.Tracker(engine, [24, 6], [1500.0, -100.0], [0.0, 0.0], [777, 5])
    with pytest.raises(RuntimeError, match="no undecoded bit events"):
        trk.decode_subframes()  # before any integrate call
    with pytest.raises(ValueError):
        trk.subframe_state(2)
    with pytest.raises(ValueError):
        trk.subframe_state(-1)
    assert trk.subframe_state(1)["processed_bit_count"] == 0
    # an integrate call whose bit events did not all fit: they never reached the device
    rec = np.zeros((2, 400), dtype=_native.TRACK_DTYPE)
    rec["symbol"] = 1
    dev = torch.from_numpy(rec.view(np.uint8).reshape(2, -1)).cuda()
    ts = np.arange(400) * 0.001
    ev = np.empty((2, 1), dtype=_native.BIT_DTYPE)
    cnt = np.empty(2, dtype=np.int32)
    lib = engine._lib
    rc = lib.gb200_tracker_integrate_bits(trk._h, 400, ts.ctypes.data, (ts + 0.001).ctypes.data, C.c_void_p(dev.data_ptr()),
                                          ev.ctypes.data, 1, cnt.ctypes.data)
    assert rc == _native.OK and (cnt > 1).all()
    with pytest.raises(ValueError, match="kept 1"):
        trk.decode_subframes()
    # a complete one decodes once
    trk.integrate_bits(400, ts, ts + 0.001, dev.data_ptr())
    trk.decode_subframes()
    assert trk.subframe_state(0)["processed_bit_count"] == trk.bit_state(0)["emitted_bit_count"] - int(cnt[0])
    with pytest.raises(RuntimeError, match="no undecoded bit events"):
        trk.decode_subframes()
    trk.close()
