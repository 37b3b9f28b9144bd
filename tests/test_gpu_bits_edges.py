"""The navigation-bit integration kernel (k_integrate_bits in bits.cu) at its batch and channel edges, against the
float64 integrator (gypsum_b200.navigation_bit_integrator, fed as tracker.py feeds it: each symbol stamped with its
chunk times delayed by code_phase / 2046 ms) bit for bit: ms index, timestamps, value, slide and final state.

Each channel carries its own symbols (its own bits, bit phase and bursts of noise that make UNKNOWN bits and force
resynchronisation) and its own nonzero, changing code phase, so a channel mix-up or a wrong delay shows.  The lanes
take 32 records at a time and the warps of a block (four) one channel each: the tests cover 1..9 channels, calls of
1, 31, 32, 33, 63, 64 and 65 ms, lost lock at lanes 0, 1, 30, 31 and 32 of a batch, at in-call index 0 and after the
channel stopped, start times that cross the 40 s resynchronisation horizon at in-call indices 0, 31 and 32, event
buffers smaller than the events, and the chain into the subframe decoder."""
import ctypes as C

import numpy as np
import pytest

from gpu_support import make_engine
from oracle import nav_oracle as nav

pytestmark = pytest.mark.gpu
N, FS = 2046, 2046000
BATCHES = (1, 31, 32, 33, 63, 64, 65)


@pytest.fixture(scope="module")
def engine(native_lib):
    e = make_engine(FS, N)
    yield e
    e.close()


def symbols(seed, n_ms, bits=None, bursts=True):
    """+-1 symbols of one channel: random bits (or the given ones) 20 symbols each from a seeded bit phase, symbols
    flipped at random, more often in bursts."""
    rng = np.random.default_rng(seed)
    off = int(rng.integers(0, 20))
    if bits is None:
        bits = rng.integers(0, 2, n_ms // 20 + 2)
    i = np.clip((np.arange(n_ms) - off) // 20, 0, len(bits) - 1)
    sym = np.where(np.arange(n_ms) < off, 1, 2 * np.asarray(bits)[i] - 1)
    flip = rng.random(n_ms) < 0.03
    for a in rng.integers(0, max(n_ms - 200, 1), n_ms // 1500 if bursts else 0):
        flip[a:a + 200] |= rng.random(min(200, n_ms - a)) < 0.4
    return np.where(flip, -sym, sym).astype(np.int32)


def records(sym, code_phase, lost=None):
    from gypsum_b200._native import TRACK_DTYPE

    rec = np.zeros(sym.shape, dtype=TRACK_DTYPE)
    rec["symbol"] = sym
    rec["code_phase"] = code_phase
    if lost is not None:
        rec["lost"] = lost
    return rec


class BitOracle:
    """One channel's NavigationBitIntegrator over TRACK_DTYPE records; stops at the first lost record."""

    def __init__(self, sv):
        from gypsum_b200.navigation_bit_integrator import NavigationBitIntegrator

        self.integ = NavigationBitIntegrator(sv)
        self.stopped = 0

    def call(self, rec, t0, t1):
        """Events (ms index in the call, start, end, value, slide) of one call."""
        from gypsum_b200.tracker import BitValue, _pseudosymbol

        code = {BitValue.ONE: 1, BitValue.ZERO: 0, BitValue.UNKNOWN: -1}
        out = []
        for k in range(rec.size):
            if self.stopped:
                break
            if rec["lost"][k]:
                self.stopped = 1
                break
            for e in self.integ.process_pseudosymbol(t0[k], _pseudosymbol(rec[k], t0[k], t1[k])):
                out.append((k, e.receiver_timestamp, e.trailing_edge_receiver_timestamp, code[e.bit_value], self.integ.slide))
        return out

    def state(self):
        h = self.integ.history
        return [h.emitted_bit_count, h.failed_bit_count, h.processed_pseudosymbol_count, self.integ.slide,
                h.determined_bit_phase, h.previous_bit_phase_decision, h.pseudosymbol_cursor_within_queue, self.stopped]


def _device(rec):
    import torch

    return torch.from_numpy(np.ascontiguousarray(rec).view(np.uint8).reshape(rec.shape[0], -1).copy()).cuda()


def _events(ev):
    return [(int(e["ms_index"]), float(e["receiver_timestamp"]), float(e["trailing_edge_receiver_timestamp"]),
             int(e["bit_value"]), int(e["slide"])) for e in ev]


def _bit_state(trk, c):
    st = trk.bit_state(c)
    return [st[k] for k in ("emitted_bit_count", "failed_bit_count", "processed_pseudosymbol_count", "slide",
                            "determined_bit_phase", "previous_bit_phase_decision", "pseudosymbol_cursor_within_queue",
                            "stopped")]


def run_calls(engine, sym, cph, lost, sizes, t_first=0.0):
    """Channels' records (sym, code phase, lost: [n_ch, n_ms]) through integrate_bits in calls of `sizes` ms, every
    call against the oracle; returns the tracker and the oracles."""
    from gypsum_b200 import _native

    n_ch, n_ms = sym.shape
    trk = _native.Tracker(engine, [(3 * c) % 32 for c in range(n_ch)], [0.0] * n_ch, [0.0] * n_ch, [0] * n_ch)
    orc = [BitOracle(c + 1) for c in range(n_ch)]
    ts = np.round(t_first + 0.001 * np.arange(n_ms), 9)
    te = np.round(ts + 0.001, 9)
    a = 0
    for n in sizes:
        b = min(a + n, n_ms)
        rec = records(sym[:, a:b], cph[:, a:b], lost[:, a:b])
        ev = trk.integrate_bits(b - a, ts[a:b], te[a:b], _device(rec).data_ptr())
        for c in range(n_ch):
            want = orc[c].call(rec[c], ts[a:b], te[a:b])
            assert _events(ev[c]) == want, (n_ch, a, b, c)
        a = b
        if a == n_ms:
            break
    for c in range(n_ch):
        assert _bit_state(trk, c) == orc[c].state(), (n_ch, c)
    return trk, orc


def _channels(n_ch, n_ms, seed):
    sym = np.stack([symbols((seed, c), n_ms) for c in range(n_ch)])
    # a distinct nonzero code phase per channel, drifting by a chip now and then
    cph = np.stack([(157 * c + 211 + (np.arange(n_ms) // 97) % 5) % 2046 for c in range(n_ch)]).astype(np.int32)
    return sym, cph, np.zeros((n_ch, n_ms), dtype=np.int32)


@pytest.mark.parametrize("n_ch", range(1, 10))
def test_distinct_channels_at_batch_edges(engine, n_ch):
    """1..9 channels of distinct symbols and code phases in calls of 1, 31, 32, 33, 63, 64 and 65 ms, round after
    round for 3 s: bit phases found, lost and re-found, every event and the final state the oracle's."""
    n_ms = 3000
    # channel 6 (code phase 1153..1157 chips) caught the delayed stamps rounded once through a fused multiply-add
    sym, cph, lost = _channels(n_ch, n_ms, 11 + n_ch)
    sizes = list(BATCHES) * (n_ms // sum(BATCHES) + 1)
    trk, orc = run_calls(engine, sym, cph, lost, sizes)
    assert all(o.integ.history.emitted_bit_count > 100 for o in orc)
    trk.close()


def test_lost_lock_edges(engine):
    """Channels losing lock at lanes 0, 1, 30, 31 and 32 of the third batch of a call, at in-call index 0 of the next
    call, and one that never does; every channel gets later calls, and a stopped one emits nothing in them."""
    n_ms = 1500
    sym, cph, lost = _channels(7, n_ms, 5)
    sizes = [700, 300, 33, 467]
    for c, k in enumerate((64, 65, 94, 95, 96)):
        lost[c, 700 + k] = 1
        lost[c, 700 + k + 1:] = 2
    lost[5, 1000] = 1
    lost[5, 1001:] = 2
    trk, orc = run_calls(engine, sym, cph, lost, sizes)
    assert [o.stopped for o in orc] == [1] * 6 + [0]
    assert [o.integ.history.processed_pseudosymbol_count for o in orc] == [764, 765, 794, 795, 796, 1000, 1500]
    trk.close()


@pytest.mark.parametrize("at", [0, 31, 32])
def test_resync_horizon(engine, at):
    """Start times that reach 40 s at in-call index `at` of a call that begins 2000 - `at` ms in, so the period's
    resynchronisation check (every 1000 ms) falls on the first millisecond past the horizon; the symbols' bit phase
    moves by 7 ms at 1700 ms and again at 2010 ms."""
    n_ms = 2600
    sym, cph, lost = _channels(5, n_ms, 40 + at)
    for c in range(5):
        s = np.concatenate([sym[c, :1700], np.repeat(sym[c, 1700], 7), sym[c, 1700:]])
        sym[c] = np.concatenate([s[:2010], s[2017:], np.ones(14, dtype=np.int32)])[:n_ms]
    sizes = [1000, 1000 - at, 100, 500]
    trk, _ = run_calls(engine, sym, cph, lost, sizes, t_first=40.0 - 0.001 * 2000)
    trk.close()


def test_event_buffer_truncation(engine):
    """An event buffer of 3 per channel for a call with more: the counts keep counting past it, and the events kept
    are the first ones."""
    from gypsum_b200 import _native

    n_ch, n_ms = 6, 900
    sym, cph, lost = _channels(n_ch, n_ms, 77)
    trk = _native.Tracker(engine, list(range(n_ch)), [0.0] * n_ch, [0.0] * n_ch, [0] * n_ch)
    ts = np.round(0.001 * np.arange(n_ms), 9)
    te = np.round(ts + 0.001, 9)
    rec = records(sym, cph, lost)
    dev = _device(rec)
    ev = np.zeros((n_ch, 3), dtype=_native.BIT_DTYPE)
    cnt = np.zeros(n_ch, dtype=np.int32)
    rc = engine._lib.gb200_tracker_integrate_bits(trk._h, n_ms, ts.ctypes.data, te.ctypes.data, C.c_void_p(dev.data_ptr()),
                                                  ev.ctypes.data, 3, cnt.ctypes.data)
    assert rc == _native.OK
    for c in range(n_ch):
        want = BitOracle(c + 1).call(rec[c], ts, te)
        assert cnt[c] == len(want) > 3 and _events(ev[c]) == want[:3], c
    trk.close()


def test_chain_into_the_subframe_decoder(engine):
    """Six channels carrying LNAV bits (more than one block of four warps), one losing lock: integrate_bits on device
    records, then decode_subframes of the chain, which reads each channel's bit events at the integrator's stride;
    the subframes are the oracle decoder's fed the oracle integrator's bits, and the channel that lost lock stops."""
    n_ch, n_ms = 6, 27000
    sym = np.stack([symbols((9, c), n_ms, np.concatenate(nav.lnav_frames(60 + c, n_ms // 6000 + 1, first_id=c % 5 + 1)),
                            bursts=False) for c in range(n_ch)])
    _, cph, lost = _channels(n_ch, n_ms, 3)
    lost[4, 24000] = 1
    lost[4, 24001:] = 2
    from gypsum_b200 import _native

    trk = _native.Tracker(engine, list(range(n_ch)), [0.0] * n_ch, [0.0] * n_ch, [0] * n_ch)
    borc = [BitOracle(c + 1) for c in range(n_ch)]
    dec = [nav.NavDecoderOracle() for _ in range(n_ch)]
    ts = np.round(0.001 * np.arange(n_ms), 9)
    te = np.round(ts + 0.001, 9)
    subframes = [0] * n_ch
    for a in range(0, n_ms, 3001):
        b = min(a + 3001, n_ms)
        rec = records(sym[:, a:b], cph[:, a:b], lost[:, a:b])
        bits = trk.integrate_bits(b - a, ts[a:b], te[a:b], _device(rec).data_ptr())
        sub = trk.decode_subframes()
        for c in range(n_ch):
            want_bits = borc[c].call(rec[c], ts[a:b], te[a:b])
            assert _events(bits[c]) == want_bits, (a, c)
            want = []
            for j, (_, t0, t1, v, _) in enumerate(want_bits):
                want += dec[c].push(v, t0, t1, j)
            want_rows, want_words = nav.events_to_arrays(want)
            e = sub[c]
            rows = np.stack([e["bit_index"], e["kind"], e["subframe_id"], e["tow"], e["phase"], e["polarity"], e["parity_ok"],
                             e["receiver_timestamp"], e["trailing_edge_receiver_timestamp"]], axis=1).astype(np.float64)
            assert np.array_equal(rows.reshape(-1, 9), want_rows), (a, c)
            assert np.array_equal(e["words"].astype(np.int64).reshape(-1, 10), want_words), (a, c)
            subframes[c] += int((e["kind"] == nav.KIND_SUBFRAME).sum())
    for c in range(n_ch):
        st = trk.subframe_state(c)
        want = dec[c].state()
        if borc[c].stopped and want[4] == 0:
            want[4] = _native.STOP_LOST_LOCK
        assert [-1 if st["determined_subframe_phase"] is None else st["determined_subframe_phase"], st["emitted_subframe_count"],
                st["polarity"], st["queued_bit_count"], st["stopped"], st["processed_bit_count"]] == want, c
    assert trk.subframe_state(4)["stopped"] == _native.STOP_LOST_LOCK
    assert min(subframes) >= 1 and sum(subframes) >= 10, subframes
    trk.close()
