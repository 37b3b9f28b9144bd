"""Small end-to-end exercise of every kernel for compute-sanitizer (memcheck / racecheck / synccheck).
usage (GPU box): compute-sanitizer --tool racecheck python tools/sanitize_small.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gypsum_b200 import _native  # noqa: E402
from gypsum_b200.gps_ca_prn_codes import ca_code_chips  # noqa: E402
from gypsum_b200 import synth as o  # noqa: E402
from gypsum_b200 import synth as to  # noqa: E402

chips = np.stack([ca_code_chips(sv) for sv in range(1, 33)]).astype(np.uint8)
for n, m in ((2046, 2), (4092, 1)):
    fs = n * 1000
    eng = _native.Engine(fs, n)
    eng.set_replicas(chips)
    x = o.synth_iq(1, n, m, fs, [(25, 1500.0, 777 % n, 0.3, 0.3)])
    eng.upload_iq(x)
    dop = np.arange(-2000, 2001, 500.0)
    g = eng.acquire_grid(1, m, [24, 0, 5], dop)                       # split path (rsplit > 1)
    c = eng.acquire_cells([24, 3, 24, 7], [1500.0, 0.0, 1000.0, -250.0], m, _native.COHERENT, probe_idx=[777 % n, 0, 1, 2])
    p = eng.correlation_profile(24, 1500.0, m, _native.NON_COHERENT)
    assert int(p.argmax()) == 777 % n == int(g["argmax"][0, 0, 7])
    if n == 2046:
        big = eng.acquire_grid(2, 1, np.arange(32), np.linspace(-10000, 10000, 161))  # full 32-PRN grid, 12-warp one-warp build
        r = eng.detect([24, 2], m)
        assert int(big["argmax"][0, 24, int(np.argmax(big["peak"][0, 24]))]) == 777 and int(r["code_phase"][0]) == 777
        sg = eng.acquire_grid_semicoherent(1, m, 2, [24, 0, 5], dop)  # k_segment_spectra<2>, one segment of two ms
        assert int(sg["argmax"][0, 0, 7]) == 777
        xs = to.synth_tracking_iq(3, n, 12, fs, [(25, 1500.3, 0.0, 777, 0.3, 0.004)])
        eng.upload_iq(xs)
        t = _native.Tracker(eng, [24, 6], [1500.0, -100.0], [0.0, 0.0], [777, 5])
        rec, prof = t.process(12, [round(k * n / fs, 6) for k in range(12)], want_profiles=True)
        assert rec["symbol"].shape == (2, 12)
        ts = np.array([round(k * n / fs, 6) for k in range(12)])
        for _ in range(9):  # > 80 symbols: bit-phase search and bit emission of the navigation-bit kernel
            t.process(12, ts)
            bits = t.integrate_bits(12, ts, ts + 0.001)
            sub = t.decode_subframes()  # subframe decoding of the bits just integrated
        assert len(bits) == 2 and t.bit_state(0)["processed_pseudosymbol_count"] == 108
        t.parse_subframes()  # subframe fields and world-model state over the chain just decoded
        assert t.observations().shape == (2, 12)
        assert t.position_fixes(ts).shape == (12,)  # plan, both passes and finish of the position fix
        assert t.receiver_state()["slide"] is None
        assert t.velocity_fixes().shape == (12,)  # the velocity fix on the tracking records' Dopplers
        # C/N0 windows on the chain's records: a window left open by the first call and closed by the second
        assert [len(w) for w in t.signal_windows(12, ts, 20)] == [0, 0]
        assert [len(w) for w in t.signal_windows(12, ts, 20)] == [1, 1]
        # subframe decoding over caller bit events: full warp preamble scan, phase, drain, a reset and a re-sync
        import torch

        nb = 1400
        sb = np.zeros((2, nb), dtype=_native.BIT_DTYPE)
        pre = [1, 0, 0, 0, 1, 0, 1, 1]
        vals = np.random.default_rng(1).integers(0, 2, nb)
        for at in range(0, nb - 8, 300):
            vals[at:at + 8] = pre
        vals[650] = -1
        sb["bit_value"] = [vals, np.where(vals < 0, vals, 1 - vals)]
        sb["receiver_timestamp"] = np.arange(nb) * 0.02
        sb["trailing_edge_receiver_timestamp"] = np.arange(nb) * 0.02 + 0.02
        sbd = torch.from_numpy(sb.view(np.uint8).reshape(2, -1)).cuda()
        sub = t.decode_subframes(sbd.data_ptr(), [nb, nb - 100], nb)
        assert t.subframe_state(0)["processed_bit_count"] >= 600 and len(sub) == 2
        t.close()
        # the least-squares fix: a second tracker on the same IQ and chain, in that mode
        t = _native.Tracker(eng, [24, 6], [1500.0, -100.0], [0.0, 0.0], [777, 5])
        t.set_fix_solver("least_squares")
        t.process(12, ts)
        t.integrate_bits(12, ts, ts + 0.001)
        t.decode_subframes()
        t.parse_subframes()
        assert t.position_fixes(ts).shape == (12,)
        t.close()
        # the velocity fix on solved fixes: the first call of a recorded fix timeline, with caller Dopplers
        from oracle import fix_oracle as fx

        rx, chans = fx.golden_calls(np.load(os.path.join(ROOT, "tests", "golden", "fix.npz")), "realistic")[0]
        stride = max(len(ev) for ev, _ in chans)
        host = np.zeros((4, stride), dtype=_native.SUBFRAME_DTYPE)
        ems = np.zeros((4, stride), dtype=np.int32)
        for c, (events, _) in enumerate(chans):
            for j, (kind, w, te, ms) in enumerate(events):
                host[c, j]["kind"], host[c, j]["words"], host[c, j]["trailing_edge_receiver_timestamp"] = kind, w, te
                ems[c, j] = ms
        t = _native.Tracker(eng, [0, 1, 2, 3], [0.0] * 4, [0.0] * 4, [0] * 4)
        evd = torch.from_numpy(host.view(np.uint8).reshape(4, -1)).cuda()
        t.parse_subframes(evd.data_ptr(), [len(ev) for ev, _ in chans], stride, ems, [d for _, d in chans], len(rx))
        t.position_fixes(rx)
        dopd = torch.full((4, len(rx)), 1234.5, dtype=torch.float64, device="cuda")
        assert (t.velocity_fixes(dopd.data_ptr())["status"] == 1).any()
        t.close()
        # pipelined batch stream: three streams, pageable staging
        gs = _native.GridStream(eng, 2, 1, [24, 0, 5], dop, _native.NON_COHERENT, depth=2)
        xb = o.synth_iq(2, n, 2, fs, [(25, 1500.0, 777, 0.3, 0.3)])
        outs = []
        for k in range(4):
            if gs.in_flight == 2:
                outs.append(gs.collect().copy())
            gs.submit(xb)
        while gs.in_flight:
            outs.append(gs.collect().copy())
        assert all(int(u["argmax"][0, 0, 7]) == 777 for u in outs)
        gs.close()
        # round 2: multi-ms one-warp kernel, graph-replayed host grid, best-bin reduction, device ring, channel pool with
        # subset launches + undo, generic-replica kernel
        x10 = o.synth_iq(4, n, 3, fs, [(25, 1500.0, 777, 0.3, 0.3)])
        eng.upload_iq(x10)
        g3 = eng.acquire_grid(1, 3, np.arange(32), dop)
        assert int(g3["argmax"][0, 24, 7]) == 777
        for _ in range(3):
            gh = eng.acquire_grid_host(x10, 1, 3, np.arange(32), dop)
        assert np.array_equal(gh["argmax"], g3["argmax"])
        eng.upload_iq(x10)
        best = eng.acquire_grid_best(1, 3, np.arange(32), dop)
        assert int(best["code_phase"][0, 24]) == 777 and float(best["doppler"][0, 24]) == 1500.0
        ring = _native.Ring(eng, 4)
        for k in range(6):
            ring.append(xs[k * n:(k + 1) * n])
        ring.bind_newest(3)
        pool = _native.Tracker.pool(eng, 4)
        pool.reset_channel(2, 24, 1500.0, 0.0, 777)
        pool.reset_channel(0, 6, -100.0, 0.0, 5)
        r1 = pool.process_channels([2, 0], 1, [0.003], keep_undo=True)
        pool.undo_channel(0)
        r2 = pool.process_channels([0], 1, [0.003])
        assert r1["symbol"][1, 0] == r2["symbol"][0, 0]
        pool.close()
        ring.close()
        eng.upload_iq(x10)
        rng = np.random.default_rng(0)
        odd = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
        pr = eng.correlation_profile_replica(odd, 250.0, 2, _native.NON_COHERENT)
        assert pr.shape == (n,)
    eng.close()
# rates where doppler_spectra runs its tail loop with separate rows and tiles: S = 5 (odd N, correlate split 1) and S = 12
# (split 12 at M = 1, 4 at M = 2)
for n in (5115, 12276):
    fs = n * 1000
    eng = _native.Engine(fs, n)
    eng.set_replicas(chips)
    x = o.synth_iq(5, n, 2, fs, [(25, 1500.0, n - 1, 0.3, 0.3)])
    eng.upload_iq(x)
    dop = np.arange(-2000, 2001, 500.0)
    for m in (1, 2):
        g = eng.acquire_grid(1, m, [24, 0, 5], dop)
        assert int(g["argmax"][0, 0, 7]) == n - 1
    # semi-coherent grid: k_segment_spectra (two-millisecond segment sums, tail loop), then its best bins
    sg = eng.acquire_grid_semicoherent(1, 2, 2, [24, 0, 5], dop)
    sb = eng.acquire_grid_semicoherent_best(1, 2, 2, [24, 0, 5], dop)
    assert int(sg["argmax"][0, 0, 7]) == n - 1 == int(sb["code_phase"][0, 0])
    c = eng.acquire_cells([24, 3, 24], [1500.0, 0.0, 1000.0], 2, _native.COHERENT, probe_idx=[n - 1, 0, n // 2])
    p = eng.correlation_profile(24, 1500.0, 2, _native.NON_COHERENT)
    r = eng.detect([24, 2], 2)
    assert int(p.argmax()) == n - 1 == int(c["argmax"][0]) == int(r["code_phase"][0])
    eng.close()
# 16.368 Msps tracking (k_track_channels_wide<16>): a channel bank with profiles, then a pool step with undo
n = 16368
fs = n * 1000
eng = _native.Engine(fs, n)
eng.set_replicas(chips)
xs = to.synth_tracking_iq(4, n, 3, fs, [(25, 1500.3, 0.0, 777, 0.3, 0.002)])
eng.upload_iq(xs)
t = _native.Tracker(eng, [24, 6], [1500.0, -100.0], [0.0, 0.0], [777, 5])
rec, prof = t.process(3, [round(k * n / fs, 6) for k in range(3)], want_profiles=True)
assert rec["symbol"].shape == (2, 3) and prof.shape == (2, 3, n)
t.close()
pool = _native.Tracker.pool(eng, 2)
pool.reset_channel(1, 24, 1500.0, 0.0, 777)
r1 = pool.process_channels([1], 1, [0.0], keep_undo=True)
pool.undo_channel(1)
r2 = pool.process_channels([1], 1, [0.0])
assert r1["symbol"][0, 0] == r2["symbol"][0, 0]
pool.close()
# the samples code-phase mode: a bank call with bits at a code phase past 2046, and a drop-in pool step
xs = to.synth_tracking_iq(5, n, 20, fs, [(25, 1500.3, 0.0, 12345, 0.3, 0.002)])
eng.upload_iq(xs)
t = _native.Tracker(eng, [24, 6], [1500.0, -100.0], [0.0, 0.0], [12345, n - 1])
t.set_code_phase_mode("samples")
ts = [round(k * n / fs, 6) for k in range(20)]
rec = t.process(20, ts)
t.integrate_bits(20, ts, [round((k + 1) * n / fs, 6) for k in range(20)])
assert (rec["code_phase"][0] >= 2046).all()
t.close()
pool = _native.Tracker.pool(eng, 2)
pool.set_code_phase_mode("samples")
pool.reset_channel(0, 24, 1500.0, 0.0, 12345)
r1 = pool.process_channels([0], 1, [0.0], keep_undo=True)
assert r1["code_phase"][0, 0] >= 2046
pool.close()
eng.close()
print("sanitize_small ok")
