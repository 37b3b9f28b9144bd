"""C/N0 and phase-lock windows on the device (gb200_tracker_signal_windows, TrackerBank.signal_quality) behind the
tracking kernel: a bank of channels at different planted C/N0 and one with no signal, at 2.046, 4.092 and 16.368 Msps.
Against the host build of the estimator core run over the downloaded records (exact, C/N0 to 1e-12 relative), the
planted C/N0, calls of other sizes, the records_device path, the stop rule, every error case, and the rest of the
receiver chain, which must not notice the call."""
import math

import numpy as np
import pytest

import signal_oracle as so
from oracle import nav_oracle as nav
from oracle import orbit_oracle as orb
from oracle import tracker_oracle as t
from signal_support import SignalEmulator, assert_windows_match, without_ms_index

pytestmark = pytest.mark.gpu
SIGMA = 0.02
# (sv, doppler, code phase, carrier phase, planted C/N0 in dB-Hz; None: the satellite is not in the IQ)
CHANNELS = [(5, 1200.0, 300, 0.7, 43.0), (12, -2100.0, 1500, 2.0, 47.0), (21, 3300.0, 40, 4.1, 51.0),
            (27, -700.0, 900, 5.5, None)]
RATES = {2046: 3000, 4092: 2000, 16368: 1200}  # samples per ms -> milliseconds of IQ


def _bank(n, channels=CHANNELS):
    from gypsum_b200.antenna_sample_provider import SampleProviderAttributes
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import TrackerBank

    codes = generate_replica_prn_signals()
    seeds = [(GpsSatellite(GpsSatelliteId(c[0]), codes[GpsSatelliteId(c[0])], n // 1023), c[1], c[3], c[2])
             for c in channels]
    return TrackerBank(seeds, SampleProviderAttributes(1000 * n, n))


def _iq(n, n_ms, seed=3):
    fs = 1000 * n
    chans = [(c[0], c[1], 0.0, c[2], c[3], math.sqrt(10 ** (c[4] / 10) * SIGMA * SIGMA / fs))
             for c in CHANNELS if c[4] is not None]
    return t.synth_tracking_iq(seed, n, n_ms, fs, chans, SIGMA)


@pytest.fixture(scope="module", params=sorted(RATES))
def tracked(request, native_lib):
    """(n, bank, records [channel][ms], start times) after one process call over the rate's IQ."""
    n = request.param
    n_ms = RATES[n]
    bank = _bank(n)
    ts = np.array([t.chunk_times(k, 1000 * n, n)[0] for k in range(n_ms)])
    rec = bank.process(_iq(n, n_ms), ts)
    yield n, bank, rec, ts
    bank.native.close()


def _device(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def _fresh(bank):
    from gypsum_b200 import _native

    nc = bank.n_channels
    return _native.Tracker(bank.engine, list(range(nc)), [0.0] * nc, [0.0] * nc, [0] * nc)


def _calls(trk, rec, ts, w, sizes):
    """The windows of calls of the given sizes (cycled) over the records, through records_device."""
    import torch

    per = [[] for _ in range(rec.shape[0])]
    a = 0
    i = 0
    while a < rec.shape[1]:
        b = min(rec.shape[1], a + sizes[i % len(sizes)])
        d = _device(rec[:, a:b])
        got = trk.signal_windows(b - a, ts[a:b], w, records_device_ptr=d.data_ptr())
        torch.cuda.synchronize()
        for c in range(rec.shape[0]):
            per[c].append(got[c])
        a, i = b, i + 1
    return [np.concatenate(p) for p in per]


@pytest.mark.parametrize("w", [20, 100])
def test_device_equals_host_core_and_planted(tracked, w):
    n, bank, rec, ts = tracked
    trk = _fresh(bank)
    d = _device(rec)
    got = trk.signal_windows(len(ts), ts, w, records_device_ptr=d.data_ptr())
    floor = so.noise_floor_dbhz(n)
    for c, ch in enumerate(CHANNELS):
        assert not rec["lost"][c].any()
        emu = SignalEmulator(w, n)
        assert_windows_match(got[c], emu.run(rec[c], ts), (n, w, c))
        assert len(got[c]) == len(ts) // w
        if ch[4] is None:
            assert (got[c]["status"] == so.NOISE).all(), got[c]["cn0_dbhz"]
            assert got[c]["cn0_dbhz"][~np.isnan(got[c]["cn0_dbhz"])].mean() <= floor + 0.3
        else:
            steady = got[c][1:]  # after the loop's pull-in
            assert (steady["status"] == so.SIGNAL).all(), steady["cn0_dbhz"]
            assert abs(steady["cn0_dbhz"].mean() - ch[4]) <= 0.8, (n, c, steady["cn0_dbhz"].mean())
    trk.close()


def test_null_path_and_split_calls(tracked):
    """TrackerBank.signal_quality over the process call's records equals records_device in one call, and calls of 1, 7,
    333 and 1000 ms give the same windows byte for byte apart from ms_index."""
    n, bank, rec, ts = tracked
    w = 100
    trk = _fresh(bank)
    one = trk.signal_windows(len(ts), ts, w, records_device_ptr=_device(rec).data_ptr())
    trk.close()
    bank2 = _bank(n)
    rec2 = bank2.process(_iq(n, len(ts)), ts)
    assert rec2.tobytes() == rec.tobytes()
    null = bank2.signal_quality(ts, window_ms=w)
    bank2.native.close()
    for c in range(len(CHANNELS)):
        assert null[c].tobytes() == one[c].tobytes(), c
    for sizes in ([1], [7], [333], [1000], [1, 7, 333, 1000]):
        m = 1200 if sizes == [1] else len(ts)  # one call per millisecond over the first 1200 only
        trk = _fresh(bank)
        split = _calls(trk, rec[:, :m], ts[:m], w, sizes)
        trk.close()
        for c in range(len(CHANNELS)):
            want = one[c][one[c]["first_ms"] + one[c]["n_ms"] <= m]
            assert without_ms_index(split[c]) == without_ms_index(want), (sizes, c)


def test_lost_channel_stops(tracked):
    """A channel whose record says `lost` emits its cut window at once and nothing afterwards, even after set_state clears
    the flag; the others go on."""
    n, bank, rec, ts = tracked
    w = 100
    cut = rec.copy()
    cut["lost"][1, 250] = 1
    cut["lost"][2, 300] = 1  # on a window boundary: no cut window
    cut["lost"][3, 5] = 1    # a cut window of 5 records: status 0
    trk = _fresh(bank)
    got = trk.signal_windows(len(ts), ts, w, records_device_ptr=_device(cut).data_ptr())
    for c in range(4):
        assert_windows_match(got[c], SignalEmulator(w, n).run(cut[c], ts), c)
    assert len(got[1]) == 3 and got[1]["n_ms"][-1] == 50 and got[1]["ms_index"][-1] == 249
    assert len(got[2]) == 3 and (got[2]["n_ms"] == w).all()
    assert len(got[3]) == 1 and got[3]["status"][0] == so.NONE and got[3]["n_ms"][0] == 5
    assert len(got[0]) == len(ts) // w
    trk.set_state(1, 0.0, 0.0, 0.0, 0)
    again = trk.signal_windows(len(ts), ts, w, records_device_ptr=_device(rec).data_ptr())
    assert [len(a) for a in again[1:]] == [0, 0, 0] and len(again[0]) == len(ts) // w
    trk.close()


def test_signal_window_errors(tracked):
    """EINVAL: W out of range, no start times, null or empty outputs; ESTATE: another W after the first call, no
    records of n_ms behind the chain; truncation: the count exceeds max_windows."""
    from gypsum_b200 import _native

    n, bank, rec, ts = tracked
    trk = _fresh(bank)
    d = _device(rec[:, :200])
    for bad in (19, 60001, 0, -5):
        with pytest.raises(ValueError, match="window_ms"):
            trk.signal_windows(200, ts[:200], bad, records_device_ptr=d.data_ptr())
    with pytest.raises(RuntimeError, match="no records of 200 ms"):
        trk.signal_windows(200, ts[:200], 20)  # this tracker has processed nothing
    lib = trk._lib
    out = np.zeros((trk.n_channels, 4), dtype=_native.SIGNAL_DTYPE)
    cnt = np.zeros(trk.n_channels, dtype=np.int32)
    tsa = np.ascontiguousarray(ts[:200])
    for args in ((200, None, 20, d.data_ptr(), out.ctypes.data, 4, cnt.ctypes.data),
                 (0, tsa.ctypes.data, 20, d.data_ptr(), out.ctypes.data, 4, cnt.ctypes.data),
                 (200, tsa.ctypes.data, 20, d.data_ptr(), None, 4, cnt.ctypes.data),
                 (200, tsa.ctypes.data, 20, d.data_ptr(), out.ctypes.data, 0, cnt.ctypes.data),
                 (200, tsa.ctypes.data, 20, d.data_ptr(), out.ctypes.data, 4, None)):
        assert lib.gb200_tracker_signal_windows(trk._h, *args) == _native.EINVAL
    # truncation: 200 ms at W = 20 is 10 windows per channel, 4 kept
    assert lib.gb200_tracker_signal_windows(trk._h, 200, tsa.ctypes.data, 20, d.data_ptr(), out.ctypes.data, 4,
                                            cnt.ctypes.data) == _native.OK
    assert (cnt == 10).all()
    full = SignalEmulator(20, n).run(rec[0, :200], ts[:200])
    assert_windows_match(out[0], full[:4])
    with pytest.raises(RuntimeError, match="window_ms = 20"):
        trk.signal_windows(200, ts[:200], 100, records_device_ptr=d.data_ptr())
    with pytest.raises(RuntimeError, match="too small"):
        trk.signal_windows(200, ts[:200], 20, records_device_ptr=d.data_ptr(), max_windows=3)
    trk.close()
    with pytest.raises(RuntimeError, match="no records of 10 ms"):
        bank.native.signal_windows(10, ts[:10], 20)  # the bank's last process call held more


def test_chain_unchanged_by_signal_quality(native_lib):
    """Calling signal_quality between process and the rest of the chain leaves the bits, subframes, subframe fields,
    position fixes and velocity fixes byte-identical to a run without it."""
    from gypsum_b200.antenna_sample_provider import SampleProviderAttributes
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite
    from gypsum_b200.tracker import TrackerBank

    n, fs = 2046, 2046000
    erng = np.random.default_rng(11)
    chans = []
    for i, (sv, dop, code, cph) in enumerate(((3, 500.3, 333, 1.0), (9, -1500.3, 999, 2.5), (17, 2500.3, 1555, 4.0),
                                              (30, -3000.3, 222, 5.5))):
        eph = orb.realistic_ephemeris(erng, sv)
        sfs = orb.ephemeris_subframes(eph, 11, first_id=1, tow0=20000, seed=i)
        chans.append((sv, dop, code, cph, 0.005, np.concatenate([np.asarray(sf, np.int8) for sf in sfs]), 7))
    codes = generate_replica_prn_signals()
    seeds = [(GpsSatellite(GpsSatelliteId(c[0]), codes[GpsSatelliteId(c[0])], n // 1023), round(c[1]), c[3], c[2])
             for c in chans]
    banks = [TrackerBank(seeds, SampleProviderAttributes(fs, n)) for _ in range(2)]
    n_fixed, n_windows = 0, 0
    for k0 in range(0, 60000, 1000):
        x = nav.synth_lnav_iq(21, n, fs, k0, 1000, chans, sigma=0.01)
        tt = np.array([t.chunk_times(k, fs, n) for k in range(k0, k0 + 1000)])
        outs = []
        for b, bank in enumerate(banks):
            recs = bank.process(x, tt[:, 0])
            if b == 1:
                q = bank.signal_quality(tt[:, 0], window_ms=500)
                n_windows += sum(len(w) for w in q)
            bits = bank.integrate_bits(tt[:, 0], tt[:, 1])
            sub = bank.decode_subframes()
            fields = bank.parse_subframes()
            fixes = bank.position_fixes(tt[:, 0])
            vel = bank.velocity_fixes()
            outs.append((recs.tobytes(), [a.tobytes() for a in bits], [a.tobytes() for a in sub],
                         repr(fields), bank.observations().tobytes(), fixes.tobytes(), vel.tobytes()))
        assert outs[0] == outs[1], k0
        n_fixed += int((fixes["status"] == 1).sum())
    assert n_windows == 4 * 120 and n_fixed > 0, (n_windows, n_fixed)
    for bank in banks:
        bank.native.close()
