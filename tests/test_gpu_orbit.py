"""GPU parity of the subframe field, world-model and per-millisecond satellite time and position kernels (orbit.cu
through gb200_tracker_parse_subframes / gb200_tracker_observations) against timelines recorded from the live reference
(tests/golden/orbit.npz), and end to end behind the tracking, bit and subframe kernels on IQ that carries planted
ephemerides, against the planted values and the oracle."""
import os

import numpy as np
import pytest

from oracle import gypsum_oracle as o
from oracle import nav_oracle as nav
from oracle import orbit_oracle as orb
from oracle import tracker_oracle as t

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "orbit.npz")
TIMELINES = ["realistic", "extreme", "week_edge", "order", "mixing", "lost"]
N, FS = 2046, 2046000


@pytest.fixture(scope="module")
def engine(native_lib):
    from gypsum_b200 import _native

    e = _native.Engine(FS, N)
    e.set_replicas(np.stack([o.ca_code(sv) for sv in range(1, 33)]).astype(np.uint8))
    yield e
    e.close()


def _rows(obs):
    return np.stack([obs["tow"], obs["x"], obs["y"], obs["z"], obs["prn_count"].astype(np.float64),
                     (obs["flags"] & ~orb.OBS_FROZEN).astype(np.float64)], axis=1)


def _parse_explicit(trk, per_channel, n_ms):
    """per_channel: [(events [(kind, words, t0, t1, ms)], drop_ms)] -> fields per channel (via device event arrays)."""
    import torch

    from gypsum_b200._native import SUBFRAME_DTYPE

    n_ch = len(per_channel)
    stride = max(1, max(len(ev) for ev, _ in per_channel))
    host = np.zeros((n_ch, stride), dtype=SUBFRAME_DTYPE)
    ems = np.zeros((n_ch, stride), dtype=np.int32)
    counts = np.zeros(n_ch, dtype=np.int32)
    drop = np.array([d for _, d in per_channel], dtype=np.int32)
    for c, (events, _) in enumerate(per_channel):
        counts[c] = len(events)
        for j, (kind, w, t0, t1, m) in enumerate(events):
            host[c, j]["kind"], host[c, j]["words"] = kind, w
            host[c, j]["receiver_timestamp"], host[c, j]["trailing_edge_receiver_timestamp"] = t0, t1
            ems[c, j] = m
    dev = torch.from_numpy(host.view(np.uint8).reshape(n_ch, -1)).cuda()
    return trk.parse_subframes(dev.data_ptr(), counts, stride, ems, drop, n_ms)


@pytest.mark.parametrize("name", TIMELINES)
def test_golden_timelines_on_the_device(engine, name):
    """Fields exact, parameter sets exact, time of week within 1 ulp, ECEF within 1e-4 m, state carried across calls."""
    from gypsum_b200 import _native

    z = np.load(GOLDEN)
    calls = orb.golden_calls(z, name)
    n_ch = len(calls[0][1])
    trk = _native.Tracker(engine, list(range(n_ch)), [0.0] * n_ch, [0.0] * n_ch, [0] * n_ch)
    fields = []
    worst = [0.0, 0.0]
    for c, (n_ms, chans) in enumerate(calls):
        got_fields = _parse_explicit(trk, chans, n_ms)
        obs = trk.observations()
        assert obs.shape == (n_ch, n_ms)
        for ch in range(n_ch):
            f = got_fields[ch]
            fields.append(np.array([[r["subframe_id"], r["tow_seconds"], *r["ints"], *r["bits"], *r["values"]] for r in f],
                                   dtype=np.float64).reshape(-1, 18))
            sel = (z[f"{name}_obs"][:, 0] == c) & (z[f"{name}_obs"][:, 1] == ch)
            want = z[f"{name}_obs"][sel]
            u, m = orb.compare_observations(_rows(obs[ch])[want[:, 2].astype(int)], want[:, 3:])
            worst = [max(worst[0], u), max(worst[1], m)]
            st = trk.orbit_state(ch)
            assert st["set_mask"] == z[f"{name}_mask"][c, ch]
            assert np.array_equal(st["params"], z[f"{name}_params"][c, ch])
    assert np.array_equal(np.concatenate(fields), z[f"{name}_fields"])
    print(f"{name}: worst time of week {worst[0]:.1f} ulp, worst ECEF {worst[1]:.3g} m")
    trk.close()


def test_observations_device_matches_host(engine):
    import torch

    from gypsum_b200 import _native

    z = np.load(GOLDEN)
    calls = orb.golden_calls(z, "realistic")
    trk = _native.Tracker(engine, [0, 1, 2], [0.0] * 3, [0.0] * 3, [0] * 3)
    n_ms, chans = calls[0]
    _parse_explicit(trk, chans, n_ms)
    host = trk.observations()
    dev = torch.empty(3 * n_ms * _native.OBSERVATION_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    trk.observations_device(dev.data_ptr())
    torch.cuda.synchronize()
    got = dev.cpu().numpy().view(_native.OBSERVATION_DTYPE).reshape(3, n_ms)
    assert np.array_equal(got.view(np.uint8), host.view(np.uint8))
    trk.close()


def test_errors_and_the_lost_channel(engine):
    from gypsum_b200 import _native

    trk = _native.Tracker(engine, [4, 4], [0.0, 0.0], [0.0, 0.0], [0, 0])
    with pytest.raises(ValueError, match="same replica row"):
        trk.parse_subframes()
    trk.close()
    trk = _native.Tracker(engine, [4, 5], [0.0, 0.0], [0.0, 0.0], [0, 0])
    with pytest.raises(RuntimeError, match="no unparsed subframe events"):
        trk.parse_subframes()
    with pytest.raises(RuntimeError, match="no gb200_tracker_parse_subframes call"):
        trk.observations()
    with pytest.raises(ValueError):
        trk.orbit_state(2)
    # a channel dropped at millisecond 40 and one never tracked before: counting per the receiver's order
    rng = np.random.default_rng(1)
    eph = orb.realistic_ephemeris(rng, 5)
    sfs = orb.ephemeris_subframes(eph, 3, tow0=100)
    events = [(0, orb.words_of(sf), 0.0, 0.5 + k, 10 + 10 * k) for k, sf in enumerate(sfs)]
    with pytest.raises(ValueError, match="out of order"):
        _parse_explicit(trk, [(events[::-1], -1), ([], -1)], 100)
    _parse_explicit(trk, [(events, 40), ([], -1)], 100)
    obs = trk.observations()
    assert list(obs["prn_count"][0, 38:42]) == [8, 9, -1, -1] and list(obs["prn_count"][1, :3]) == [1, 2, 3]
    assert np.isnan(obs["tow"][0, 40:]).all() and not np.isnan(obs["tow"][0, 39])
    st = trk.orbit_state(0)
    assert not st["counting"] and not (st["set_mask"] >> orb.TOW_LAST) & 1
    # the next call counts again from 1
    _parse_explicit(trk, [([], -1), ([], -1)], 5)
    assert list(trk.observations()["prn_count"][0]) == [1, 2, 3, 4, 5]
    trk.close()


def _ephemeris_end_to_end(n, fs, chans, seconds, seed, block_ms=1000):
    """chans: (sv, doppler, code_phase, carrier_phase, amplitude, subframes, first_bit_ms).  Tracks them through
    TrackerBank in blocks, then integrate_bits, decode_subframes, parse_subframes and observations after every block."""
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
    blocks = []
    for k0 in range(0, seconds * 1000, block_ms):
        x = nav.synth_lnav_iq(seed, n, fs, k0, block_ms, iq_chans, sigma=0.01)
        tt = np.array([t.chunk_times(k, fs, n) for k in range(k0, k0 + block_ms)])
        recs = bank.process(x, tt[:, 0])
        bits = bank.integrate_bits(tt[:, 0], tt[:, 1])
        sub = bank.decode_subframes()
        parsed = bank.parse_subframes()
        blocks.append((recs["lost"].copy(), bits, sub, parsed, bank.observations()))
    return bank, blocks


def _check_end_to_end(bank, blocks, ephs, block_ms, planted):
    """planted[c]: the channel's transmitted subframes.  A subframe the decoder took from a coincidental preamble pair in
    the data (as the reference can) is not one of them; every one that is must parse to the planted values."""
    svs = [orb.OrbitOracle() for _ in ephs]
    words = [{orb.words_of(sf) for sf in p} for p in planted]
    worst = [0.0, 0.0]
    n_sub = [0] * len(ephs)
    for lost, bits, sub, parsed, obs in blocks:
        for c, eph in enumerate(ephs):
            sent = {float(e["trailing_edge_receiver_timestamp"]) for e in sub[c]
                    if e["kind"] == 0 and tuple(int(w) for w in e["words"]) in words[c]}
            for sf, _, te, ms in parsed[c]:
                if te not in sent:
                    continue
                k = sf.subframe_id.value
                n_sub[c] += 1
                if k in (1, 2, 3):
                    want = orb.planted_values(k, eph)
                    got = {1: lambda s: [s.estimated_group_delay_differential, s.t_oc, s.a_f2, s.a_f1, s.a_f0],
                           2: lambda s: [s.correction_to_orbital_radius_sin, s.mean_motion_difference_from_computed_value,
                                         s.mean_anomaly_at_reference_time, s.correction_to_latitude_cos, s.eccentricity,
                                         s.correction_to_latitude_sin, s.sqrt_semi_major_axis, s.reference_time_ephemeris],
                           3: lambda s: [s.correction_to_inclination_angle_cos, s.longitude_of_ascending_node,
                                         s.correction_to_inclination_angle_sin, s.inclination_angle,
                                         s.correction_to_orbital_radius_cos, s.argument_of_perigee, s.rate_of_right_ascension,
                                         s.rate_of_inclination_angle]}[k](sf)
                    assert got == want
                if k == 1:
                    assert sf.week_num == eph["wn"] + 2048
            # the oracle fed the device's own subframe events, each at its bit's millisecond
            events = [(int(e["kind"]), tuple(int(w) for w in e["words"]), float(e["trailing_edge_receiver_timestamp"]),
                       int(bits[c][int(e["bit_index"])]["ms_index"])) for e in sub[c]]
            drops = [m for kind, _, _, m in events if kind == nav.KIND_CANNOT] + list(np.flatnonzero(lost[c])[:1])
            drop = int(min(drops)) if drops else -1
            _, want = orb.run_call(svs[c], events, drop, block_ms)
            want = np.array([[w[0], w[2], w[3], w[4], w[5], w[6]] for w in want])
            u, m = orb.compare_observations(_rows(obs[c]), want)
            worst = [max(worst[0], u), max(worst[1], m)]
    # Every channel's observations equal the oracle's above, lost lock and false subframe locks included.  Those depend
    # on the synthetic signal and the data (a channel can lose lock, or the decoder can lock onto a preamble pair in the
    # data, as the reference's can), so the planted values are checked on the subframes that did come through, and the
    # positions on the channels that end tracked with a full set.
    assert max(n_sub) >= 5, n_sub
    kept = [c for c in range(len(ephs)) if not blocks[-1][0][c].any() and (blocks[-1][4][c]["flags"] & orb.OBS_COMPLETE).all()]
    assert kept
    for c in kept:
        fin = blocks[-1][4][c]
        assert (fin["flags"] & orb.OBS_COMPLETE).all() and (fin["flags"] & orb.OBS_TIMING).all()
        r = np.sqrt(fin["x"] ** 2 + fin["y"] ** 2 + fin["z"] ** 2)
        assert ((r > 2.4e7) & (r < 2.9e7)).all()
    print(f"true subframes per channel {n_sub}, channels with positions {kept}; worst time of week {worst[0]:.1f} ulp, "
          f"worst ECEF {worst[1]:.3g} m")


def test_ephemerides_behind_the_tracking_kernel():
    """4 channels x 48 s at 2.046 Msps carrying planted ephemerides, in 1-s calls (state carried across calls)."""
    rng = np.random.default_rng(3)  # the signal parameters of the subframe decoding test, which track throughout
    erng = np.random.default_rng(11)
    chans, ephs, planted = [], [], []
    for i, sv in enumerate((5, 12, 19, 27)):
        eph = orb.realistic_ephemeris(erng, sv)
        ephs.append(eph)
        sfs = orb.ephemeris_subframes(eph, 9, first_id=1 + i, tow0=20000 + 50 * i, seed=i)
        planted.append(sfs)
        chans.append((sv, float(rng.integers(-4000, 4000)) + 0.3, int(rng.integers(0, N)), float(rng.uniform(0, 6)), 0.004,
                      sfs, int(rng.integers(0, 20))))
    bank, blocks = _ephemeris_end_to_end(N, FS, chans, 48, seed=9)
    _check_end_to_end(bank, blocks, ephs, 1000, planted)
    bank.native.close()


def test_ephemerides_behind_the_tracking_kernel_4092():
    """1 channel x 48 s at 4.092 Msps, with the week edge in the planted toe so that tk wraps."""
    rng = np.random.default_rng(13)
    eph = orb.realistic_ephemeris(rng, 14)
    eph["toe"] = eph["toc"] = 37799
    sfs = orb.ephemeris_subframes(eph, 9, first_id=1, tow0=3, seed=5)
    chans = [(14, -1733.3, 1501, 2.0, 0.004, sfs, 11)]
    bank, blocks = _ephemeris_end_to_end(4092, 4092000, chans, 48, seed=14, block_ms=2000)
    _check_end_to_end(bank, blocks, [eph], 2000, [sfs])
    bank.native.close()
