"""k_parse_subframes and k_sv_observations (orbit.cu) at every block, call and change-table edge, through the
explicit-event path of gb200_tracker_parse_subframes.  The scenarios of tests/orbit_support.py (each channel its own;
tests/test_orbit_edges_cpu.py shows on the CPU that each reaches its edge) run on 1, 3, 4, 5, 8, 31 and 32 channels
(partial 4-warp blocks, idle warps) in calls of 1, 127, 128, 129, 256 and 257 ms (the 128-thread observation blocks),
and around the 6000-count fix gate.  Every call against the oracle: fields, event indices, milliseconds, counts, flags,
set masks and parameters exact, time of week within 1 ulp, ECEF within 1e-4 m; and against the host build of the same
core within the same bounds.  Observations also go through observations_device into a 0xFF-filled buffer one channel
row longer: every (channel, ms) written, the guard row untouched."""
import numpy as np
import pytest

import orbit_support as os_
from gpu_support import make_engine
from oracle import orbit_oracle as orb

pytestmark = pytest.mark.gpu
N, FS = 2046, 2046000
CASES = [(c, m) for c in os_.CHANNELS for m in os_.CALL_MS]


@pytest.fixture(scope="module")
def engine(native_lib):
    e = make_engine(FS, N)
    yield e
    e.close()


def _parse(trk, chans, n_ms):
    """One call through device event arrays; returns the fields per channel and the stride."""
    import torch

    from gypsum_b200._native import SUBFRAME_DTYPE

    n_ch = len(chans)
    stride = max(1, max(len(ev) for ev, _ in chans))
    host = np.zeros((n_ch, stride), dtype=SUBFRAME_DTYPE)
    ems = np.zeros((n_ch, stride), dtype=np.int32)
    for c, (events, _) in enumerate(chans):
        for j, (kind, w, t0, t1, m) in enumerate(events):
            host[c, j]["kind"], host[c, j]["words"] = kind, w
            host[c, j]["receiver_timestamp"], host[c, j]["trailing_edge_receiver_timestamp"] = t0, t1
            ems[c, j] = m
    dev = torch.from_numpy(host.view(np.uint8).reshape(n_ch, -1).copy()).cuda()
    counts = np.array([len(ev) for ev, _ in chans], dtype=np.int32)
    drop = np.array([d for _, d in chans], dtype=np.int32)
    return trk.parse_subframes(dev.data_ptr(), counts, stride, ems, drop, n_ms), stride


def _run(engine, calls, what):
    """calls on one tracker, every call checked; returns the oracle's run and the worst (ulp, metres) against it."""
    import torch

    from gypsum_b200 import _native

    n_ch = len(calls[0][1])
    want = os_.OracleRun(calls)
    emu = os_.OrbitEmulator(n_ch)
    trk = _native.Tracker(engine, list(range(n_ch)), [0.0] * n_ch, [0.0] * n_ch, [0] * n_ch)
    size = _native.OBSERVATION_DTYPE.itemsize
    worst = [0.0, 0.0]
    for k, (n_ms, chans) in enumerate(calls):
        fields, stride = _parse(trk, chans, n_ms)
        obs = trk.observations()
        assert obs.shape == (n_ch, n_ms)
        buf = torch.full(((n_ch + 1) * n_ms * size,), 0xFF, dtype=torch.uint8, device="cuda")
        trk.observations_device(buf.data_ptr())
        torch.cuda.synchronize()
        raw = buf.cpu().numpy()
        assert raw[:n_ch * n_ms * size].tobytes() == obs.tobytes(), (what, k)
        assert (raw[n_ch * n_ms * size:] == 0xFF).all(), (what, k)  # the guard row
        for c, (events, drop) in enumerate(chans):
            w = (what, k, c)
            assert np.array_equal(os_.fields_rows(fields[c]), want.fields[k][c]), w
            u, m = orb.compare_observations(os_.obs_rows(obs[c]), want.obs[k][c])
            worst = [max(worst[0], u), max(worst[1], m)]
            st = trk.orbit_state(c)
            os_.assert_state((st["params"], st["set_mask"], st["prn_count"], st["counting"]), want.state[k][c], w)
            hf, ho, _ = emu.call(c, events, drop, n_ms)
            assert np.array_equal(os_.fields_rows(hf), os_.fields_rows(fields[c])), w
            orb.compare_observations(os_.obs_rows(obs[c]), os_.obs_rows(ho))
    trk.close()
    return want, worst


@pytest.mark.parametrize("n_ch,n_ms", CASES, ids=[f"{c}ch-{m}ms" for c, m in CASES])
def test_grid_case(engine, n_ch, n_ms):
    """Each channel's scenario (subframes at ms 0, 127, 128 and n_ms - 1; two and three in one millisecond with kinds 1
    and 2 between; raises at ms 0, at n_ms - 1, after and sharing a millisecond with subframes; drops at 0, 1, 127,
    128 and n_ms - 1 with events at and after them; a change table filled to stride + 2 beside channels with 0 and
    stride - 1 events) in two calls, then a call without events, where dropped channels count again from 1."""
    calls, names = os_.case_calls(n_ch, n_ms)
    want, (u, m) = _run(engine, calls, (n_ch, n_ms))
    for c in range(n_ch):  # a channel dropped in the second call counts from 1 in the third (the device equals want)
        if calls[-2][1][c][1] >= 0 and not int(want.obs[-2][c][-1, 5]) & orb.OBS_FROZEN:
            assert list(want.obs[-1][c][:2, 4]) == [1, 2][:n_ms]
    print(f"{n_ch} channels x {n_ms} ms ({', '.join(sorted(set(names)))}): worst time of week {u:.1f} ulp, "
          f"worst ECEF {m:.3g} m")


def test_fix_gate_inside_and_across_calls(engine):
    """Five channels in calls of 6100, 5990 and 100 ms: the gate left inside the first call, and by counts carried
    across both call boundaries (tests/orbit_support.py GATE_LEFT)."""
    calls = os_.gate_calls()
    want, (u, m) = _run(engine, calls, "gate")
    for c, (k, i) in enumerate(os_.GATE_LEFT):
        flags = want.obs[k][c][:, 5].astype(int)
        assert flags[i - 1] & orb.OBS_FIX_GATE and not flags[i] & orb.OBS_FIX_GATE
    print(f"gate: worst time of week {u:.1f} ulp, worst ECEF {m:.3g} m")
