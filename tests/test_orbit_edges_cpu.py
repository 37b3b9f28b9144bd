"""The orbit edge scenarios of tests/orbit_support.py on the CPU: each reaches the edge it is named for on the oracle's
own output, and the host build of orbit_core.cuh equals the oracle on every one of them (fields, parameter sets and
counts exact, time of week within 1 ulp, ECEF within 1e-4 m).  tests/test_gpu_orbit_edges.py runs the same calls on the
device."""
import numpy as np
import pytest

import orbit_support as os_
from oracle import orbit_oracle as orb

CASES = [(c, m) for c in os_.CHANNELS for m in os_.CALL_MS]


def _check_host(calls, want, what):
    emu = os_.OrbitEmulator(len(calls[0][1]))
    worst = [0.0, 0.0]
    for k, (n_ms, chans) in enumerate(calls):
        for c, (events, drop) in enumerate(chans):
            f, obs, st = emu.call(c, events, drop, n_ms)
            assert np.array_equal(os_.fields_rows(f), want.fields[k][c]), (what, k, c)
            u, m = orb.compare_observations(os_.obs_rows(obs), want.obs[k][c])
            worst = [max(worst[0], u), max(worst[1], m)]
            os_.assert_state(st, want.state[k][c], (what, k, c))
    return worst


@pytest.mark.parametrize("n_ch,n_ms", CASES, ids=[f"{c}ch-{m}ms" for c, m in CASES])
def test_grid_case(n_ch, n_ms):
    """Every channel's scenario reaches its edge on the oracle, and the host build equals the oracle."""
    calls, names = os_.case_calls(n_ch, n_ms)
    want = os_.OracleRun(calls)
    shown = []
    for k, (_, chans) in enumerate(calls[:-1]):
        stride = max(len(ev) for ev, _ in chans)
        for c, (name, (events, drop)) in enumerate(zip(names, chans)):
            prev = None if k == 0 else (int(want.obs[k - 1][c][-1, 4]), bool(int(want.obs[k - 1][c][-1, 5]) & orb.OBS_FROZEN))
            shown += os_.assert_edge(name, events, drop, n_ms, k, want.obs[k][c], want.state[k][c], prev)
            if name == "capacity":
                assert len(events) == stride
            elif name == "short":
                assert len(events) == stride - 1
        if n_ch >= 3:
            assert max(len(ev) for ev, _ in chans) == len(chans[0][0]) and not chans[1][0]
    # the last call has no events: a channel dropped in the call before counts again from 1
    for c, name in enumerate(names):
        cnt = want.obs[-1][c][:, 4]
        frozen = int(want.obs[-2][c][-1, 5]) & orb.OBS_FROZEN
        if calls[-2][1][c][1] >= 0 and not frozen:
            assert list(cnt[:2]) == [1, 2][:n_ms], (name, cnt[:2])
            shown.append("counts from 1 after a drop")
    _check_host(calls, want, (n_ch, n_ms))
    print(f"{n_ch} channels x {n_ms} ms: {sorted(set(shown))}")


def test_grid_reaches_every_edge():
    """Across the grid: subframes at ms 0, 127, 128 and n_ms - 1 for every n_ms, drops at 0, 1, 127, 128 and n_ms - 1,
    every scenario in a one-channel case and with 31 and 32 channels, and full change tables."""
    placed, drops, one = set(), set(), set()
    for n_ch, n_ms in CASES:
        calls, names = os_.case_calls(n_ch, n_ms)
        if n_ch == 1:
            one.add(names[0])
        if n_ch >= 31:
            assert set(os_.SCENARIOS) <= set(names)
        for _, chans in calls:
            for name, (events, drop) in zip(names, chans):
                if name == "placed":
                    placed.update((n_ms, m) for k, _, _, _, m in events if k == os_.SUB)
                if name.startswith("drop_") and drop >= 0:
                    drops.add((n_ms, drop))
    for n_ms in os_.CALL_MS:
        assert {(n_ms, m) for m in (0, 127, 128, n_ms - 1) if m < n_ms} <= placed
    assert {d for _, d in drops} >= {0, 1, 127, 128} and all((m, m - 1) in drops for m in os_.CALL_MS)
    assert len(one) == len([n for n in os_.CHANNELS if n == 1]) * len(os_.CALL_MS)


def test_fix_gate_inside_and_across_calls():
    """The 6000-count gate: left inside a 6100-ms call, and by counts carried across call boundaries."""
    calls = os_.gate_calls()
    want = os_.OracleRun(calls)
    for c, (k, i) in enumerate(os_.GATE_LEFT):
        cnt = np.concatenate([call[c][:, 4] for call in want.obs]).astype(int)
        gate = np.concatenate([(call[c][:, 5].astype(int) & orb.OBS_FIX_GATE) > 0 for call in want.obs])
        at = sum(n for n, _ in calls[:k]) + i
        assert (cnt >= 0).all() and np.array_equal(gate, cnt <= 6000), c
        assert gate[at - 1] and not gate[at] and cnt[at] == 6001, c
        if k > 0:
            assert 0 < i < calls[k][0] and gate[at - i - 1]  # carried into the call under the gate
    _check_host(calls, want, "gate")
