"""k_velocity_fixes (velocity.cu) at every call edge and on each of its three branches: the record's four rows, every
ready row in the world model's order (the least-squares mode), and the geodetic position alone when the ready count
disagrees with the fix record's n_ready.

The recorded fix timelines (fix.npz, fix_repair.npz) in the reference mode, and the scripted six-channel timeline and
`five` in the least-squares mode, are re-cut (fix_support.resplit / edge_splits) so that every millisecond where the fix
plan decides something falls at in-call index 0, 1, 127, 128 and 129, last in its call and alone in a 1-ms call, and run
in calls of 127, 128 and 129 ms.  Dopplers are planted from each solved fix's geometry (test_gpu_velocity.planted) and
every record is checked by test_gpu_velocity.compare against the host core and the oracle.  The rows of a fix over
more than four satellites are taken from the fix oracle's world-model order at that millisecond (OracleTimeline), not
from the device's receiver_state()."""
import os

import numpy as np
import pytest

import fix_lsq_oracle as lo
import velocity_oracle as vo
from fix_support import OracleTimeline, call_starts, edge_ms, edge_splits, parse_events, resplit, scripted_timeline, \
    sweep_cuts
from gpu_support import make_engine
from oracle import fix_oracle as fx
from test_gpu_velocity import HOST_DEG, HOST_M, compare, expected, planted
from velocity_support import velocity_emulator

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, FS = 2046, 2046000
TIMELINES = [("fix", n, "reference") for n in ("realistic", "three", "gate", "lost", "five", "raise")] + \
            [("fix_repair", n, "reference") for n in ("gap_mid", "gap_two", "gap_back", "gap_first", "gap_carry",
                                                      "gap_five", "gap_raise", "singular")] + \
            [(None, "scripted", "least_squares"), ("fix", "five", "least_squares")]
IDS = [f"{n}-{s}" for _, n, s in TIMELINES]
PLACEMENTS = (0, 1, 127, 128, 129, "last", "alone")


@pytest.fixture(scope="module")
def engine(native_lib):
    e = make_engine(FS, N)
    yield e
    e.close()


@pytest.fixture(scope="module")
def emu():
    return velocity_emulator()


def _timeline(group, name, solver):
    if group is None:
        calls = scripted_timeline()
    else:
        calls = fx.golden_calls(np.load(os.path.join(ROOT, "tests", "golden", f"{group}.npz")), name)
    tl = OracleTimeline(lo if solver == "least_squares" else fx, calls)
    return calls, tl


def _order_at(tl, m):
    """The world model's order at the end of global millisecond m, from the oracle."""
    return [ch for t, ch in tl.touches if t <= m]


def _run_split(engine, emu, split, tl, solver, what):
    """One split on one tracker; returns the solved records checked and those over more than four rows."""
    import torch

    from gypsum_b200 import _native

    n_ch = len(split[0][1])
    trk = _native.Tracker(engine, list(range(n_ch)), [0.0] * n_ch, [0.0] * n_ch, [0] * n_ch)
    trk.set_fix_solver(solver)
    sv, n_many, n_checked = None, 0, 0
    starts, _ = call_starts(split)
    for s, (rx, chans) in zip(starts, split):
        parse_events(trk, chans, len(rx))
        fixes = trk.position_fixes(rx)
        obs = trk.observations()
        params, sv = vo.params_timeline(chans, len(rx), sv)
        solved = np.flatnonzero(fixes["status"] == fx.FIX_SOLVED)
        # the rows of each solved fix: the record's four, or the ready channels in the oracle's order at m
        orders = {m: _order_at(tl, s + m) for m in solved}
        dev_order = trk.receiver_state()["order"]
        for m in solved:
            if fixes[m]["n_ready"] != 4:
                mine = [c for c in orders[m] if (obs[c, m]["flags"] & 6) == 6]
                assert mine == [c for c in dev_order if (obs[c, m]["flags"] & 6) == 6], (what, s, m)
                assert len(mine) == fixes[m]["n_ready"], (what, s, m)
                n_many += 1
        dopp = np.zeros(obs.shape)
        for m in solved:  # planted per millisecond with that millisecond's oracle order
            dopp[:, m] = planted(fixes[m:m + 1], obs[:, m:m + 1], params[:, m:m + 1], orders[m])[:, 0]
        size = len(rx) * vo.VELOCITY_DTYPE.itemsize
        d = torch.from_numpy(dopp).cuda()
        buf = torch.full((size + vo.VELOCITY_DTYPE.itemsize,), 0xFF, dtype=torch.uint8, device="cuda")
        trk.velocity_fixes_device(buf.data_ptr(), d.data_ptr())
        torch.cuda.synchronize()
        raw = buf.cpu().numpy()
        assert (raw[size:] == 0xFF).all(), (what, s)  # the guard record
        got = raw[:size].view(vo.VELOCITY_DTYPE)
        assert got.tobytes() == trk.velocity_fixes(d.data_ptr()).tobytes(), (what, s)
        host = np.zeros(len(rx), dtype=vo.VELOCITY_DTYPE)
        orc = host.copy()
        for m in solved:
            h, o = expected(emu, fixes[m:m + 1], obs[:, m:m + 1], params[:, m:m + 1], dopp[:, m:m + 1], orders[m])
            host[m], orc[m] = h[0], o[0]
        compare(got, fixes, host, orc, sample=set(solved.tolist()), plant=True)
        n_checked += len(solved)
    trk.close()
    return n_checked, n_many


@pytest.mark.parametrize("group,name,solver", TIMELINES, ids=IDS)
def test_edge_placements_and_call_sizes(engine, emu, group, name, solver):
    """Every fix-plan edge at in-call index 0, 1, 127, 128 and 129, last and alone, and calls of 127, 128 and 129 ms:
    every record against the host core and the oracle, planted velocity and drift recovered."""
    calls, tl = _timeline(group, name, solver)
    edges = edge_ms(calls, tl)
    _, total = call_starts(calls)
    runs = [(p, cuts, on) for p, cuts, on in edge_splits(calls, edges, PLACEMENTS)]
    runs += [(f"{w}-ms calls", sweep_cuts(calls, 0, w), []) for w in (127, 128, 129)]
    placed = {p: 0 for p in PLACEMENTS}
    n_checked = n_many = 0
    for p, cuts, on in runs:
        split = resplit(calls, cuts)
        starts, _ = call_starts(split)
        ends = starts[1:] + [total]
        for e in on:
            k = max(i for i, st in enumerate(starts) if st <= e)
            assert (e == ends[k] - 1) if p == "last" else (starts[k] == e and ends[k] == e + 1) if p == "alone" \
                else (e - starts[k] == p), (p, e)
            placed[p] += 1
        c, mny = _run_split(engine, emu, split, tl, solver, (name, p))
        n_checked, n_many = n_checked + c, n_many + mny
    assert placed["last"] == placed["alone"] == placed[0] == len(edges)
    if name == "scripted" or (name == "five" and solver == "least_squares"):
        assert n_many > 0
    print(f"{name} ({solver}): {len(edges)} edges, placed {placed}; {len(runs)} splits, {n_checked} records checked, "
          f"{n_many} over more than four rows")


def _solved_call(engine, group, name, solver="reference"):
    """A tracker after the first call of a timeline with a solved fix: (tracker, fixes, observations, order)."""
    from gypsum_b200 import _native

    calls, _ = _timeline(group, name, solver)
    n_ch = len(calls[0][1])
    trk = _native.Tracker(engine, list(range(n_ch)), [0.0] * n_ch, [0.0] * n_ch, [0] * n_ch)
    trk.set_fix_solver(solver)
    for rx, chans in calls:
        parse_events(trk, chans, len(rx))
        fixes = trk.position_fixes(rx)
        if (fixes["status"] == fx.FIX_SOLVED).any():
            return trk, fixes, trk.observations(), trk.receiver_state()["order"]
    raise AssertionError("no solved fix")


@pytest.mark.parametrize("group,name,solver", [("fix", "realistic", "reference"), (None, "scripted", "least_squares")],
                         ids=["realistic", "scripted"])
def test_ready_count_disagrees(engine, emu, group, name, solver):
    """Caller fix records whose n_ready disagrees with the ready rows: status 2, n_rows the ready count, velocity and
    drift NaN, the geodetic position the host core's; the records left alone are those of the kept fixes."""
    import torch

    _, _, geodetic = emu
    trk, fixes, obs, order = _solved_call(engine, group, name, solver)
    d = torch.from_numpy(np.random.default_rng(5).uniform(-3000, 3000, obs.shape)).cuda()
    base = trk.velocity_fixes(d.data_ptr())
    solved = np.flatnonzero(fixes["status"] == fx.FIX_SOLVED)
    bad = solved[::3]
    changed = fixes.copy()
    for i, m in enumerate(bad):
        n = int(fixes[m]["n_ready"])
        changed[m]["n_ready"] = (3, 5, 6, 7)[i % 4] if n == 4 else (n + 1, 14)[i % 2]  # never 4: that takes the record's rows
    fdev = torch.from_numpy(changed.view(np.uint8).copy()).cuda()
    got = trk.velocity_fixes(d.data_ptr(), fdev.data_ptr())
    for m in bad:
        ready = sum((obs[c, m]["flags"] & 6) == 6 for c in order)
        if ready == changed[m]["n_ready"]:
            continue  # n_ready 4 on a fix over four ready rows of the world model
        g = got[m]
        assert g["status"] == vo.VEL_UNSOLVABLE and g["n_rows"] == ready, (m, g["status"], g["n_rows"], ready)
        assert all(np.isnan(g[k]) for k in ("vx", "vy", "vz", "clock_drift")), m
        lat, lon, h = geodetic(fixes[m]["x"], fixes[m]["y"], fixes[m]["z"])
        assert abs(g["latitude_deg"] - lat) <= HOST_DEG and abs(g["longitude_deg"] - lon) <= HOST_DEG, m
        assert abs(g["height"] - h) <= HOST_M, m
    keep = np.setdiff1d(np.arange(len(fixes)), bad)
    assert got[keep].tobytes() == base[keep].tobytes()
    trk.close()


def test_nan_doppler(engine, emu):
    """A NaN Doppler at one (channel, ms) used by a solved fix: status 2 there, every other record unchanged."""
    import torch

    trk, fixes, obs, order = _solved_call(engine, "fix", "realistic")
    d = np.random.default_rng(9).uniform(-3000, 3000, obs.shape)
    base = trk.velocity_fixes(torch.from_numpy(d).cuda().data_ptr())
    solved = np.flatnonzero(fixes["status"] == fx.FIX_SOLVED)
    for m in (solved[0], solved[len(solved) // 2], solved[-1]):
        dn = d.copy()
        dn[int(fixes[m]["channel"][1]), m] = np.nan
        got = trk.velocity_fixes(torch.from_numpy(dn).cuda().data_ptr())
        assert got[m]["status"] == vo.VEL_UNSOLVABLE and all(np.isnan(got[m][k]) for k in ("vx", "vy", "vz")), m
        others = np.setdiff1d(np.arange(len(fixes)), [m])
        assert got[others].tobytes() == base[others].tobytes(), m
    trk.close()
