"""The position-fix kernels' serial repair on the device (fix.cu through gb200_tracker_position_fixes), on the timelines
with a receiver-clock jump recorded from the live reference's GpsWorldModel (tests/golden/fix_repair.npz).  On each of
them the chain check misses and k_fix_repair runs; fx.device_passes over the host core and the device's own
observations predicts every record and the repair count exactly (tests/test_fix_repair_cpu.py runs the same model on
the CPU)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import fix_oracle as fx
from oracle import gypsum_oracle as o

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "fix_repair.npz")
GAPS = ["gap_mid", "gap_two", "gap_back", "gap_first", "gap_carry", "gap_five", "gap_raise"]
N, FS = 2046, 2046000
# DESIGN.md §6: the bounds of tests/test_gpu_fix.py
POS_M, BIAS_S, SLIDE_ULPS = 2e-6, 1e-14, 4


def slide_tol(s):
    return SLIDE_ULPS * 2.0 ** -52 * np.abs(s)


@pytest.fixture(scope="module")
def engine(native_lib):
    from gypsum_b200 import _native

    e = _native.Engine(FS, N)
    e.set_replicas(np.stack([o.ca_code(sv) for sv in range(1, 33)]).astype(np.uint8))
    yield e
    e.close()


@pytest.fixture(scope="module")
def fix_emu(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "emu", "fix_emu.cu")
    out = str(tmp_path_factory.mktemp("fix_emu") / "libfixemu.so")
    subprocess.run(["nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-o", out, src], check=True,
                   capture_output=True)
    lib = C.CDLL(out)
    lib.fix_emu_compute.restype = C.c_int
    lib.fix_emu_compute.argtypes = [C.c_void_p, C.c_double, C.c_double, C.c_void_p]

    def compute(rows, rx, slide):
        r = np.ascontiguousarray(rows, dtype=np.float64).reshape(4, 4)
        out = np.zeros(1, dtype=fx.FIX_DTYPE)
        lib.fix_emu_compute(r.ctypes.data, float(rx), float(slide), out.ctypes.data)
        return out[0]

    return compute


def _parse(trk, chans, n_ms):
    """chans: [(events [(kind, words, trailing_edge, ms)], drop_ms)] through device event arrays."""
    import torch

    from gypsum_b200._native import SUBFRAME_DTYPE

    n_ch = len(chans)
    stride = max(1, max(len(ev) for ev, _ in chans))
    host = np.zeros((n_ch, stride), dtype=SUBFRAME_DTYPE)
    ems = np.zeros((n_ch, stride), dtype=np.int32)
    counts = np.array([len(ev) for ev, _ in chans], dtype=np.int32)
    for c, (events, _) in enumerate(chans):
        for j, (kind, w, te, m) in enumerate(events):
            host[c, j]["kind"], host[c, j]["words"], host[c, j]["trailing_edge_receiver_timestamp"] = kind, w, te
            ems[c, j] = m
    dev = torch.from_numpy(host.view(np.uint8).reshape(n_ch, -1)).cuda()
    trk.parse_subframes(dev.data_ptr(), counts, stride, ems, np.array([d for _, d in chans], dtype=np.int32), n_ms)


def _run(engine, name, device_out=False):
    """The timeline call after call; per call the records, the device's observations and receiver_state()."""
    import torch

    from gypsum_b200 import _native

    z = np.load(GOLDEN)
    calls = fx.golden_calls(z, name)
    n_ch = len(calls[0][1])
    trk = _native.Tracker(engine, list(range(n_ch)), [0.0] * n_ch, [0.0] * n_ch, [0] * n_ch)
    out = []
    for rx, chans in calls:
        _parse(trk, chans, len(rx))
        if device_out:
            dev = torch.empty(len(rx) * _native.FIX_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
            trk.position_fixes_device(rx, dev.data_ptr())
            torch.cuda.synchronize()
            rec = dev.cpu().numpy().view(_native.FIX_DTYPE).copy()
        else:
            rec = trk.position_fixes(rx)
        out.append((rec, trk.observations(), trk.receiver_state()))
    trk.close()
    return z, calls, out


def _rows(obs, channels, m):
    return [(obs[ch, m]["tow"], obs[ch, m]["x"], obs[ch, m]["y"], obs[ch, m]["z"]) for ch in channels]


@pytest.mark.parametrize("name", GAPS + ["singular"])
def test_repair_on_the_device(engine, fix_emu, name):
    """Against the recording and the oracle: status, ready count and rows exact; slides and round-0 pseudoranges within
    4 ulp, clock bias within 1e-14 s, position within 2e-6 m.  Against the model of the passes on the device's own
    observations: every record bit for bit and receiver_state()["repaired"] after every call.  Every solved record is
    the host core's fix from its own slide_in; a fix that does not start a segment starts from the slide the fix
    before it left, exactly where the repair ran and within 4 ulp elsewhere; slide, order and stopped are the
    oracle's."""
    z, calls, out = _run(engine, name)
    rcv = fx.ReceiverOracle(len(calls[0][1]))
    carried, repaired, worst = None, 0, [0.0, 0.0, 0.0]
    for c, ((rx, chans), (got, obs, state)) in enumerate(zip(calls, out)):
        want = rcv.call(chans, rx)
        rec = fx.golden_fix_rows(z, name, c)
        assert np.array_equal(got["status"], rec[:, 3].astype(int))
        assert np.array_equal(got["n_ready"], want["n_ready"]) and np.array_equal(got["channel"], want["channel"])
        fixing = np.flatnonzero(np.isin(want["status"], [fx.FIX_SOLVED, fx.FIX_RAISED]))
        solved = np.flatnonzero(want["status"] == fx.FIX_SOLVED)
        for k in ("slide_in", "slide_out"):
            d = np.abs(got[k][fixing] - want[k][fixing])
            assert (d <= slide_tol(want[k][fixing])).all(), k
            worst[0] = max([worst[0], *d])
        if len(solved):
            d = np.abs(got["pseudorange"][solved] - want["pseudorange"][solved]).max(axis=1)
            assert (d <= slide_tol(want["slide_in"][solved])).all()
            worst[1] = max(worst[1], float(np.abs(got["clock_bias"][solved] - want["clock_bias"][solved]).max()))
            worst[2] = max([worst[2], *(float(np.abs(got[k][solved] - want[k][solved]).max()) for k in "xyz")])
        assert worst[1] <= BIAS_S and worst[2] <= POS_M, worst
        assert np.isnan(got["x"][got["status"] != fx.FIX_SOLVED]).all()
        # the model of the passes, on the rows the device observed
        rows = {m: _rows(obs, want[m]["channel"], m) for m in fixing if want[m]["n_ready"] == 4}
        model = fx.device_passes(fix_emu, want, rows, rcv.resets, carried)
        carried = model["slide"]
        assert sorted(model["out"]) == list(fixing)
        for m in fixing:  # the numbers (slides, solution, pseudoranges) of a solved record; the slides of a raise
            p = model["out"][m]
            assert p["status"] == got[m]["status"] and p["slide_in"] == got[m]["slide_in"], m
            assert p["slide_out"] == got[m]["slide_out"], m
            if m in solved:
                assert p.tobytes()[:88] == got[m].tobytes()[:88], m
        for m in solved:
            host = fix_emu(rows[m], got[m]["receiver_timestamp"], got[m]["slide_in"])
            assert host.tobytes()[:88] == got[m].tobytes()[:88] and host["status"] == got[m]["status"], m
        repaired += len(model["repaired"])
        assert state["repaired"] == repaired, (c, state["repaired"], repaired)
        # the chain relation
        for a, b in zip(fixing[:-1], fixing[1:]):
            if b in rcv.resets or any(r in rcv.resets for r in range(a + 1, b)):
                assert got[b]["slide_in"] == rcv.resets[max(r for r in rcv.resets if r <= b)]
            elif model["first_miss"] is not None and b > model["first_miss"]:
                assert got[b]["slide_in"] == got[a]["slide_out"], b
            else:
                assert abs(got[b]["slide_in"] - got[a]["slide_out"]) <= slide_tol(got[a]["slide_out"]), b
        print(f"{name} call {c}: first miss {model['first_miss']}, repaired {len(model['repaired'])}, "
              f"receiver_state repaired {state['repaired']}")
    st = out[-1][2]
    assert st["order"] == rcv.order and st["stopped"] == rcv.stopped
    if rcv.slide is not None:
        assert abs(st["slide"] - rcv.slide) <= slide_tol(rcv.slide)
    if name in GAPS:
        assert out[0][2]["repaired"] > 0
    print(f"{name}: worst slide / pseudorange {worst[0]:.3g} s, clock bias {worst[1]:.3g} s, position {worst[2]:.3g} m")


def test_carried_slide_needs_no_repair(engine):
    """gap_carry repairs to the end of call 0; call 1 continues from the repaired slide and repairs nothing."""
    _, _, out = _run(engine, "gap_carry")
    (first, _, s0), (second, _, s1) = out
    assert s0["repaired"] > 0 and s1["repaired"] == s0["repaired"]
    assert (first["status"][-100:] == fx.FIX_SOLVED).all() and second["status"][0] == fx.FIX_SOLVED
    assert second[0]["slide_in"] == first[-1]["slide_out"]


def test_gap_five_stops_at_the_raise(engine):
    z, _, out = _run(engine, "gap_five")
    got, _, state = out[0]
    assert np.flatnonzero(got["status"] == fx.FIX_RAISED).tolist() == [400]
    assert (got["status"][401:] == fx.FIX_STOPPED).all() and (out[1][0]["status"] == fx.FIX_STOPPED).all()
    assert state["stopped"] and state["slide"] == got[400]["slide_out"] == fx.golden_fix_rows(z, "gap_five", 0)[400, 6]


def test_singular_matrix_stops_the_receiver(engine):
    """Two channels with one ephemeris: the device raises at the millisecond the reference raised, with the slide the
    reference kept, and stops."""
    z, _, out = _run(engine, "singular")
    want = fx.golden_fix_rows(z, "singular", 0)
    got, _, state = out[0]
    assert np.flatnonzero(got["status"] == fx.FIX_RAISED).tolist() == [300] == np.flatnonzero(want[:, 3] == 2).tolist()
    assert got[300]["slide_out"] == want[300, 6] and np.isnan(got[300]["x"])
    assert (got["status"][301:] == fx.FIX_STOPPED).all() and (out[1][0]["status"] == fx.FIX_STOPPED).all()
    assert state["stopped"] and out[1][2]["stopped"] and state["repaired"] == 0


def test_fixes_device_matches_host_on_a_repair(engine):
    _, _, host = _run(engine, "gap_mid")
    _, _, dev = _run(engine, "gap_mid", device_out=True)
    assert host[0][2]["repaired"] > 0
    for (a, _, _), (b, _, _) in zip(host, dev):
        assert a.tobytes() == b.tobytes()
