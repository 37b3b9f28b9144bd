"""Tracking loop, CPU side: the oracle tracker against the live reference's recorded trajectories, and the
product's scalar loop code (gypsum_b200/csrc/tracker_core.cuh, run by the lane emulator) teacher-forced with
the oracle's correlator outputs."""
import ctypes

import numpy as np
import pytest

from oracle import tracker_oracle as t
from tracker_support import load_tracker_case, oracle_row

TRACK_REC = np.dtype([("doppler", "<f8"), ("carrier_phase", "<f8"), ("error", "<f8"), ("disc", "<f8"), ("phase_acc", "<f8"),
                      ("doppler_hist", "<f8"), ("carrier_phase_hist", "<f8"), ("peak_re", "<f4"), ("peak_im", "<f4"), ("strength", "<f4"), ("early_re", "<f4"), ("early_im", "<f4"),
                      ("late_re", "<f4"), ("late_im", "<f4"), ("code_phase", "<i4"), ("symbol", "<i4"), ("locked", "<i4"),
                      ("lost", "<i4"), ("peak_offset", "<i4"), ("pad0", "<i4"), ("pad1", "<i4")])


@pytest.mark.parametrize("name,limit", [("short", 700), ("long", 1200), ("fs4", 500), ("adjust", 6100)])
def test_oracle_tracker_bit_exact_with_reference(name, limit):
    """fs4: 4.092 Msps, where the reference keeps its hard-wired 2046 (tracker.py:301-303, :319; SURVEY F12)."""
    z, ch, x, n, fs = load_tracker_case(name)
    init = z["init"]
    tr = t.TrackerOracle(ch[0], init[0], init[1], int(init[2]), fs, n)
    for k in range(min(limit, len(z["rows"]))):
        a, b = t.chunk_times(k, fs, n)
        r = tr.step(x[k * n:(k + 1) * n], a, b)
        assert np.array_equal(oracle_row(tr, r), z["rows"][k]), k
    if name == "adjust":  # the 6-second nudge fired: histories hold the value before it, current_* the value after
        assert z["rows"][6000, 6] - z["rows"][6000, 12] == 5.0 and z["rows"][6000, 7] != z["rows"][6000, 13]


@pytest.mark.parametrize("name", ["short", "long", "noise"])
def test_scalar_loop_teacher_forced(emu_lib, name):
    """track_update (DLL, PLL, is_locked with sliding sums, 6-s constellation check) fed the oracle's per-ms E/L/peak
    reproduces the reference's Doppler / phase / code-phase / lock-loss trajectory."""
    assert TRACK_REC.itemsize == 112
    z, ch, x, n, fs = load_tracker_case(name)
    init = z["init"]
    tr = t.TrackerOracle(ch[0], init[0], init[1], int(init[2]), fs, n)
    st = ctypes.create_string_buffer(emu_lib.emu_track_state_size())
    emu_lib.emu_track_init.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_int]
    emu_lib.emu_track_update.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_int, ctypes.c_double,
                                         ctypes.c_double, ctypes.c_void_p]
    emu_lib.emu_track_init(st, ch[0] - 1, float(init[0]), float(init[1]), int(init[2]))
    rec = np.zeros(1, TRACK_REC)
    rows = z["rows"]
    lost_at = -1
    locked_ref = locked_mine = 0
    for k in range(int(z["n_ms"])):
        a, b = t.chunk_times(k, fs, n)
        raised = False
        try:
            r = tr.step(x[k * n:(k + 1) * n], a, b)
        except t.LostLock as exc:
            r, raised = exc.args[0], True
        elp = np.array([r["early"].real, r["early"].imag, r["late"].real, r["late"].imag, r["peak"].real, r["peak"].imag],
                       dtype=np.float32)
        emu_lib.emu_track_update(st, elp.ctypes.data, np.float32(r["strength"]), r["peak_offset"], a, float(fs), rec.ctypes.data)
        if raised:  # tracker.py:378: the scalar loop must flag the same millisecond
            assert rec["lost"][0] == 1
            lost_at = k
            break
        g = rows[k]
        assert rec["code_phase"][0] == int(g[8]) and rec["symbol"][0] == int(g[3]), k
        assert abs(rec["doppler"][0] - g[6]) <= 1e-6 * max(1.0, abs(g[6])), k
        d = abs(rec["carrier_phase"][0] - g[7])
        assert min(d, 2 * np.pi - d) <= 1e-5, k
        assert abs(rec["error"][0] - g[4]) <= 2e-6 * max(1.0, abs(g[4])), k
        assert rec["locked"][0] == int(r["locked"]), k
        assert rec["lost"][0] == 0
        locked_ref += int(r["locked"])
    if name == "noise":
        assert lost_at == int(z["lost_at"]) == 6000
    else:
        assert lost_at == -1 and locked_ref > 0


def test_fast_angle_test_decides_like_the_reference_arithmetic(emu_lib):
    """track_rot_ok_fast (|mi| vs tan(6 deg)|mr| with a guard band, experimental) == track_rot_ok (the atan2 / modulo
    arithmetic of tracker.py:191-197) everywhere: random directions, a dense sweep across both 6-degree boundaries in all
    four quadrants, the axes, the origin, NaN and infinities."""
    f = emu_lib.emu_track_rot_ok
    f.argtypes = [ctypes.c_double, ctypes.c_double, ctypes.c_int]
    rng = np.random.default_rng(0)
    cases = [(0.0, 0.0), (-0.0, 0.0), (1.0, 0.0), (-1.0, 0.0), (0.0, 1.0), (0.0, -1.0), (float("nan"), 1.0), (1.0, float("nan")),
             (float("inf"), 1.0), (-3.0, float("inf"))]
    cases += [tuple(v) for v in rng.standard_normal((20000, 2)) * np.exp(rng.uniform(-20, 20, (20000, 1)))]
    for base in (6.0, 174.0, 186.0, 354.0):
        for d in np.linspace(-0.02, 0.02, 4001):
            a = np.radians(base + d)
            r = np.exp(rng.uniform(-5, 5))
            cases.append((r * np.cos(a), r * np.sin(a)))
    got_true = 0
    for mr, mi in cases:
        slow, fast = f(mr, mi, 0), f(mr, mi, 1)
        assert slow == fast, (mr, mi)
        got_true += slow
    assert 0 < got_true < len(cases)
