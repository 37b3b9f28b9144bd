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


# Late starts, gaps and long stream times: the 6-second check compares a chunk's start time with the time of the last check,
# which starts at 0 (tracker.py:221-222, :370-374).  name -> (start time of ms 0, ms of each nudge, ms the lock is lost at)
LATE = {"join55": (5.5, [500], -1), "join6": (6.0, [6000], -1), "join575_noise": (5.75, [], 250), "gap": (0.0, [600], -1),
        "hour": (3599.5, [], 6000), "day": (86399.5, [], 6000)}


def test_late_cases_have_the_edges_they_are_named_for():
    """join55: the 6.0-s check at ms 500 sees 501 peaks and nudges; join6: the check runs on the first millisecond (one
    peak, nothing to do) and nudges at 12.0 s; join575_noise: lost at 6.0 s after 251 peaks; gap: 7 s missing after
    ms 599, the check fires on ms 600; hour / day: the reference loop cannot hold lock at such stream times (each Doppler
    update moves the wiped-off phase by 2 pi df t) and is lost at the second check."""
    for name, (t0, nudges, lost_at) in LATE.items():
        z, _, _, _, _, tt = load_tracker_case(name)
        rows = z["rows"]
        assert tt[0, 0] == t0 and int(z["lost_at"]) == lost_at and len(rows) == (lost_at if lost_at >= 0 else int(z["n_ms"]))
        assert list(np.flatnonzero(rows[:, 6] != rows[:, 12])) == nudges, name
        assert all(abs(rows[k, 6] - rows[k, 12]) == 5.0 for k in nudges)
    tt = load_tracker_case("join55")[5]
    assert tt[500, 0] == 6.0 and tt[499, 0] < 6.0
    tt = load_tracker_case("join6")[5]
    assert tt[0, 0] == 6.0 and tt[6000, 0] == 12.0
    tt = load_tracker_case("gap")[5]
    assert tt[600, 0] - tt[599, 0] > 7.0 and np.all(np.diff(tt[:600, 0]) < 0.0011) and np.all(np.diff(tt[600:, 0]) < 0.0011)


@pytest.mark.parametrize("name,limit", [("short", 700), ("long", 1200), ("fs4", 500), ("adjust", 6100)] +
                         [(name, 6100) for name in LATE])
def test_oracle_tracker_bit_exact_with_reference(name, limit):
    """fs4: 4.092 Msps, where the reference keeps its hard-wired 2046 (tracker.py:301-303, :319; SURVEY F12)."""
    z, ch, x, n, fs, tt = load_tracker_case(name)
    init = z["init"]
    tr = t.TrackerOracle(ch[0], init[0], init[1], int(init[2]), fs, n)
    for k in range(min(limit, len(z["rows"]))):
        r = tr.step(x[k * n:(k + 1) * n], *tt[k])
        assert np.array_equal(oracle_row(tr, r), z["rows"][k]), k
    if name == "adjust":  # the 6-second nudge fired: histories hold the value before it, current_* the value after
        assert z["rows"][6000, 6] - z["rows"][6000, 12] == 5.0 and z["rows"][6000, 7] != z["rows"][6000, 13]
    lost_at = int(z["lost_at"])
    if 0 <= lost_at < limit:  # tracker.py:378 raised on this millisecond
        with pytest.raises(t.LostLock):
            tr.step(x[lost_at * n:(lost_at + 1) * n], *tt[lost_at])


@pytest.mark.parametrize("name", ["short", "long", "noise"] + list(LATE))
def test_scalar_loop_teacher_forced(emu_lib, name):
    """track_update (DLL, PLL, is_locked with sliding sums, 6-s constellation check) fed the oracle's per-ms E/L/peak
    reproduces the reference's Doppler / phase / code-phase / lock-loss trajectory."""
    assert TRACK_REC.itemsize == 112
    z, ch, x, n, fs, tt = load_tracker_case(name)
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
        a, b = tt[k]
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
    assert lost_at == int(z["lost_at"])
    if name == "noise":
        assert lost_at == 6000
    elif lost_at < 0:
        assert locked_ref > 0


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
