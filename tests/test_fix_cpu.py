"""The position fix on the CPU: the oracle against timelines recorded from the live reference's GpsWorldModel
(tests/golden/fix.npz), the device code (fix_core.cuh compiled for the host) against the oracle, the solver on exact
pseudoranges, the measurement that a fix does not depend on the slide it enters with, and the record layout."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from fix_support import BIAS_S, POS_M, fix_emulator, slide_tol
from hostbuild import host_library
from oracle import fix_oracle as fx
from oracle import orbit_oracle as orb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "fix.npz")
TIMELINES = ["realistic", "three", "gate", "lost", "five", "raise"]


def slide_close(a, b) -> bool:
    """Slides (about 3e5 s here) within SLIDE_ULPS units in the last place."""
    return abs(a - b) <= slide_tol(b)


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def fix_emu():
    return fix_emulator()


def oracle_timeline(z, name):
    """The oracle's records of every call, and its rows per (call, ms)."""
    rcv = None
    recs, rows = [], {}
    for c, (rx, chans) in enumerate(fx.golden_calls(z, name)):
        rcv = rcv or fx.ReceiverOracle(len(chans))
        recs.append(rcv.call(chans, rx))
        rows.update({(c, m): r for m, r in rcv.rows.items()})
    return recs, rows, rcv


@pytest.mark.parametrize("name", TIMELINES)
def test_oracle_equals_reference(golden, name):
    """Status, ready count, rows, slides and solution of the oracle equal the reference's bit for bit."""
    recs, _, _ = oracle_timeline(golden, name)
    for c, got in enumerate(recs):
        want = fx.golden_fix_rows(golden, name, c)
        assert np.array_equal(got["status"], want[:, 3].astype(int))
        assert np.array_equal(got["n_ready"], want[:, 4].astype(int))
        assert np.array_equal(got["channel"], want[:, 11:15].astype(int))
        fixing = np.isin(got["status"], [fx.FIX_SOLVED, fx.FIX_RAISED])
        assert np.array_equal(got["slide_in"][fixing], want[fixing, 5])
        assert np.array_equal(got["slide_out"][fixing], want[fixing, 6])
        for k, col in (("clock_bias", 7), ("x", 8), ("y", 9), ("z", 10)):
            assert np.array_equal(got[k], want[:, col], equal_nan=True), k


def test_golden_covers_every_case(golden):
    z = golden
    st = {n: z[f"{n}_fix"][:, 3].astype(int) for n in TIMELINES}
    assert (st["realistic"] == 1).sum() > 2000 and (z["realistic_calls"].size == 2)
    assert (st["three"] == 0).all() and (z["three_fix"][:, 4] == 3).any()
    gate = z["gate_fix"]
    assert (gate[:, 3] == 1).any() and ((gate[:, 0] == 1) & (gate[:, 1] == 301) & (gate[:, 4] == 3)).any()
    lost = z["lost_fix"]
    assert list(lost[lost[:, 3] == 1][0, 11:15]) == [2, 3, 1, 0]  # first-touch order, not channel order
    assert ((lost[:, 0] == 1) & (lost[:, 1] == 800) & (lost[:, 3] == 0)).any()
    assert (st["five"] == 2).sum() == 1 and st["five"][-1] == 3
    assert (st["raise"][500:] == 3).all() and (st["raise"][:500] != 3).all()
    # two resets in one millisecond with different trailing edges: the last channel's wins
    ev = z["realistic_events"]
    same = np.flatnonzero((ev[:, 0] == 0) & (ev[:, 2] == 300))
    assert len(same) == 4 and len(set(ev[same, 5])) == 4 and list(ev[same, 1]) == [0, 1, 2, 3]
    fix = z["realistic_fix"]
    s = fix[(fix[:, 0] == 0) & (fix[:, 1] == 300)][0]
    last = same[-1]
    assert s[5] == orb.parse(tuple(int(w) for w in z["realistic_words"][last]))["tow_seconds"] - ev[last, 5]


def _emu_chain(compute, recs, rows):
    """The host core along the oracle's chain: each fix from the slide the core's previous fix left, or from the
    oracle's slide where a reset set it.  Slides and pseudoranges within SLIDE_ULPS; returns the largest clock-bias
    (s) and position (m) differences."""
    worst_t = worst_m = 0.0
    prev_oracle = prev_emu = None
    for c, rec in enumerate(recs):
        for m in np.flatnonzero(rec["status"] == fx.FIX_SOLVED):
            r = rec[m]
            s = r["slide_in"] if prev_oracle is None or r["slide_in"] != prev_oracle else prev_emu
            got = compute(rows[(c, m)], r["receiver_timestamp"], s)
            assert got["status"] == fx.FIX_SOLVED
            assert slide_close(got["slide_in"], r["slide_in"]) and slide_close(got["slide_out"], r["slide_out"])
            # round 0's pseudoranges: (slide + receiver_timestamp) - tow, differences of numbers of the slide's size
            assert np.abs(got["pseudorange"] - r["pseudorange"]).max() <= slide_tol(r["slide_in"])
            worst_t = max(worst_t, abs(got["clock_bias"] - r["clock_bias"]))
            worst_m = max(worst_m, *(abs(got[k] - r[k]) for k in "xyz"))
            prev_oracle, prev_emu = r["slide_out"], got["slide_out"]
    return worst_t, worst_m


@pytest.mark.parametrize("name", ["realistic", "gate", "lost", "five", "raise"])
def test_device_code_on_host(golden, fix_emu, name):
    """fix_core.cuh compiled for the host, chained as the receiver chains its fixes, against the oracle: slides and
    round-0 pseudoranges within 4 ulp, clock bias within 1e-14 s, position within 2e-6 m."""
    recs, rows, _ = oracle_timeline(golden, name)
    worst_t, worst_m = _emu_chain(fix_emu, recs, rows)
    print(f"{name}: worst clock bias {worst_t:.3g} s, worst position {worst_m:.3g} m")
    assert worst_t <= BIAS_S and worst_m <= POS_M


def _satellites(seed, n=4):
    """Four realistic satellite positions from the orbit oracle."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        sv = orb.OrbitOracle()
        eph = orb.realistic_ephemeris(rng, 3 + k)
        for sf in (1, 2, 3):
            sv.subframe(orb.parse(orb.words_of(orb.encode_subframe(sf, 5000, eph))), 1.0)
        sv.count, sv.counting = 1234 + 7 * k, True
        tow, _ = sv.time_of_week()
        out.append((tow, *sv.position(tow)))
    return out


def test_solver_recovers_a_planted_position(fix_emu):
    """Exact pseudoranges from a planted receiver position and clock bias: the core recovers both."""
    worst = 0.0
    for seed, pos, bias in ((1, (-2.7e6, -4.3e6, 3.9e6), 0.0123), (2, (4.0e6, 3.0e5, 4.9e6), -0.071),
                            (3, (1.1e6, -6.2e6, 1.0e5), 0.0)):
        sats = _satellites(seed)
        # slide 0: a slide of 4e5 s would round the pseudoranges to 6e-11 s (1.7 cm), as the reference's does
        rx, slide = 0.5, 0.0
        rows = []
        for _, x, y, z in sats:
            rng_ = np.sqrt((pos[0] - x) ** 2 + (pos[1] - y) ** 2 + (pos[2] - z) ** 2)
            rows.append(((slide + rx) - (rng_ / fx.SPEED_OF_LIGHT + bias), x, y, z))
        got = fix_emu(rows, rx, slide)
        assert got["status"] == fx.FIX_SOLVED
        err = max(abs(got[k] - p) for k, p in zip("xyz", pos))
        worst = max(worst, err)
        assert err <= POS_M, err
        # round 0 finds the bias, the slide absorbs it, and rounds 1-4 find nothing left
        assert abs(got["slide_out"] - (slide - bias)) <= BIAS_S and abs(got["clock_bias"]) <= BIAS_S
        ora = fx.compute_position(rows, rx, slide)
        assert max(abs(a - b) for a, b in zip(ora[2], pos)) <= POS_M
    print(f"planted position recovered within {worst:.3g} m")


@pytest.mark.parametrize("name", ["realistic", "gate", "lost", "five", "raise"])
def test_fix_from_the_segment_slide_equals_the_chained_fix(golden, fix_emu, name):
    """What the two device passes rest on: at every fixing millisecond of the recorded chains, the fix from the slide
    its segment's reset left (pass 1) equals the fix from the slide the previous fix left (the chain)."""
    recs, rows, _ = oracle_timeline(golden, name)
    worst_t = worst_m = 0.0
    prev_out = base = None
    for c, rec in enumerate(recs):
        for m in np.flatnonzero(rec["status"] == fx.FIX_SOLVED):
            r = rec[m]
            if prev_out is None or r["slide_in"] != prev_out:
                base = r["slide_in"]  # a reset set the slide here
            a = fix_emu(rows[(c, m)], r["receiver_timestamp"], base)
            b = fix_emu(rows[(c, m)], r["receiver_timestamp"], r["slide_in"])
            assert a["slide_out"] == b["slide_out"]  # what the device's chain check (fix_same_slide) relies on
            worst_t = max(worst_t, abs(a["clock_bias"] - b["clock_bias"]))
            worst_m = max(worst_m, *(abs(a[k] - b[k]) for k in "xyz"))
            prev_out = r["slide_out"]
    print(f"{name}: segment slide vs chained slide: clock bias {worst_t:.3g} s, position {worst_m:.3g} m")
    assert worst_t <= BIAS_S and worst_m <= POS_M


@pytest.mark.parametrize("name", ["realistic", "gate", "lost"])
def test_fix_against_its_entering_slide(golden, fix_emu, name):
    """F_m(s) against F_m(s + d) for d up to 0.1 s, on every 7th chained fix of the recorded timelines and on
    synthetic cases, on the host core (and on numpy's solve for a subset).  Measured: up to d = 0.07 s the slide a fix
    leaves and its solution do not depend on the slide it entered with; at d = 0.1 s, or a negative d at a reset, Newton
    can reach the other root of the squared-range equations.  So the device does not rely on independence: every fix
    checks the chain, and a miss runs the chain serially (k_fix_repair, DESIGN.md §8c)."""
    recs, rows, _ = oracle_timeline(golden, name)
    cases = [(rows[(c, m)], rec[m]["receiver_timestamp"], rec[m]["slide_in"])
             for c, rec in enumerate(recs) for m in np.flatnonzero(rec["status"] == fx.FIX_SOLVED)[::7]]
    for seed in range(4):
        sats = _satellites(10 + seed)
        cases.append((sats, 3.0 + seed, sats[0][0] - 0.07 - (3.0 + seed)))
    spread = {}
    for d in (1e-9, 3e-8, 1e-6, 1e-3, 0.01, 0.03, 0.05, 0.07, 0.1):
        worst_s = worst_t = worst_m = 0.0
        for rows_, rx, s in cases:
            base = fix_emu(rows_, rx, s)
            got = fix_emu(rows_, rx, s + d)
            worst_s = max(worst_s, abs(got["slide_out"] - base["slide_out"]))
            worst_t = max(worst_t, abs(got["clock_bias"] - base["clock_bias"]))
            worst_m = max(worst_m, *(abs(got[k] - base[k]) for k in "xyz"))
        spread[d] = (worst_s, worst_t, worst_m)
    for rows_, rx, s in cases[::10]:
        base = fx.compute_position(rows_, rx, s)
        got = fx.compute_position(rows_, rx, s + 0.07)
        assert got[0] == base[0] and abs(got[1] - base[1]) <= BIAS_S
        assert max(abs(a - b) for a, b in zip(got[2], base[2])) <= POS_M
    print(f"{name}: {len(cases)} cases; d -> slide_out spread, clock bias spread, position spread:")
    for d, (ws, wt, wm) in spread.items():
        print(f"  {d:g}: {ws:.3g} s, {wt:.3g} s, {wm:.3g} m")
    for d, (ws, wt, wm) in spread.items():
        if d <= 0.07:
            assert ws == 0.0 and wt <= BIAS_S and wm <= POS_M, d


def test_layout_python_c_and_cpp(tmp_path):
    from gypsum_b200._native import FIX_DTYPE

    names = ["receiver_timestamp", "slide_in", "slide_out", "clock_bias", "x", "y", "z", "pseudorange", "status", "n_ready",
             "channel"]
    py = [FIX_DTYPE.fields[k][1] for k in names] + [FIX_DTYPE.itemsize]
    assert py == [0, 8, 16, 24, 32, 40, 48, 56, 88, 92, 96, 112]
    assert fx.FIX_DTYPE == FIX_DTYPE
    cpp = np.zeros(12, dtype=np.int64)
    host_library("fix_emu").fix_emu_layout(cpp.ctypes.data_as(C.c_void_p))
    assert list(cpp) == py
    src = tmp_path / "layout.c"
    src.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"gypsum_b200.h\"\nint main(void) {\n"
                   + "".join(f'    printf("%d\\n", (int)offsetof(gb200_position_fix, {k}));\n' for k in names)
                   + '    printf("%d\\n", (int)sizeof(gb200_position_fix));\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", f"-I{os.path.join(ROOT, 'include')}", str(src),
                    "-o", str(exe)], check=True, capture_output=True)
    c = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert c == py


def test_python_solution_types():
    from gypsum_b200 import _native
    from gypsum_b200.world_model import EcefCoordinates, ReceiverSolution, solution_from_fix

    rec = np.zeros(1, dtype=_native.FIX_DTYPE)[0]
    rec["status"], rec["clock_bias"], rec["x"], rec["y"], rec["z"] = _native.FIX_SOLVED, 1e-12, 1.0, 2.0, 3.0
    assert solution_from_fix(rec) == ReceiverSolution(1e-12, EcefCoordinates(1.0, 2.0, 3.0))
    assert str(EcefCoordinates.zero()) == "(self.x=0.00, self.y=0.00, self.z=0.00)"
    rec["status"] = _native.FIX_NONE
    with pytest.raises(ValueError):
        solution_from_fix(rec)
