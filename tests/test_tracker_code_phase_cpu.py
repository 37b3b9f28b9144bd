"""The tracker's code-phase modes on the CPU (DESIGN.md §7): the tracker oracle with its DLL wrapped at N against every
trajectory recorded from the live reference, the host build of track_update with the modulus N teacher-forced against
that oracle at code phases across [0, N), and the pseudosymbol delay rule of the bit integrator and the drop-in."""
import numpy as np
import pytest

from code_phase_support import HostTrack, WrapOracle, planted_phases, stamps
from oracle import tracker_oracle as t
from test_tracker_cpu import TRACK_REC
from tracker_support import load_tracker_case, oracle_row

GOLDEN_CASES = ["short", "long", "noise", "adjust", "join55", "join6", "join575_noise", "gap", "hour", "day", "fs1", "fs4",
                "fs8", "fs16", "fs16_long"]
LIMIT = 1500  # milliseconds of each file; the oracle costs about 10 ms per millisecond at 16.368 Msps
LOOP = [0, 1, 2, 3, 4, 5, 6, 7, 12, 13]  # the golden columns the modulus does not touch (all but code phase, stamps, phase)


def _accumulators(z, rows):
    """The reference's DLL accumulator before each millisecond's wrap: the previous phase plus disc * 0.002."""
    before = np.concatenate([[float(z["init"][2])], rows[:-1, 11]])
    return before + rows[:, 5] * 0.002


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_wrapped_oracle_against_every_golden_trajectory(name):
    """TrackerOracle with the DLL wrapped at N.  Where the reference's accumulator never leaves [0, min(N, 2046)) the
    trajectory is the reference's bit for bit, stamps aside: they are the chunk times plus code_phase / N ms.  On fs1
    (1.023 Msps, code phases of 1499 and 1500 >= N in the reference) the code phase is the reference's mod 1023 and the
    accumulator its value mod 1023 to within rounding; everything the correlators and loop filters produce is exact,
    bar milliseconds whose accumulator sits within rounding of an integer, proved one by one."""
    z, ch, x, n, fs, tt = load_tracker_case(name)
    init, rows = z["init"], z["rows"]
    n_run = min(LIMIT, len(rows))
    acc = _accumulators(z, rows[:n_run])
    wraps = not ((acc >= 0) & (acc < min(n, 2046))).all()
    print(f"{name}: N = {n}, the reference's accumulator {'leaves' if wraps else 'stays in'} [0, {min(n, 2046)})")
    assert wraps == (name == "fs1")
    tr = WrapOracle(ch[0], init[0], init[1], int(init[2]), fs, n, wrap=n)
    for k in range(n_run):
        mine, ref = oracle_row(tr, tr.step(x[k * n:(k + 1) * n], *tt[k])), rows[k]
        delay = (int(mine[8]) / n) * 0.001
        assert (mine[9], mine[10]) == (tt[k, 0] + delay, tt[k, 1] + delay), k
        if not wraps:
            assert np.array_equal(mine[[8, 11]], ref[[8, 11]]) and np.array_equal(mine[LOOP], ref[LOOP]), k
            continue
        assert np.array_equal(mine[LOOP], ref[LOOP]), k
        assert int(mine[8]) % n == int(ref[8]) % n, k
        d = (mine[11] - ref[11]) % n
        assert min(d, n - d) <= 1e-9, k


def test_wrapped_oracle_is_the_oracle_at_2046():
    """wrap = 2046 leaves TrackerOracle's rows byte for byte, on the recorded loss of lock too."""
    z, ch, x, n, fs, tt = load_tracker_case("noise")
    init = z["init"]
    a = t.TrackerOracle(ch[0], init[0], init[1], int(init[2]), fs, n)
    b = WrapOracle(ch[0], init[0], init[1], int(init[2]), fs, n)
    for k in range(int(z["lost_at"]) + 1):
        try:
            ra = oracle_row(a, a.step(x[k * n:(k + 1) * n], *tt[k]))
        except t.LostLock as exc:
            with pytest.raises(t.LostLock) as got:
                b.step(x[k * n:(k + 1) * n], *tt[k])
            assert exc.args[0] == got.value.args[0] and a.phase == b.phase and k == int(z["lost_at"])
            break
        assert oracle_row(b, b.step(x[k * n:(k + 1) * n], *tt[k])).tobytes() == ra.tobytes(), k


CORE_MS = 100  # teacher-forced milliseconds per channel: the oracle's cost grows with N


@pytest.mark.parametrize("s", [1, 3, 8, 16])
def test_core_wrapped_at_n_teacher_forced(s):
    """track_update with the modulus N, fed each millisecond's correlator outputs of the free-running oracle wrapped at
    N, follows it: code phase, symbol and lock exact, Doppler, carrier phase and error within the §6 bounds.  Planted
    code phases 2046 and 2047, N / 2 + r on every polyphase branch r, N - 2 and N - 1; each channel's signal sits one
    sample off its seed in alternate directions, so that the accumulators move and the ones at N - 2 and N - 1 cross
    the wrap."""
    n, fs = 1023 * s, 1023000 * s
    phases = sorted(set(planted_phases(s) + [2046, 2047, n - 2]))
    crossed = 0
    for c, cp in enumerate(phases):
        sig = (cp + (1 if c % 2 else -1)) % n if cp < n else cp % n
        x = t.synth_tracking_iq(300 + c, n, CORE_MS, fs, [(1 + c, 800.3, 0.0, sig, 0.7, 40.0 / n)])
        tr = WrapOracle(1 + c, 800.0, 0.0, cp, fs, n, wrap=n)
        core = HostTrack(c, 800.0, 0.0, cp, fs, n)
        rec = np.zeros(1, TRACK_REC)
        seen = []
        for k in range(CORE_MS):
            a, b = t.chunk_times(k, fs, n)
            r = tr.step(x[k * n:(k + 1) * n], a, b)
            core.update(r, a, rec)
            assert rec["code_phase"][0] == r["code_phase"] and rec["symbol"][0] == r["symbol"], (cp, k)
            d = abs(rec["phase_acc"][0] - tr.phase)
            assert 0 <= rec["phase_acc"][0] < n and min(d, n - d) <= 1e-3, (cp, k)
            assert abs(rec["doppler"][0] - r["doppler"]) <= 1e-6 * max(1.0, abs(r["doppler"])), (cp, k)
            d = abs(rec["carrier_phase"][0] - r["carrier_phase"])
            assert min(d, 2 * np.pi - d) <= 1e-5, (cp, k)
            assert abs(rec["error"][0] - r["error"]) <= 2e-6 * max(1.0, abs(r["error"])), (cp, k)
            assert rec["locked"][0] == int(r["locked"]) and rec["lost"][0] == 0, (cp, k)
            seen.append(r["code_phase"])
        crossed += any(abs(p - q) > n // 2 for p, q in zip(seen, seen[1:]))
    assert crossed >= 1, "no accumulator crossed the wrap"


@pytest.mark.parametrize("s", [1, 2, 3, 4, 5, 6, 8, 10, 12, 16])
def test_delay_rule(s):
    """track_symbol_delay: the chunk times plus (code_phase / N) * 1e-3, each sum rounded on its own, bit for bit, for
    code phases across [-N, 2N) and chunk times up to a day; the drop-in's _pseudosymbol gives the same stamps."""
    from gypsum_b200 import _native
    from gypsum_b200.tracker import _pseudosymbol

    n = 1023 * s
    rng = np.random.default_rng(s)
    cp = np.concatenate([np.arange(-3, 3), np.arange(n - 3, n + 3), [2045, 2046, 2047], rng.integers(-n, 2 * n, 2000)])
    t0 = np.round(rng.choice([0.0, 5.5, 3599.5, 86399.5], cp.size) + rng.integers(0, 100000, cp.size) * 1e-3, 6)
    t1 = np.round(t0 + 1e-3, 6)
    for wrap in (n, 2046):
        ts, te = stamps(cp, t0, t1, wrap)
        for k in range(cp.size):
            delay = (int(cp[k]) / wrap) * 1e-3
            assert (ts[k], te[k]) == (t0[k] + delay, t1[k] + delay), (wrap, int(cp[k]))
        rec = np.zeros(cp.size, _native.TRACK_DTYPE)
        rec["code_phase"], rec["symbol"] = cp, 1
        for k in range(0, cp.size, 7):
            ps = _pseudosymbol(rec[k], float(t0[k]), float(t1[k]), wrap)
            assert (ps.start_of_pseudosymbol, ps.end_of_pseudosymbol) == (ts[k], te[k])


@pytest.mark.parametrize("name", ["short", "fs1", "fs16"])
def test_reference_stamps_unchanged(name):
    """With the modulus 2046 the delay rule gives the stamps the live reference recorded, byte for byte, at every rate
    (tracker.py:319), and _pseudosymbol's default is that modulus."""
    from gypsum_b200 import _native
    from gypsum_b200.tracker import _pseudosymbol

    z, _, _, _, _, tt = load_tracker_case(name)
    rows = z["rows"]
    ts, te = stamps(rows[:, 8].astype(int), tt[:len(rows), 0], tt[:len(rows), 1], 2046)
    assert ts.tobytes() == rows[:, 9].tobytes() and te.tobytes() == rows[:, 10].tobytes()
    rec = np.zeros(1, _native.TRACK_DTYPE)
    for k in range(0, len(rows), 13):
        rec["code_phase"], rec["symbol"] = int(rows[k, 8]), 1
        ps = _pseudosymbol(rec[0], float(tt[k, 0]), float(tt[k, 1]))
        assert (ps.start_of_pseudosymbol, ps.end_of_pseudosymbol) == (rows[k, 9], rows[k, 10])
