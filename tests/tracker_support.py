"""What the tracking test modules share: the trajectories recorded from the live reference tracker (tests/golden/
tracker_*.npz) and the bounds a device trajectory is held to against them (DESIGN.md section 6)."""
import os

import numpy as np

from oracle import tracker_oracle as t

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_tracker_case(name):
    """(golden file, channel, IQ, n, fs, times) of tracker_<name>.npz, the IQ re-synthesised from the recorded seed and
    times[k] = (start, end) of millisecond k.  A file that records no n / fs is at 2.046 Msps; one that records no start
    times starts at 0 without gaps.  A file that records them (a late join, a gap, long stream times) has its samples
    synthesised from the first start time on."""
    z = np.load(os.path.join(GOLDEN, f"tracker_{name}.npz"))
    ch = z["channel"]
    ch = (int(ch[0]), ch[1], ch[2], int(ch[3]), ch[4], ch[5])
    n, fs = (int(z["n"]), int(z["fs"])) if "n" in z.files else (2046, 2046000)
    n_ms = int(z["n_ms"])
    if "start_times" in z.files:
        times = np.stack([z["start_times"], z["end_times"]], axis=1)
    else:
        times = np.array([t.chunk_times(k, fs, n) for k in range(n_ms)])
    x = t.synth_tracking_iq(int(z["seed"]), n, n_ms, fs, [ch], float(z["sigma"]), t0=float(times[0, 0]))
    return z, ch, x, n, fs, times


def start_times(n_ms, fs, n):
    """The receiver start time of each of the first n_ms milliseconds."""
    return np.array([t.chunk_times(k, fs, n)[0] for k in range(n_ms)])


def oracle_row(tr, r):
    """One row in the layout of the golden files' rows, from TrackerOracle tr and the result r of its last step."""
    return np.array([r["peak"].real, r["peak"].imag, r["strength"], r["symbol"], r["error"], r["disc"], r["doppler"],
                     r["carrier_phase"], r["code_phase"], r["start"], r["end"], tr.phase, r["doppler_hist"],
                     r["carrier_phase_hist"]], dtype=np.float64)


def assert_ms_matches_oracle(rec, r, k):
    """One teacher-forced millisecond: device record rec against the oracle's step result r from the same state.
    Correlator outputs within 1e-5 of the prompt peak's magnitude (float32 against float64), strength, disc and error
    within 1e-4, peak offset, symbol and code phase exact."""
    scale = abs(r["peak"])
    assert abs(complex(rec["peak_re"], rec["peak_im"]) - r["peak"]) <= 1e-5 * scale, k
    assert abs(complex(rec["early_re"], rec["early_im"]) - r["early"]) <= 1e-5 * scale, k
    assert abs(complex(rec["late_re"], rec["late_im"]) - r["late"]) <= 1e-5 * scale, k
    assert abs(rec["strength"] - r["strength"]) <= 1e-4 * r["strength"], k
    assert rec["peak_offset"] == r["peak_offset"] and rec["symbol"] == r["symbol"], k
    assert rec["code_phase"] == r["code_phase"], k
    assert abs(rec["disc"] - r["disc"]) <= 1e-4 * max(1.0, abs(r["disc"])), k
    assert abs(rec["error"] - r["error"]) <= 1e-4 * max(1.0, abs(r["error"])), k


def _assert_phase_close(got, want, tol):
    d = np.abs(got - want)
    assert np.minimum(d, 2 * np.pi - d).max() <= tol


def assert_follows_reference(rec, rows, histories=False):
    """A device trajectory that never lost lock against the reference's rows (the golden layout, oracle_row).
    Pseudosymbols and code phase are EXACT, bar per-millisecond proofs taken from the reference's own float64 trajectory:
    a symbol may differ only where the reference's in-phase prompt value is float32 noise around zero; the code phase
    (int() of the DLL accumulator, tracker.py:298-299) only where the reference's accumulator sits within 5e-3 of an integer
    and ours within 5e-3 of the reference's.  Doppler within 5e-3 Hz, carrier phase within 2e-3 rad; with histories, the
    same for the history values (tracker.py:352-353, columns 12 and 13)."""
    assert not rec["lost"].any()
    scale = np.abs(rows[:, 0]).max()
    for k in np.flatnonzero(rec["symbol"] != rows[:, 3].astype(int)):
        assert abs(rows[k, 0]) <= 1e-4 * scale, k
    for k in np.flatnonzero(rec["code_phase"] != rows[:, 8].astype(int)):
        frac = rows[k, 11] - np.floor(rows[k, 11])
        assert min(frac, 1 - frac) <= 5e-3 and abs(rec["phase_acc"][k] - rows[k, 11]) <= 5e-3, k
    assert np.abs(rec["doppler"] - rows[:, 6]).max() <= 5e-3
    _assert_phase_close(rec["carrier_phase"], rows[:, 7], 2e-3)
    if histories:
        assert np.abs(rec["doppler_hist"] - rows[:, 12]).max() <= 5e-3
        _assert_phase_close(rec["carrier_phase_hist"], rows[:, 13], 2e-3)
