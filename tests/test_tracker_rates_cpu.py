"""Tracking at the sample rates other than 2.046 / 4.092 Msps, CPU side: the tracker oracle bit-exact against the live
reference's trajectories at 1.023, 8.184 and 16.368 Msps (tools/make_golden_tracker.py).  The reference keeps its
hard-wired 2046 at every rate (tracker.py:301-303, :319)."""
import os

import numpy as np
import pytest

from oracle import tracker_oracle as t

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("name", ["fs1", "fs8", "fs16", "fs16_long"])
def test_oracle_tracker_bit_exact_with_reference_at_other_rates(name):
    z = np.load(os.path.join(GOLDEN, f"tracker_{name}.npz"))
    ch = z["channel"]
    ch = (int(ch[0]), ch[1], ch[2], int(ch[3]), ch[4], ch[5])
    n, fs, init, rows = int(z["n"]), int(z["fs"]), z["init"], z["rows"]
    x = t.synth_tracking_iq(int(z["seed"]), n, int(z["n_ms"]), fs, [ch], float(z["sigma"]))
    tr = t.TrackerOracle(ch[0], init[0], init[1], int(init[2]), fs, n)
    for k in range(len(rows)):
        a, b = t.chunk_times(k, fs, n)
        r = tr.step(x[k * n:(k + 1) * n], a, b)
        mine = np.array([r["peak"].real, r["peak"].imag, r["strength"], r["symbol"], r["error"], r["disc"], r["doppler"],
                         r["carrier_phase"], r["code_phase"], r["start"], r["end"], tr.phase, r["doppler_hist"],
                         r["carrier_phase_hist"]], dtype=np.float64)
        assert np.array_equal(mine, rows[k]), k
    assert int(z["lost_at"]) == -1 and len(rows) == int(z["n_ms"])
    if name == "fs1":  # the accumulator wraps at 2046 > N: code phases beyond the millisecond, np.roll is modular
        assert (rows[:, 8] >= n).all()
    if name == "fs16_long":  # the 6-second constellation check ran (no adjustment: the constellation is circular enough)
        assert len(rows) > 6000 and np.array_equal(rows[:, 6], rows[:, 12])
