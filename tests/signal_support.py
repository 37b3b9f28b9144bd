"""What the signal test modules share: the host build of the estimator core (tests/emu/signal_emu.cu) and tracking
records built from the golden files' rows."""
import ctypes as C
import os

import numpy as np

import signal_oracle as so
from hostbuild import host_library
from oracle import tracker_oracle as t
from tracker_support import GOLDEN

# golden files with a planted signal (amplitude > 0), and those with noise only
SIGNAL_CASES = ("adjust", "day", "fs1", "fs16", "fs16_long", "fs4", "fs8", "gap", "hour", "join55", "join6", "long",
                "short")
NOISE_CASES = ("noise", "join575_noise")


def track_dtype():
    from gypsum_b200 import _native

    return _native.TRACK_DTYPE


def signal_dtype():
    from gypsum_b200 import _native

    return _native.SIGNAL_DTYPE


class SignalEmulator:
    """One channel's estimator in the host build of signal_core.cuh, kept across run() calls like the device's."""

    def __init__(self, window_ms, n):
        self.lib = host_library("signal_emu")
        self.lib.signal_emu_run.restype = C.c_int
        self.lib.signal_emu_run.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_void_p,
                                            C.c_int]
        self.lib.signal_emu_floor.restype = C.c_double
        self.lib.signal_emu_state_bytes.restype = C.c_int
        self.state = np.zeros(self.lib.signal_emu_state_bytes(), dtype=np.uint8)
        self.lib.signal_emu_init(self.state.ctypes.data_as(C.c_void_p))
        self.w = int(window_ms)
        self.floor = float(self.lib.signal_emu_floor(int(n)))

    def run(self, records, start_times):
        """SIGNAL_DTYPE windows of one call over one channel's TRACK_DTYPE records."""
        rec = np.ascontiguousarray(records, dtype=track_dtype())
        ts = np.ascontiguousarray(start_times, dtype=np.float64)
        cap = rec.size // self.w + 2
        out = np.zeros(cap, dtype=signal_dtype())
        k = self.lib.signal_emu_run(self.state.ctypes.data_as(C.c_void_p), rec.ctypes.data_as(C.c_void_p),
                                    ts.ctypes.data_as(C.c_void_p), rec.size, self.w, self.floor,
                                    out.ctypes.data_as(C.c_void_p), cap)
        assert k <= cap
        return out[:k].copy()


def golden_records(name):
    """(TRACK_DTYPE records, start times, n, planted C/N0 or None) of golden file tracker_<name>.npz: prompt I, Q and
    strength from the rows (columns 0-2) as float32, `lost` set on the row lost_at, records past the rows zero."""
    z = np.load(os.path.join(GOLDEN, f"tracker_{name}.npz"))
    n, fs = int(z["n"]), int(z["fs"])
    if "start_times" in z.files:
        times = np.asarray(z["start_times"], dtype=np.float64)
    else:
        times = np.array([t.chunk_times(k, fs, n)[0] for k in range(int(z["n_ms"]))])
    rows, lost_at = z["rows"], int(z["lost_at"])
    rec = np.zeros(len(times), dtype=track_dtype())
    m = len(rows)
    rec["peak_re"][:m], rec["peak_im"][:m], rec["strength"][:m] = rows[:, 0], rows[:, 1], rows[:, 2]
    if lost_at >= 0:
        rec["lost"][lost_at] = 1
    amp = float(z["channel"][5])
    planted = so.planted_cn0_dbhz(amp, float(z["sigma"]), fs) if amp > 0 else None
    return rec, times, n, planted


def oracle_windows(records, start_times, window_ms, floor_dbhz, oracle=None):
    """The oracle's windows of one call over TRACK_DTYPE records, as a SIGNAL_DTYPE array."""
    o = oracle or so.SignalOracle(window_ms, floor_dbhz)
    rows = o.feed(records["peak_re"], records["peak_im"], records["strength"], records["locked"], records["lost"],
                  start_times)
    return np.array(rows, dtype=signal_dtype())


def assert_windows_match(got, want, what=""):
    """Every field exact except cn0_dbhz, held to 1e-12 relative (NaN where the other is NaN)."""
    assert got.shape == want.shape, what
    for f in signal_dtype().names:
        if f == "cn0_dbhz":
            g, w = got[f], want[f]
            assert np.array_equal(np.isnan(g), np.isnan(w)), what
            ok = ~np.isnan(w)
            assert (np.abs(g[ok] - w[ok]) <= 1e-12 * np.abs(w[ok])).all(), what
        else:
            assert np.array_equal(got[f], want[f], equal_nan=got[f].dtype.kind == "f"), (what, f)


def without_ms_index(w):
    """The bytes of windows with ms_index cleared: what calls of any sizes must agree on."""
    w = w.copy()
    w["ms_index"] = 0
    return w.tobytes()
