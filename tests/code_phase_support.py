"""What the code-phase mode tests share (DESIGN.md §7): the tracker oracle with its DLL accumulator wrapped at a chosen
modulus, the host build of track_update and the delay rule with that modulus, and the planted channels of every rate."""
import ctypes

import numpy as np

from hostbuild import host_library
from oracle import tracker_oracle as t

ALL_RATES = [1, 2, 3, 4, 5, 6, 8, 10, 12, 16]


class WrapOracle(t.TrackerOracle):
    """TrackerOracle whose DLL accumulator wraps at `wrap` (tracker.py:301-303 wraps at 2046) and whose pseudosymbol
    delay is code_phase / wrap ms (:319).  The step runs the oracle's own arithmetic; the accumulator before the wrap is
    formed again from the step's discriminator by the same float64 operations, so wrap = 2046 is the oracle itself."""

    def __init__(self, sv, doppler, carrier_phase, code_phase, fs, n, wrap=2046):
        super().__init__(sv, doppler, carrier_phase, code_phase, fs, n)
        self.wrap = wrap

    def step(self, samples, start_time, end_time):
        before = self.phase
        try:
            out = super().step(samples, start_time, end_time)
        except t.LostLock as exc:
            self._rewrap(before, exc.args[0], start_time, end_time)
            raise
        self._rewrap(before, out, start_time, end_time)
        return out

    def _rewrap(self, before, out, start_time, end_time):
        acc = before + np.float64(out["disc"]) * 0.002
        assert int(acc) == out["code_phase"]
        self.phase = acc % self.wrap
        delay = (out["code_phase"] / self.wrap) * 0.001
        out["start"], out["end"] = start_time + delay, end_time + delay


def stamps(code_phase, t0, t1, wrap):
    """The bit integrator's start / end stamps for these records' code phases and chunk times (track_symbol_delay)."""
    lib = host_library("track_emu")
    cp = np.ascontiguousarray(code_phase, dtype=np.int32)
    a = np.ascontiguousarray(t0, dtype=np.float64)
    b = np.ascontiguousarray(t1, dtype=np.float64)
    ts, te = np.empty_like(a), np.empty_like(a)
    lib.track_emu_stamps.argtypes = [ctypes.c_int] + [ctypes.c_void_p] * 3 + [ctypes.c_double] + [ctypes.c_void_p] * 2
    lib.track_emu_stamps(cp.size, cp.ctypes.data, a.ctypes.data, b.ctypes.data, float(wrap), ts.ctypes.data, te.ctypes.data)
    return ts, te


class HostTrack:
    """One channel of the host build of track_update with the DLL wrapping at `wrap`."""

    def __init__(self, prn_idx, doppler, carrier_phase, code_phase, fs, wrap):
        self.lib = lib = host_library("track_emu")
        lib.track_emu_init.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_double, ctypes.c_int]
        lib.track_emu_update.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float, ctypes.c_int, ctypes.c_double,
                                         ctypes.c_double, ctypes.c_double, ctypes.c_void_p]
        self.st = ctypes.create_string_buffer(lib.track_emu_state_size())
        lib.track_emu_init(self.st, int(prn_idx), float(doppler), float(carrier_phase), int(code_phase))
        self.fs, self.wrap = float(fs), float(wrap)

    def update(self, r, t0, out):
        """Teacher-forced with oracle step result r; writes the 112-byte record into out (a 1-element record array)."""
        elp = np.array([r["early"].real, r["early"].imag, r["late"].real, r["late"].imag, r["peak"].real, r["peak"].imag],
                       dtype=np.float32)
        self.lib.track_emu_update(self.st, elp.ctypes.data, np.float32(r["strength"]), int(r["peak_offset"]), float(t0),
                                  self.fs, self.wrap, out.ctypes.data)


def amplitude(s):
    """The planted amplitude the golden trajectories use at S samples per chip (sigma 0.02): 0.004 up to 4.092 Msps,
    then halved per doubling of the rate, where the reference's DLL drifts about a chip in 6 s."""
    return 0.004 * min(1.0, 4.0 / s)


def planted_phases(s):
    """Code phases across [0, N): N - 1, N / 2 + r on every polyphase branch r, and 2046 and 2047 where N > 2046."""
    n = 1023 * s
    phases = [n - 1] + [n // 2 - (n // 2) % s + r for r in range(s)]
    if n > 2046:
        phases += [p for p in (2046, 2047) if p not in phases]
    assert sorted({p % s for p in phases}) == list(range(s)) and len(set(phases)) == len(phases)
    return phases


def planted_channels(s, phases):
    """(sv, doppler, rate, code phase, carrier phase, amplitude) per phase, each on its own satellite."""
    return [(1 + c, 1000.3 - 97.1 * c, 0.0, p, 0.3 + 0.1 * c, amplitude(s)) for c, p in enumerate(phases)]


def oracle_rows(args):
    """The free-running WrapOracle's rows (tracker_support.oracle_row layout) over the first n_ms milliseconds of x, and
    the millisecond it lost lock at (-1: none).  args = (x, n, fs, seed, n_ms, wrap) with seed = (sv, doppler, carrier
    phase, code phase); a top-level function, so that a process pool can run channels side by side."""
    from tracker_support import oracle_row

    x, n, fs, seed, n_ms, wrap = args
    tr = WrapOracle(*seed, fs, n, wrap=wrap)
    rows = []
    for k in range(n_ms):
        try:
            rows.append(oracle_row(tr, tr.step(x[k * n:(k + 1) * n], *t.chunk_times(k, fs, n))))
        except t.LostLock:
            return np.array(rows), k
    return np.array(rows), -1
