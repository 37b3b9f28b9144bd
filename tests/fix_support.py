"""What the position-fix tests share, on the CPU and the GPU: the parity bounds, the host build of the fix core
(tests/emu/fix_emu.cu) and the way a scripted timeline reaches the device.  torch and gypsum_b200 are imported inside the
functions that need them, so the CPU tests collect and run without the library."""
import ctypes as C

import numpy as np

from hostbuild import host_library
from oracle import fix_oracle as fx

# parity bounds of the host and device core against the reference's numpy (DESIGN.md §6), a small multiple of the
# spread measured on the recorded timelines (clock bias 1.2e-15 s, position 2.7e-7 m, slides identical)
POS_M, BIAS_S, SLIDE_ULPS = 2e-6, 1e-14, 4
# the least-squares mode on five or more rows of the recorded and scripted timelines (DESIGN.md §8c).  The golden rows
# are 1e4 km off any common solution, and Gauss-Newton on the squared ranges does not converge there (numpy's last step
# is up to 1.4e7 m in `five`): host and numpy follow the same cycle apart by rounding, measured up to 1.3 m, 2.7e-9 s and
# 34 ulp of the slide.  tests/test_gpu_fix_lsq.py's scripted six rows converge, on a poorer geometry: 5.6e-4 m,
# 6.1e-13 s, 0 ulp.
MANY_POS_M, MANY_BIAS_S, MANY_SLIDE_ULPS = 4.0, 1e-8, 100


def slide_tol(s):
    """SLIDE_ULPS units in the last place of a slide (about 3e5 s on the recorded timelines)."""
    return SLIDE_ULPS * 2.0 ** -52 * np.abs(s)


def fix_emulator():
    """compute(rows, rx, slide) -> one fx.FIX_DTYPE record: fix_core.cuh on the host, as the device computes the fix of
    one millisecond from rows [n][4] of (tow, x, y, z), n >= 4 (more than four rows: the least-squares mode)."""
    lib = host_library("fix_emu")
    lib.fix_emu_compute_n.restype = C.c_int
    lib.fix_emu_compute_n.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_void_p]

    def compute(rows, rx, slide):
        r = np.ascontiguousarray(rows, dtype=np.float64).reshape(-1, 4)
        out = np.zeros(1, dtype=fx.FIX_DTYPE)
        lib.fix_emu_compute_n(r.ctypes.data, len(r), float(rx), float(slide), out.ctypes.data)
        return out[0]

    return compute


def parse_events(trk, chans, n_ms):
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


def rows_at(obs, channels, m):
    """The rows (tow, x, y, z) of the given channels at millisecond m, from the device's observations."""
    return [(obs[ch, m]["tow"], obs[ch, m]["x"], obs[ch, m]["y"], obs[ch, m]["z"]) for ch in channels]


def run_calls(engine, calls, device_out=False, solver=None):
    """A timeline ([(rx, chans)], the layout of fx.golden_calls) through one tracker, call after call; per call the
    records (read back from a device buffer if device_out), the device's observations and receiver_state().  A solver
    is set before the first call; None leaves the tracker's own."""
    import torch

    from gypsum_b200 import _native

    n_ch = len(calls[0][1])
    trk = _native.Tracker(engine, list(range(n_ch)), [0.0] * n_ch, [0.0] * n_ch, [0] * n_ch)
    if solver is not None:
        trk.set_fix_solver(solver)
    out = []
    for rx, chans in calls:
        parse_events(trk, chans, len(rx))
        if device_out:
            dev = torch.empty(len(rx) * _native.FIX_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
            trk.position_fixes_device(rx, dev.data_ptr())
            torch.cuda.synchronize()
            rec = dev.cpu().numpy().view(_native.FIX_DTYPE).copy()
        else:
            rec = trk.position_fixes(rx)
        out.append((rec, trk.observations(), trk.receiver_state()))
    trk.close()
    return out


def run_golden(engine, golden_path, name, device_out=False, solver=None):
    """run_calls on a recorded timeline: the golden file, its calls and what run_calls returns."""
    z = np.load(golden_path)
    calls = fx.golden_calls(z, name)
    return z, calls, run_calls(engine, calls, device_out, solver)
