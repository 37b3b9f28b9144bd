"""Times gb200_tracker_signal_windows: 132 channels x 60 000 ms of tracking records at 2.046 Msps, with W = 20 and
W = 1000, next to the tracking launch that wrote them (132 channels x 60 s of device-resident IQ, a 1-s synthetic base
of eight satellites repeated).  The call reads the records through records_device; each is bracketed by CUDA events on
the engine's stream and by the host clock (it returns with the windows on the host), and one round is profiled for the
two kernels alone.  The first call of each W allocates and is not counted.  The card's name and power limit are read
in the same run.
usage (GPU box): python tools/bench_signal.py [--reps 5] [--channels 132] [--ms 60000]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gypsum_b200 import _native  # noqa: E402
from gypsum_b200 import synth as to  # noqa: E402
from gypsum_b200.gps_ca_prn_codes import ca_code_chips  # noqa: E402

N, FS = 2046, 2046000
SVS = (5, 12, 19, 27, 2, 9, 15, 23)
KERNELS = ("k_signal_stop", "k_signal_windows")


def timed(stream, fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    out = fn()
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b), out


def power_limit() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--channels", type=int, default=132)
    ap.add_argument("--ms", type=int, default=60000, help="milliseconds of records (a multiple of 1000)")
    args = ap.parse_args()
    n_ch, n_ms = args.channels, args.ms
    eng = _native.Engine(FS, N)
    eng.set_replicas(np.stack([ca_code_chips(sv) for sv in range(1, 33)]).astype(np.uint8))
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)
    sats = [(sv, 1000.0 + 373.1 * i, 0.0, (211 * i) % N, 0.4 * i, 0.002 + 0.0005 * i) for i, sv in enumerate(SVS)]
    base = to.synth_tracking_iq(5, N, 1000, FS, sats)
    xd = torch.from_numpy(base).cuda().repeat(n_ms // 1000)
    eng.bind_iq_device(xd.data_ptr(), xd.numel())
    times = np.array([round(k * N / FS, 6) for k in range(n_ms)])
    rec = torch.empty(n_ch * n_ms * _native.TRACK_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    chans = [sats[c % len(sats)] for c in range(n_ch)]
    trk = _native.Tracker(eng, [c[0] - 1 for c in chans], [c[1] for c in chans], [c[4] for c in chans],
                          [c[3] for c in chans])
    track_ms, _ = timed(stream, lambda: trk.process_device(n_ms, times, rec.data_ptr()))
    trk.close()

    result = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "channels": n_ch, "ms": n_ms,
              "record_bytes": n_ch * n_ms * _native.TRACK_DTYPE.itemsize, "track_launch_ms": round(track_ms, 2)}
    for w in (20, 1000):
        # one estimator over the same records again and again: n_ms is a multiple of W, so every call starts with no
        # window open and does the same work
        est = _native.Tracker(eng, [0] * n_ch, [0.0] * n_ch, [0.0] * n_ch, [0] * n_ch)
        call_ms, event_ms, kernel_ms, windows = [], [], {}, None
        for rep in range(args.reps + 1):
            prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) if rep == 1 else None
            if prof:
                prof.__enter__()
            t0 = time.perf_counter()
            de, windows = timed(stream, lambda: est.signal_windows(n_ms, times, w, records_device_ptr=rec.data_ptr()))
            dt = (time.perf_counter() - t0) * 1e3
            if prof:
                prof.__exit__(None, None, None)
                for k in prof.key_averages():
                    for name in KERNELS:
                        if name + "(" in k.key or k.key.endswith(name):
                            kernel_ms[name] = getattr(k, "device_time_total", getattr(k, "cuda_time_total", 0.0)) / 1e3
            if rep:  # the first round allocates
                call_ms.append(dt)
                event_ms.append(de)
        est.close()
        found = sum(int((a["status"] == _native.SIGNAL_FOUND).sum()) for a in windows)
        result[f"w{w}"] = {"call_ms": round(float(np.median(call_ms)), 3),
                           "event_ms": round(float(np.median(event_ms)), 3),
                           "kernel_ms": {k: round(v, 4) for k, v in kernel_ms.items()},
                           "windows": sum(len(a) for a in windows), "status1": found,
                           "cn0_median": round(float(np.median(np.concatenate([a["cn0_dbhz"] for a in windows]))), 2)}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
