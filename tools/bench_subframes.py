"""Times gb200_tracker_decode_subframes: 132 channels x 60 s of navigation bits (3000 per channel, LNAV from
oracle/nav_oracle.py, every other channel inverted) decoded from a fresh decoder in one call, next to the tracking
launch those bits would follow (132 channels x 60 s of device-resident IQ, a 1-s synthetic base repeated).  Both are
bracketed by CUDA events on the engine's stream; the decode figure includes the call's count upload and event download
(each tracker's buffers are allocated beforehand by a call without bits), and one round is also profiled for the kernel
alone.
usage (GPU box): python tools/bench_subframes.py [--reps 5]"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gypsum_b200 import _native  # noqa: E402
from gypsum_b200 import synth as to  # noqa: E402
from gypsum_b200.gps_ca_prn_codes import ca_code_chips  # noqa: E402
from oracle import nav_oracle as nav  # noqa: E402

N, FS = 2046, 2046000
N_CH, N_MS, N_BITS = 132, 60000, 3000


def timed(stream, fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    out = fn()
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    eng = _native.Engine(FS, N)
    eng.set_replicas(np.stack([ca_code_chips(sv) for sv in range(1, 33)]).astype(np.uint8))
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)
    sv = [c % 32 + 1 for c in range(N_CH)]
    chans = [(s, 1000.0 + 37.3 * c, 0.0, (53 * c) % N, 0.1 * c, 0.004) for c, s in enumerate(sv)]
    base = to.synth_tracking_iq(5, N, 1000, FS, chans[:32])  # 32 distinct signals; channels 32.. track copies
    xd = torch.from_numpy(base).cuda().repeat(N_MS // 1000)
    eng.bind_iq_device(xd.data_ptr(), xd.numel())
    times = np.array([round(k * N / FS, 6) for k in range(N_MS)])
    rec = torch.empty(N_CH * N_MS * _native.TRACK_DTYPE.itemsize, dtype=torch.uint8, device="cuda")

    # LNAV bits per channel, each starting at its own place in a subframe
    host = np.zeros((N_CH, N_BITS), dtype=_native.BIT_DTYPE)
    for c in range(N_CH):
        bits = np.concatenate([np.asarray(sf, np.int8) for sf in nav.lnav_frames(c, 12, first_id=c % 5 + 1)])
        bits = bits[(37 * c) % 300:][:N_BITS]
        host["bit_value"][c] = bits if c % 2 == 0 else 1 - bits
        t0, t1 = nav.bit_times(N_BITS, t_first=0.001 * (c % 20))
        host["receiver_timestamp"][c], host["trailing_edge_receiver_timestamp"][c] = t0, t1
    bits_dev = torch.from_numpy(host.view(np.uint8).reshape(N_CH, -1)).cuda()
    counts = np.full(N_CH, N_BITS, dtype=np.int32)

    cap = _native.subframe_event_capacity(N_BITS)
    zeros = np.zeros(N_CH, dtype=np.int32)
    warm_ev = np.empty((N_CH, cap), dtype=_native.SUBFRAME_DTYPE)
    warm_cnt = np.empty(N_CH, dtype=np.int32)
    track_ms, decode_ms, wall_ms, kernel_ms = [], [], [], []
    n_sub = None
    for rep in range(args.reps + 1):
        trk = _native.Tracker(eng, [c[0] - 1 for c in chans], [c[1] for c in chans], [0.0] * N_CH, [c[3] for c in chans])
        dt, _ = timed(stream, lambda: trk.process_device(N_MS, times, rec.data_ptr()))
        # a call with no bits allocates the decoder state and the event buffers of this tracker, and decodes nothing
        eng._check(eng._lib.gb200_tracker_decode_subframes(trk._h, _native._P(bits_dev.data_ptr()), zeros.ctypes.data, N_BITS,
                                                           warm_ev.ctypes.data, cap, warm_cnt.ctypes.data), "warm-up")
        assert trk.subframe_state(0)["processed_bit_count"] == 0
        prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) if rep == 1 else None
        if prof:
            prof.__enter__()
        w0 = time.perf_counter()
        dd, ev = timed(stream, lambda: trk.decode_subframes(bits_dev.data_ptr(), counts, N_BITS))
        wall = (time.perf_counter() - w0) * 1e3
        if prof:
            prof.__exit__(None, None, None)
            for k in prof.key_averages():
                if "k_decode_subframes" in k.key:
                    kernel_ms.append(getattr(k, "device_time_total", getattr(k, "cuda_time_total", 0.0)) / 1e3)
        if rep:  # the first round allocates
            track_ms.append(dt)
            decode_ms.append(dd)
            wall_ms.append(wall)
        n_sub = sum(int((e["kind"] == 0).sum()) for e in ev)
        # a coincidental preamble pair in the data can win the first search, as in the reference: then a reset and a
        # re-sync, or a raise on a "subframe 5" with the wrong data id
        n_raised = sum(int((e["kind"] == _native.RAISED).sum()) for e in ev)
        trk.close()
    dev = torch.cuda.get_device_properties(0)
    print(json.dumps({
        "workload": f"decode_subframes: {N_CH} channels x {N_BITS} bits (60 s) from fresh decoders, one call",
        "gpu": dev.name,
        "decode_call_ms_median": float(np.median(decode_ms)), "decode_call_ms": decode_ms,
        "decode_host_wall_ms_median": float(np.median(wall_ms)),
        "decode_kernel_ms_profiled": kernel_ms[0] if kernel_ms else None,
        "tracking_launch_ms_median": float(np.median(track_ms)),
        "decode_fraction_of_tracking": float(np.median(decode_ms) / np.median(track_ms)),
        "subframes_decoded": n_sub, "channels_raised": n_raised}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
