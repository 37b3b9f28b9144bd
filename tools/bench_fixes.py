"""Times gb200_tracker_position_fixes_device: 4 channels x 60 000 ms with a fix on every millisecond from the third,
next to the tracking launch it follows (4 channels x 60 s of device-resident IQ, a 1-s synthetic base repeated).  The
four channels carry their own planted ephemerides (oracle/orbit_oracle.py) with the same TOW counts: subframes 1-3 land
in milliseconds 0-2 and then one every 6 s on all four, so their times of week stay consistent.  Each call is
bracketed by CUDA events on the engine's stream (the fix call includes the upload of the receiver timestamps and the
observations it computes first); one round is also profiled for the kernels alone.

--jump J puts a receiver-clock jump of J seconds (a gap in the sample stream) at millisecond --jump-ms: from there on,
J is added to the fix call's receiver timestamps and to every later trailing edge.  Inside a segment that makes the
device's chain check miss, and k_fix_repair recomputes the rest of the segment serially (DESIGN.md §8c); the result
line then also reports the repaired fixes and the cost of each.

--channels N tracks and fixes N channels (4 to 12) on the same schedule, so every fixing millisecond has N ready;
--solver least_squares fixes them by least squares (gb200_tracker_set_fix_solver).  The reference mode raises at the
first fix with more than four channels.

--velocity also times gb200_tracker_velocity_fixes_device right after each fix call, on the fix records that call wrote
and the tracking records' Dopplers, and reports its median and its kernel next to the fix call's.
usage (GPU box): python tools/bench_fixes.py [--reps 5] [--jump -0.2 [--jump-ms 1000]] [--channels 8 --solver least_squares]
                 [--velocity]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gypsum_b200 import _native  # noqa: E402
from gypsum_b200 import synth as to  # noqa: E402
from gypsum_b200.gps_ca_prn_codes import ca_code_chips  # noqa: E402
from oracle import orbit_oracle as orb  # noqa: E402

N, FS = 2046, 2046000
N_MS, N_SUB = 60000, 12
SVS = (5, 12, 19, 27, 2, 9, 15, 23, 30, 7, 17, 25)


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
    ap.add_argument("--jump", type=float, default=0.0, help="receiver-clock jump in seconds (0: none)")
    ap.add_argument("--jump-ms", type=int, default=1000, help="the millisecond the jump lands on")
    ap.add_argument("--channels", type=int, default=4, choices=range(4, len(SVS) + 1), metavar="N")
    ap.add_argument("--solver", default="reference", choices=sorted(_native.FIX_SOLVERS))
    ap.add_argument("--velocity", action="store_true", help="also time the velocity call after each fix call")
    args = ap.parse_args()
    n_ch = args.channels
    eng = _native.Engine(FS, N)
    eng.set_replicas(np.stack([ca_code_chips(sv) for sv in range(1, 33)]).astype(np.uint8))
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)
    svs = SVS[:n_ch]
    chans = [(sv, 1000.0 + 37.3 * c, 0.0, (53 * c) % N, 0.1 * c, 0.004) for c, sv in enumerate(svs)]
    base = to.synth_tracking_iq(5, N, 1000, FS, chans)
    xd = torch.from_numpy(base).cuda().repeat(N_MS // 1000)
    eng.bind_iq_device(xd.data_ptr(), xd.numel())
    times = np.array([round(k * N / FS, 6) for k in range(N_MS)])
    rec = torch.empty(n_ch * N_MS * _native.TRACK_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    fix_times = times.copy()
    fix_times[args.jump_ms:] += args.jump

    rng = np.random.default_rng(1)
    host = np.zeros((n_ch, N_SUB), dtype=_native.SUBFRAME_DTYPE)
    ems = np.zeros((n_ch, N_SUB), dtype=np.int32)
    for c, sv in enumerate(svs):
        sfs = orb.ephemeris_subframes(orb.realistic_ephemeris(rng, sv), N_SUB, first_id=1, tow0=20000, seed=c)
        for k, sf in enumerate(sfs):
            m = k if k < 3 else 2 + 6000 * (k - 2)
            host[c, k]["words"] = orb.words_of(sf)
            host[c, k]["trailing_edge_receiver_timestamp"] = fix_times[min(m, N_MS - 1)] - 0.0003 * c
            ems[c, k] = min(m, N_MS - 1)
    ev_dev = torch.from_numpy(host.view(np.uint8).reshape(n_ch, -1)).cuda()
    counts = np.full(n_ch, N_SUB, dtype=np.int32)
    drop = np.full(n_ch, -1, dtype=np.int32)
    out = torch.empty(N_MS * _native.FIX_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    vout = torch.empty(N_MS * _native.VELOCITY_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    rec_doubles = _native.TRACK_DTYPE.itemsize // 8  # the Doppler is the record's first field

    track_ms, fix_ms, vel_ms, kernel_ms, repaired = [], [], [], {}, []
    for rep in range(args.reps + 1):
        trk = _native.Tracker(eng, list(range(n_ch)), [c[1] for c in chans], [0.0] * n_ch, [c[3] for c in chans])
        trk.set_fix_solver(args.solver)
        dt, _ = timed(stream, lambda: trk.process_device(N_MS, times, rec.data_ptr()))
        trk.parse_subframes(ev_dev.data_ptr(), counts, N_SUB, ems, drop, N_MS)
        prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) if rep == 1 else None
        if prof:
            prof.__enter__()
        df, _ = timed(stream, lambda: trk.position_fixes_device(fix_times, out.data_ptr()))
        if args.velocity:
            with torch.cuda.stream(stream):
                dop = rec.view(torch.float64).view(n_ch, N_MS, rec_doubles)[:, :, 0].contiguous()
            dv, _ = timed(stream, lambda: trk.velocity_fixes_device(vout.data_ptr(), dop.data_ptr(), out.data_ptr()))
        if prof:
            prof.__exit__(None, None, None)
            for k in prof.key_averages():
                for name in ("k_sv_observations", "k_fix_plan", "k_fix_pass<1>", "k_fix_pass<2>", "k_fix_repair",
                             "k_fix_finish", "k_fix_plan_lsq", "k_fix_pass_lsq<1>", "k_fix_pass_lsq<2>",
                             "k_fix_repair_lsq", "k_velocity_fixes"):
                    if name + "(" in k.key or k.key.endswith(name):
                        kernel_ms[name] = getattr(k, "device_time_total", getattr(k, "cuda_time_total", 0.0)) / 1e3
        if rep:  # the first round allocates
            track_ms.append(dt)
            fix_ms.append(df)
            if args.velocity:
                vel_ms.append(dv)
        repaired.append(trk.receiver_state()["repaired"])
        trk.close()
    f = out.cpu().numpy().view(_native.FIX_DTYPE)
    dev = torch.cuda.get_device_properties(0)
    jump = {}
    if args.jump:
        jump = {"jump_s": args.jump, "jump_ms": args.jump_ms, "repaired_fixes": repaired[-1],
                "repair_kernel_us_per_fix": kernel_ms.get("k_fix_repair_lsq" if args.solver == "least_squares" else "k_fix_repair", 0.0) * 1e3 / max(1, repaired[-1])}
    vel = {}
    if args.velocity:
        v = vout.cpu().numpy().view(_native.VELOCITY_DTYPE)
        vel = {"velocity_call_ms_median": float(np.median(vel_ms)), "velocity_call_ms": vel_ms,
               "velocity_fraction_of_fix": float(np.median(vel_ms) / np.median(fix_ms)),
               "velocity_status_counts": [int(c) for c in np.bincount(v["status"], minlength=3)]}
    print(json.dumps({
        "workload": f"position_fixes_device: {n_ch} channels x {N_MS} ms after the parse call, {args.solver} solver",
        "gpu": dev.name, "power_limit": power_limit(),
        "fix_call_ms_median": float(np.median(fix_ms)), "fix_call_ms": fix_ms,
        "kernel_ms_profiled": kernel_ms,
        "tracking_launch_ms_median": float(np.median(track_ms)),
        "fix_fraction_of_tracking": float(np.median(fix_ms) / np.median(track_ms)),
        "fixes": int((f["status"] == _native.FIX_SOLVED).sum()),
        "status_counts": [int(v) for v in np.bincount(f["status"], minlength=4)], **jump, **vel}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
