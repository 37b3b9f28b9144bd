"""Times gb200_tracker_parse_subframes and gb200_tracker_observations_device: 132 channels x 60 s, every channel with
its own planted ephemeris (oracle/orbit_oracle.py) and a subframe every 6 s, from a fresh world model, next to the
tracking launch the chain starts from (132 channels x 60 s of device-resident IQ, a 1-s synthetic base repeated).  Each
call is bracketed by CUDA events on the engine's stream (parse includes its uploads and the fields' download; the
observations stay on the device), and one round is also profiled for the kernels alone.
usage (GPU box): python tools/bench_orbit.py [--reps 5]"""
import argparse
import json
import os
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
N_CH, N_MS, N_SUB = 132, 60000, 10


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
    # one replica row per channel (rows repeat the 32 codes): the world model is keyed by row
    eng.set_replicas(np.stack([ca_code_chips(c % 32 + 1) for c in range(N_CH)]).astype(np.uint8))
    stream = torch.cuda.Stream()
    eng.set_stream(stream.cuda_stream)
    chans = [(c % 32 + 1, 1000.0 + 37.3 * c, 0.0, (53 * c) % N, 0.1 * c, 0.004) for c in range(N_CH)]
    base = to.synth_tracking_iq(5, N, 1000, FS, chans[:32])
    xd = torch.from_numpy(base).cuda().repeat(N_MS // 1000)
    eng.bind_iq_device(xd.data_ptr(), xd.numel())
    times = np.array([round(k * N / FS, 6) for k in range(N_MS)])
    rec = torch.empty(N_CH * N_MS * _native.TRACK_DTYPE.itemsize, dtype=torch.uint8, device="cuda")

    rng = np.random.default_rng(1)
    host = np.zeros((N_CH, N_SUB), dtype=_native.SUBFRAME_DTYPE)
    ems = np.zeros((N_CH, N_SUB), dtype=np.int32)
    for c in range(N_CH):
        sfs = orb.ephemeris_subframes(orb.realistic_ephemeris(rng, c % 32 + 1), N_SUB, first_id=c % 5 + 1, tow0=1000 + c, seed=c)
        for k, sf in enumerate(sfs):
            host[c, k]["words"] = orb.words_of(sf)
            host[c, k]["trailing_edge_receiver_timestamp"] = 6.0 * (k + 1) + 0.001 * c
            ems[c, k] = 6000 * k + 3 * c
    ev_dev = torch.from_numpy(host.view(np.uint8).reshape(N_CH, -1)).cuda()
    counts = np.full(N_CH, N_SUB, dtype=np.int32)
    drop = np.full(N_CH, -1, dtype=np.int32)
    obs = torch.empty(N_CH * N_MS * _native.OBSERVATION_DTYPE.itemsize, dtype=torch.uint8, device="cuda")

    track_ms, parse_ms, obs_ms, kernel_ms = [], [], [], {}
    for rep in range(args.reps + 1):
        trk = _native.Tracker(eng, list(range(N_CH)), [c[1] for c in chans], [0.0] * N_CH, [c[3] for c in chans])
        dt, _ = timed(stream, lambda: trk.process_device(N_MS, times, rec.data_ptr()))
        prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) if rep == 1 else None
        if prof:
            prof.__enter__()
        dp, _ = timed(stream, lambda: trk.parse_subframes(ev_dev.data_ptr(), counts, N_SUB, ems, drop, N_MS))
        do, _ = timed(stream, lambda: trk.observations_device(obs.data_ptr()))
        if prof:
            prof.__exit__(None, None, None)
            for k in prof.key_averages():
                for name in ("k_parse_subframes", "k_sv_observations"):
                    if name in k.key:
                        kernel_ms[name] = getattr(k, "device_time_total", getattr(k, "cuda_time_total", 0.0)) / 1e3
        if rep:  # the first round allocates
            track_ms.append(dt)
            parse_ms.append(dp)
            obs_ms.append(do)
        trk.close()
    o = obs.cpu().numpy().view(_native.OBSERVATION_DTYPE)
    dev = torch.cuda.get_device_properties(0)
    print(json.dumps({
        "workload": f"parse_subframes + observations: {N_CH} channels x {N_MS} ms, {N_SUB} subframes per channel",
        "gpu": dev.name,
        "parse_call_ms_median": float(np.median(parse_ms)),
        "observations_call_ms_median": float(np.median(obs_ms)), "observations_call_ms": obs_ms,
        "kernel_ms_profiled": kernel_ms,
        "tracking_launch_ms_median": float(np.median(track_ms)),
        "orbit_fraction_of_tracking": float((np.median(parse_ms) + np.median(obs_ms)) / np.median(track_ms)),
        "positions_computed": int(((o["flags"] & _native.OBS_COMPLETE) > 0).sum())}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
