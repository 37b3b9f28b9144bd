"""Secondary measurements on one H100 (not the driver's bench line): BASELINE configs 2 (single block), 3, 5,
the real 10-pass detector, and config 4 (tracking, at 2.046 and at 16.368 Msps).  Prints one JSON line per workload.
usage: python tools/bench_configs.py [--quick]
       python tools/bench_configs.py --code-phase-modes R   config 4 only, both code-phase modes alternating, R rounds"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from gypsum_b200 import _native  # noqa: E402
from gypsum_b200.gps_ca_prn_codes import ca_code_chips  # noqa: E402
from gypsum_b200 import synth as o  # noqa: E402
from gypsum_b200 import synth as to  # noqa: E402

quick = "--quick" in sys.argv
CHIPS = np.stack([ca_code_chips(sv) for sv in range(1, 33)]).astype(np.uint8)


def noise(n_samples, seed):
    rng = np.random.default_rng(seed)
    return ((rng.standard_normal(n_samples, dtype=np.float32) + 1j * rng.standard_normal(n_samples, dtype=np.float32)) *
            np.float32(0.7071)).astype(np.complex64)


def grid_case(name, n, m, n_dop, n_blocks, reps):
    fs = n * 1000
    eng = _native.Engine(fs, n)
    eng.set_replicas(CHIPS)
    x = noise(n * m * n_blocks, 1)
    x[: n * m] += o.synth_iq(0, n, m, fs, [(25, 1500.0, 777, 0.3, 0.3)], sigma=0.0)
    dop = np.linspace(-10000, 10000, n_dop)
    prn = np.arange(32, dtype=np.int32)
    xd = torch.from_numpy(x).cuda()
    out = torch.empty(n_blocks * 32 * n_dop * 32, dtype=torch.uint8, device="cuda")
    st = torch.cuda.Stream()
    torch.cuda.set_stream(st)
    eng.set_stream(st.cuda_stream)
    eng.bind_iq_device(xd.data_ptr(), x.size)
    for _ in range(3):
        eng.acquire_grid_device(n_blocks, m, prn, dop, 2, out.data_ptr())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(st)
    for _ in range(reps):
        eng.acquire_grid_device(n_blocks, m, prn, dop, 2, out.data_ptr())
    e1.record(st)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    eng.enable_kernel_timing(True)
    for _ in range(reps):
        eng.acquire_grid_device(n_blocks, m, prn, dop, 2, out.data_ptr())
    ks, ns = eng.kernel_timing(0)
    kc, nc = eng.kernel_timing(1)
    eng.enable_kernel_timing(False)
    # host to host
    eng.upload_iq(x)
    eng.acquire_grid(n_blocks, m, prn, dop)  # warm-up: pinned staging buffers get allocated here
    t0 = time.perf_counter()
    for _ in range(max(1, reps // 4)):
        eng.upload_iq(x)
        rec = eng.acquire_grid(n_blocks, m, prn, dop)
    e2e = (time.perf_counter() - t0) / max(1, reps // 4)
    b = int(np.argmax(rec["peak"][0, 24]))
    alg = n_blocks * (32 * n_dop * m * 16 * n + 32 * 32 * n_dop)
    print(json.dumps({"workload": name, "N": n, "ms": m, "dopplers": n_dop, "blocks": n_blocks,
                      "device_ms": ms, "Msamples_per_s": n * m * n_blocks / ms / 1e3,
                      "e2e_ms": e2e * 1e3, "e2e_Msamples_per_s": n * m * n_blocks / e2e / 1e6,
                      "doppler_spectra_ms": ks / max(ns, 1) * (ns / reps), "correlate_cells_ms": kc / max(nc, 1) * (nc / reps),
                      "alg_GBs_correlate": alg / (kc / reps * 1e-3) / 1e9,
                      "sv25_found": [float(dop[b]), int(rec["argmax"][0, 24, b])]}), flush=True)
    eng.set_stream(0)
    eng.close()


def fused_case(n, m, n_dop, reps):
    """Same cells through the fused block-per-(PRN, Doppler) kernel and through the de-duplicated pair (list mode)."""
    fs = n * 1000
    eng = _native.Engine(fs, n)
    eng.set_replicas(CHIPS)
    x = noise(n * m, 1)
    eng.upload_iq(x)
    dop = np.linspace(-10000, 10000, n_dop)
    prn = np.repeat(np.arange(32), n_dop)
    dd = np.tile(dop, 32)
    out = {}
    for label, dops in (("shared Doppler bins", dd), ("unique Doppler per cell", dd + np.arange(dd.size) * 0.37)):
        for name, on in (("split", False), ("fused", True)):
            eng.set_fused(on)
            eng.acquire_cells(prn, dops, m)
            t0 = time.perf_counter()
            for _ in range(reps):
                eng.acquire_cells(prn, dops, m)
            host_ms = (time.perf_counter() - t0) / reps * 1e3
            eng.enable_kernel_timing(True)
            for _ in range(reps):
                eng.acquire_cells(prn, dops, m)
            k0, _n0 = eng.kernel_timing(0)
            k1, _n1 = eng.kernel_timing(1)
            eng.enable_kernel_timing(False)
            out[f"{label}: {name}"] = {"host_to_host_ms": host_ms, "kernels_ms": (k0 + k1) / reps}
    eng.set_fused(None)
    print(json.dumps({"workload": f"fused vs split kernels, list of 32x{n_dop} cells, {m} ms @ N={n}", **out}), flush=True)
    eng.close()


def detector_case():
    from gypsum_b200.acquisition import GpsSatelliteDetector
    from gypsum_b200.gps_ca_prn_codes import GpsSatelliteId, generate_replica_prn_signals
    from gypsum_b200.satellite import GpsSatellite

    class A:
        samples_per_second, samples_per_prn_transmission = 2046000, 2046

    planted = [(25, 1504.0, 777, 0.3, 0.12), (3, -3250.0, 5, 1.0, 0.1), (32, 4875.5, 2045, 2.5, 0.15)]
    x = o.synth_iq(7, 2046, 10, 2046000, planted)
    codes = generate_replica_prn_signals()
    det = GpsSatelliteDetector({sid: GpsSatellite(sid, c, 2) for sid, c in codes.items()})
    ids = [GpsSatelliteId(i) for i in range(1, 33)]
    det.detect_satellites_in_antenna_data(ids, x, A)
    ts = []
    for _ in range(5):
        t0 = time.perf_counter()
        found = det.detect_satellites_in_antenna_data(ids, x, A)
        ts.append(time.perf_counter() - t0)
    print(json.dumps({"workload": "real detector: 32 SV x 10 passes (222 bins) + coherent, 10 ms @ 2.046 Msps",
                      # gb200_detect takes the fused kernel at 2.046 and 4.092 Msps, the split kernels at other rates
                      "detect_kernel": "fused" if A.samples_per_prn_transmission in (2046, 4092) else "split",
                      "seconds_per_scan": float(np.median(ts)), "cell_ms_per_scan": 32 * 223 * 10,
                      "found": [[r.satellite_id.id, r.doppler_shift, r.prn_phase_shift] for r in found]}), flush=True)


def gpu_card():
    """The card's name and power limit, read where the numbers are measured."""
    import subprocess

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def tracker_case(n_ch, n_ms, code_phase="reference"):
    n, fs = 2046, 2046000
    eng = _native.Engine(fs, n)
    eng.set_replicas(CHIPS)
    chans = [(sv, 1000.0 + 37.3 * sv, 0.0, (53 * sv) % n, 0.1 * sv, 0.004) for sv in range(1, n_ch + 1)]
    base = to.synth_tracking_iq(5, n, 2000, fs, chans)
    x = np.tile(base, -(-n_ms // 2000))[: n_ms * n]  # periodic signal; noise repeats, which tracking does not care about
    trk = _native.Tracker(eng, [c[0] - 1 for c in chans], [c[1] for c in chans], [0.0] * n_ch, [c[3] for c in chans])
    trk.set_code_phase_mode(code_phase)
    times = np.array([round(k * n / fs, 6) for k in range(n_ms)])
    xd = torch.from_numpy(x).cuda()
    eng.bind_iq_device(xd.data_ptr(), x.size)
    out = torch.empty(n_ch * n_ms * _native.TRACK_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    trk.process_device(n_ms, times, out.data_ptr())
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    # navigation bits from the records where the tracking kernel left them (SURVEY 8f N4)
    ends = times + n / fs
    trk.integrate_bits(min(n_ms, 1000), times[:1000], ends[:1000], out.data_ptr())  # warm-up (allocations); state is reset below
    trk.close()
    trk = _native.Tracker(eng, [c[0] - 1 for c in chans], [c[1] for c in chans], [0.0] * n_ch, [c[3] for c in chans])
    trk.set_code_phase_mode(code_phase)
    t0 = time.perf_counter()
    bits = trk.integrate_bits(n_ms, times, ends, out.data_ptr())
    dt_bits = time.perf_counter() - t0
    rec = out.cpu().numpy().view(_native.TRACK_DTYPE).reshape(n_ch, n_ms)
    print(json.dumps({"workload": f"config 4: {n_ch}-channel E/P/L tracking, {n_ms / 1000:.0f} s of IQ @ 2.046 Msps",
                      "code_phase": code_phase,
                      "seconds": dt, "channel_ms_per_s": n_ch * n_ms / dt, "us_per_ms_per_channel_stream": dt / n_ms * 1e6,
                      "realtime_factor": (n_ms / 1000) / dt, "Msamples_per_s_stream": n_ms * n / dt / 1e6,
                      "locked_fraction_last_second": float(rec["locked"][:, -1000:].mean()),
                      "lost_channels": int((rec["lost"] > 0).any(axis=1).sum()),
                      "bit_integration_seconds": dt_bits, "bits_emitted": int(sum(len(b) for b in bits)),
                      "bits_unknown": int(sum((b["bit_value"] < 0).sum() for b in bits))}), flush=True)
    trk.close()
    eng.close()


def tracker_case_16368(n_ch, n_ms, code_phase="reference"):
    """Config 4 at 16.368 Msps (k_track_channels_wide<16>): device-resident IQ, a 1-s synthetic base repeated.  Planted code
    phases stay below 2046, the only ones the reference's tracker keeps at this rate.  The symbols of 3 channels over the
    first second are checked against the tracker oracle."""
    from oracle import tracker_oracle as t

    n, fs, base_ms = 16368, 16368000, 1000
    eng = _native.Engine(fs, n)
    eng.set_replicas(CHIPS)
    st = torch.cuda.Stream()  # the engine launches on this stream; the events are recorded on it
    eng.set_stream(st.cuda_stream)
    chans = [(sv, 1000.0 + 37.3 * sv, 0.0, (53 * sv) % 2046, 0.1 * sv, 0.002) for sv in range(1, n_ch + 1)]
    base = to.synth_tracking_iq(5, n, base_ms, fs, chans)
    xd = torch.from_numpy(base.view(np.float32)).cuda().repeat(-(-n_ms // base_ms))[: n_ms * n * 2]
    eng.bind_iq_device(xd.data_ptr(), n_ms * n)
    seeds = ([c[0] - 1 for c in chans], [c[1] for c in chans], [0.0] * n_ch, [c[3] for c in chans])
    times = np.array([round(k * n / fs, 6) for k in range(n_ms)])
    out = torch.empty(n_ch * n_ms * _native.TRACK_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()  # the stream and its buffers are ready before the engine's stream reads them
    trk = _native.Tracker(eng, *seeds)
    trk.set_code_phase_mode(code_phase)
    trk.process_device(200, times[:200], out.data_ptr())  # warm-up
    trk.close()
    trk = _native.Tracker(eng, *seeds)
    trk.set_code_phase_mode(code_phase)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(st)
    trk.process_device(n_ms, times, out.data_ptr())
    e1.record(st)
    torch.cuda.synchronize()
    dt = e0.elapsed_time(e1) * 1e-3
    rec = out.cpu().numpy().view(_native.TRACK_DTYPE).reshape(n_ch, n_ms)
    trk.close()
    check_ms, mism = min(n_ms, base_ms), {}
    for i in (0, 13, 31):
        sv, f, _, cp = chans[i][:4]
        tr = t.TrackerOracle(sv, f, 0.0, cp, fs, n)  # planted below 2046: both modes follow the same trajectory
        want = [tr.step(base[k * n:(k + 1) * n], *t.chunk_times(k, fs, n))["symbol"] for k in range(check_ms)]
        mism[sv] = int(np.count_nonzero(rec["symbol"][i, :check_ms] != np.array(want)))
    print(json.dumps({"workload": f"config 4 @ 16.368 Msps: {n_ch}-channel tracking, {n_ms / 1000:.0f} s of device-resident IQ",
                      "kernel": "k_track_channels_wide<16>", "code_phase": code_phase, "device_seconds": dt, "us_per_stream_ms": dt / n_ms * 1e6,
                      "realtime_factor": (n_ms / 1000) / dt, "channel_ms_per_s": n_ch * n_ms / dt,
                      "lost_channels": int((rec["lost"] > 0).any(axis=1).sum()),
                      "oracle_symbol_mismatches": {"ms": check_ms, "by_sv": mism},
                      "gpu": torch.cuda.get_device_name()}), flush=True)
    eng.set_stream(0)
    eng.close()


if __name__ == "__main__" and "--code-phase-modes" in sys.argv:
    rounds = int(sys.argv[sys.argv.index("--code-phase-modes") + 1])
    print(json.dumps({"gpu": gpu_card()}), flush=True)
    for _ in range(rounds):
        for mode in ("reference", "samples"):
            tracker_case(32, 5000 if quick else 60000, mode)
            tracker_case_16368(32, 2000 if quick else 10000, mode)
elif __name__ == "__main__":
    grid_case("config 2, one block", 2046, 1, 41, 1, 200)
    grid_case("config 2 x 32 blocks", 2046, 1, 41, 32, 50)
    grid_case("config 3: 32x41x10 ms @ 4.092 Msps", 4092, 10, 41, 1, 20)
    grid_case("config 5 shape: 32x81 @ 16.368 Msps, 1-ms blocks", 16368, 1, 81, 4 if quick else 16, 5)
    fused_case(2046, 1, 41, 50)
    fused_case(2046, 10, 24, 10)
    detector_case()
    tracker_case(32, 5000 if quick else 60000)
    tracker_case_16368(32, 2000 if quick else 10000)
