"""Semi-coherent acquisition on one H100: one 100-ms window at 2.046 Msps, 32 PRNs, +-7 kHz at 50 Hz (281 bins),
T = 10, K = 10, through gb200_acquire_grid_semicoherent_best_device; against it on the same IQ the non-coherent M = 100
grid over the same 281 bins and over 29 bins at 500 Hz, and config 2's grid (32 PRN x 41 Doppler x 1 ms, 256 blocks) for
its per-transform rate.  Prints the card, its power limit and one JSON line per workload, then the noise-only strength
distribution of the best bin of the main workload over 32 noise-only PRNs.
With --weak the main workload is the weak grid instead (gb200_acquire_grid_weak_best_device): one 995-ms window at
2.046 Msps, 32 PRNs, +-7 kHz at 25 Hz (561 bins), T = 20 with B = 4 bit phases 5 ms apart (K = 49 segments per phase),
with config 2's grid for its per-transform rate and the same noise-only distribution.
usage: python tools/bench_semicoherent.py [--reps R] [--weak]"""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from gypsum_b200 import _native  # noqa: E402
from gypsum_b200 import synth as o  # noqa: E402
from gypsum_b200.gps_ca_prn_codes import ca_code_chips  # noqa: E402

N, FS = 2046, 2046000
S = N // 1023
CHIPS = np.stack([ca_code_chips(sv) for sv in range(1, 33)]).astype(np.uint8)
REPS = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def noise(n_samples, seed):
    rng = np.random.default_rng(seed)
    return ((rng.standard_normal(n_samples, dtype=np.float32) + 1j * rng.standard_normal(n_samples, dtype=np.float32)) *
            np.float32(0.7071)).astype(np.complex64)


def timed(eng, call, reps):
    """(device ms per call from events, spectra ms per call, correlate ms per call) after three warm-up calls."""
    for _ in range(3):
        call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    eng.enable_kernel_timing(True)
    for _ in range(reps):
        call()
    ks, _ = eng.kernel_timing(0)
    kc, _ = eng.kernel_timing(1)
    eng.enable_kernel_timing(False)
    return ms, ks / reps, kc / reps


def config2_row(eng, prn):
    """Config 2's grid: 256 one-millisecond blocks of 32 PRN x 41 Doppler."""
    nb = 256
    x2 = noise(nb * N, 2)
    x2d = torch.from_numpy(x2).cuda()
    dop2 = np.linspace(-10000, 10000, 41)
    out2 = torch.empty(nb * 32 * 41 * 32, dtype=torch.uint8, device="cuda")
    eng.bind_iq_device(x2d.data_ptr(), x2.size)
    ms, ks, kc = timed(eng, lambda: eng.acquire_grid_device(nb, 1, prn, dop2, _native.NON_COHERENT, out2.data_ptr()), REPS)
    t2 = nb * 32 * 41 * S
    return dict(workload="config 2 grid, 256 blocks", call_ms=ms, spectra_ms=ks, correlate_ms=kc, inverse_transforms=t2,
                forward_transforms=nb * 41 * S, inverse_per_s=t2 / (kc * 1e-3), call_transforms_per_s=t2 / (ms * 1e-3))


def print_rows(rows):
    for r in rows:
        r["correlate_rate_vs_config2"] = r["inverse_per_s"] / rows[-1]["inverse_per_s"]
        print(json.dumps(r), flush=True)


def print_noise(best_strengths):
    s = np.array(best_strengths)
    print(json.dumps({"noise_only_best_strength": {"n": int(s.size), "mean": float(s.mean()), "p50": float(np.median(s)),
                                                   "p99": float(np.quantile(s, 0.99)), "max": float(s.max())}}), flush=True)


def weak(eng, prn):
    t, b, m = 20, 4, 995
    k = (m - (b - 1) * (t // b)) // t
    x = noise(m * N, 1)
    x += o.synth_iq(0, N, m, FS, [(25, 1234.0, 777, 0.3, 0.016)], sigma=0.0)  # 27.2 dB-Hz
    xd = torch.from_numpy(x).cuda()
    eng.bind_iq_device(xd.data_ptr(), x.size)
    fine = np.arange(-7000.0, 7012.5, 25.0)
    out = torch.empty(32 * 32, dtype=torch.uint8, device="cuda")
    ms, ks, kc = timed(eng, lambda: eng.acquire_grid_weak_best_device(1, m, t, b, prn, fine, out.data_ptr()), REPS)
    transforms = 32 * b * fine.size * k * S  # inverse DFT-1023 per (PRN, phase, bin, segment, branch)
    row = dict(workload=f"weak T={t} B={b} K={k} M={m}, {fine.size} bins (best)", call_ms=ms, spectra_ms=ks, correlate_ms=kc,
               inverse_transforms=transforms, forward_transforms=b * fine.size * k * S,
               wiped_ms=b * fine.size * k * t, inverse_per_s=transforms / (kc * 1e-3),
               call_transforms_per_s=transforms / (ms * 1e-3))
    best = eng.acquire_grid_weak_best(1, m, t, b, prn, fine)[0]
    row["sv25_found"] = [float(best["doppler"][24]), int(best["code_phase"][24]), int(best["bin"][24]) // fine.size,
                         float(best["strength"][24])]
    del xd
    print_rows([row, config2_row(eng, prn)])
    strengths = []
    for seed in range(8):
        xn = torch.from_numpy(noise(m * N, 100 + seed)).cuda()
        eng.bind_iq_device(xn.data_ptr(), m * N)
        strengths.extend(eng.acquire_grid_weak_best(1, m, t, b, prn, fine)[0]["strength"].tolist())
    print_noise(strengths)


def main():
    print(json.dumps({"card": card()}), flush=True)
    eng = _native.Engine(FS, N)
    eng.set_replicas(CHIPS)
    st = torch.cuda.Stream()  # the events and the engine share one stream
    torch.cuda.set_stream(st)
    eng.set_stream(st.cuda_stream)
    prn = np.arange(32, dtype=np.int32)
    if "--weak" in sys.argv:
        weak(eng, prn)
        eng.set_stream(0)
        eng.close()
        return
    m = 100
    x = noise(m * N, 1)
    x += o.synth_iq(0, N, m, FS, [(25, 1234.0, 777, 0.3, 0.03)], sigma=0.0)  # 32.7 dB-Hz, 20-ms data bits off
    xd = torch.from_numpy(x).cuda()
    eng.bind_iq_device(xd.data_ptr(), x.size)
    fine = np.arange(-7000.0, 7025.0, 50.0)
    coarse = np.arange(-7000.0, 7250.0, 500.0)
    out = torch.empty(32 * fine.size * 32, dtype=torch.uint8, device="cuda")
    rows = []
    cases = [
        ("semicoherent T=10 K=10, 281 bins (best)", 10, fine, lambda: eng.acquire_grid_semicoherent_best_device(
            1, m, 10, prn, fine, out.data_ptr())),
        ("non-coherent M=100, 281 bins (best)", 1, fine, lambda: eng.acquire_grid_best_device(
            1, m, prn, fine, _native.NON_COHERENT, out.data_ptr())),
        ("non-coherent M=100, 29 bins (best)", 1, coarse, lambda: eng.acquire_grid_best_device(
            1, m, prn, coarse, _native.NON_COHERENT, out.data_ptr())),
    ]
    for name, t, dop, call in cases:
        ms, ks, kc = timed(eng, call, REPS)
        transforms = 32 * dop.size * (m // t) * S  # inverse DFT-1023 per (PRN, bin, segment, branch)
        fwd = dop.size * (m // t) * S               # forward DFT-1023 per (bin, segment, branch)
        rows.append(dict(workload=name, call_ms=ms, spectra_ms=ks, correlate_ms=kc, inverse_transforms=transforms,
                         forward_transforms=fwd, wiped_samples=dop.size * m * N,
                         inverse_per_s=transforms / (kc * 1e-3), call_transforms_per_s=transforms / (ms * 1e-3)))
    best = eng.acquire_grid_semicoherent_best(1, m, 10, prn, fine)[0]
    rows[0]["sv25_found"] = [float(best["doppler"][24]), int(best["code_phase"][24]), float(best["strength"][24])]
    rows.append(config2_row(eng, prn))
    print_rows(rows)
    # noise-only strength of the main workload's best bin: 32 PRNs x 8 windows of pure noise
    strengths = []
    for seed in range(8):
        xn = torch.from_numpy(noise(m * N, 100 + seed)).cuda()
        eng.bind_iq_device(xn.data_ptr(), m * N)
        strengths.extend(eng.acquire_grid_semicoherent_best(1, m, 10, prn, fine)[0]["strength"].tolist())
    print_noise(strengths)
    eng.set_stream(0)
    eng.close()


if __name__ == "__main__":
    main()
