"""A/B timing of library builds on the split acquisition path (doppler_spectra + the correlate kernel).  Every build runs in its
own child process (GB200_LIB selects the library); the builds take turns for --rounds rounds, so clock and neighbour drift
spread over all of them.

usage: python tools/ab_correlate.py LIB_A LIB_B [LIB ...] [--workload W[,W ...]] [--rounds 5] [--calls 24] [--out DIR]

Workloads (seeded IQ: bench.make_ring's noise with bench.py's planted satellites):
  config2             bench.py's config-2 call (default): 256 blocks x 32 PRN x 41 Doppler, 1 ms, non-coherent, 2.046 Msps,
                      from a device-resident IQ ring larger than L2 (seed 1000)
  coherent-grid-256   the same call, coherent
  coherent-grid-4092  32 PRN x 41 Doppler x 10 ms coherent at 4.092 Msps, one window per call
  coherent-cells      32 cells (one per PRN, own Doppler, probed) x 10 ms coherent at 16.368 Msps: gb200_detect's coherent
                      pass at a rate the fused kernel does not cover
  detect              gb200_detect, 32 satellites x 10 ms at 16.368 Msps, whole call
  profile-K-mM-N      correlation_profile of one cell, K = nc | c, M ms, N samples per ms (e.g. profile-nc-m10-2046), call
                      latency

Prints one JSON line per workload: per build the per-launch ms of doppler_spectra and correlate (enable_kernel_timing; median,
min, max over rounds) and the call time (CUDA events around a synchronised run of calls), the card's name, power limit and SM
clock (sampled during the rounds), and, for every build after the first, whether its output of the first call is
byte-identical to LIB_A's -- or else the largest differences (see compare).  --out also writes the lines to
DIR/ab_correlate.json."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def setup(workload: str, stream):
    """Engine and IQ of a workload: returns (engine, call(j), output() after call(0), warm-up calls, the device IQ to keep
    alive)."""
    import torch

    import bench
    from gypsum_b200 import _native
    from gypsum_b200.gps_ca_prn_codes import ca_code_chips

    def engine(n):
        eng = _native.Engine(n * 1000, n)
        eng.set_replicas(np.stack([ca_code_chips(sv) for sv in range(1, 33)]).astype(np.uint8))
        eng.set_stream(stream.cuda_stream)
        return eng

    def window(n, m):  # one seeded block of m ms, resident on the device
        x = torch.from_numpy(bench.make_ring(1, seed=1000, n=n, fs=n * 1000, m=m)).cuda()
        eng = engine(n)
        eng.bind_iq_device(x.data_ptr(), m * n)
        return eng, x

    prn = np.arange(bench.N_PRN, dtype=np.int32)
    dop = np.ascontiguousarray(bench.DOPPLERS, dtype=np.float64)
    if workload in ("config2", "coherent-grid-256"):
        kind = _native.NON_COHERENT if workload == "config2" else _native.COHERENT
        B = 256
        block_bytes = bench.N * 8
        ring_blocks = (bench.L2_BYTES // block_bytes // B + 2) * B  # bench.py's ring: larger than L2
        ring = torch.from_numpy(bench.make_ring(ring_blocks, seed=1000)).cuda()
        n_slots = ring_blocks // B
        eng = engine(bench.N)
        rec = torch.empty(B * bench.N_PRN * dop.size * 32, dtype=torch.uint8, device="cuda")

        def call(j: int):
            eng.bind_iq_device(ring.data_ptr() + (j % n_slots) * B * block_bytes, B * bench.N)
            eng.acquire_grid_device(B, 1, prn, dop, kind, rec.data_ptr())

        return eng, call, lambda: rec.cpu().numpy(), 2 * n_slots, ring
    if workload == "coherent-grid-4092":
        eng, x = window(4092, 10)
        rec = torch.empty(bench.N_PRN * dop.size * 32, dtype=torch.uint8, device="cuda")
        return (eng, lambda j: eng.acquire_grid_device(1, 10, prn, dop, _native.COHERENT, rec.data_ptr()),
                lambda: rec.cpu().numpy(), 4, x)
    if workload in ("coherent-cells", "detect"):
        n = 16368
        eng, x = window(n, 10)
        if workload == "detect":
            out = {}
            return eng, lambda j: out.__setitem__(0, eng.detect(prn, 10)), lambda: out[0], 4, x
        # planted satellites at their Doppler and code phase, the others at seeded Dopplers and probes
        rng = np.random.default_rng(1000)
        cdop = rng.integers(-20, 21, prn.size) * 500.0
        probe = rng.integers(0, n, prn.size).astype(np.int32)
        for sv, f, tau, _, _ in bench.PLANTED:
            cdop[sv - 1], probe[sv - 1] = f, tau
        out = {}
        return (eng, lambda j: out.__setitem__(0, eng.acquire_cells(prn, cdop, 10, _native.COHERENT, probe_idx=probe)),
                lambda: out[0], 4, x)
    if workload.startswith("profile-"):
        _, k, m, n = workload.split("-")
        kind = {"nc": _native.NON_COHERENT, "c": _native.COHERENT}[k]
        m, n = int(m[1:]), int(n)
        eng, x = window(n, m)
        out = {}
        return eng, lambda j: out.__setitem__(0, eng.correlation_profile(24, 1500.0, m, kind)), lambda: out[0], 4, x
    raise SystemExit(f"unknown workload {workload}")


def worker(workload: str, calls: int) -> None:
    """Child: one library build, `calls` calls per round.  Reads 'round' / 'output PATH' / 'quit' lines on stdin and answers
    each with one JSON line."""
    import torch

    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    eng, call, output, warm, keep = setup(workload, stream)
    for j in range(warm):  # warm-up
        call(j)
    torch.cuda.synchronize()
    print(json.dumps({"ready": True}), flush=True)
    for line in sys.stdin:
        cmd = line.split()
        if cmd[0] == "round":
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for j in range(calls):
                call(j)
            e1.record(stream)
            torch.cuda.synchronize()
            call_ms = e0.elapsed_time(e1) / calls
            eng.enable_kernel_timing(True)
            for j in range(calls):
                call(j)
            ks, ns = eng.kernel_timing(0)
            kc, nc = eng.kernel_timing(1)
            eng.enable_kernel_timing(False)
            print(json.dumps({"call_ms": call_ms, "spectra_ms": ks / max(ns, 1), "correlate_ms": kc / max(nc, 1)}), flush=True)
        elif cmd[0] == "output":
            call(0)
            torch.cuda.synchronize()
            np.save(cmd[1], output())
            print(json.dumps({"saved": cmd[1]}), flush=True)
        else:
            break
    del keep
    eng.set_stream(0)
    eng.close()


class ClockSampler:
    """SM clock of GPU 0 every 0.25 s while the rounds run (nvidia-smi, one short query per sample)."""

    def __init__(self):
        self.mhz: list[int] = []
        self._stop = threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()

    def _run(self) -> None:
        while not self._stop.is_set():
            q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                               capture_output=True, text=True)
            if q.returncode == 0 and q.stdout.strip().isdigit():
                self.mhz.append(int(q.stdout.strip()))
            self._stop.wait(0.25)

    def stop(self) -> list[int]:
        self._stop.set()
        self._t.join()
        return self.mhz


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, max_sm = (s.strip() for s in q.stdout.strip().split(","))
    return {"name": name, "power_limit": power, "clocks_max_sm": max_sm}


def spread(v: list[float]) -> dict:
    return {"median": statistics.median(v), "min": min(v), "max": max(v)}


def compare(a: np.ndarray, b: np.ndarray, kind: str) -> dict:
    """Byte identity, or else the largest differences: records relative to the largest peak (probes too), acquisition
    results as mismatched (Doppler, code phase) pairs, strength relative and carrier phase in rad, profiles relative to the
    largest magnitude."""
    if a.tobytes() == b.tobytes():
        return {"byte_identical": True}
    from gypsum_b200 import _native

    if kind == "profile":
        return {"byte_identical": False, "max_diff_over_max_abs": float(np.max(np.abs(a - b)) / np.max(np.abs(a)))}
    if kind == "acquisition":
        ra, rb = a.view(_native.ACQ_DTYPE), b.view(_native.ACQ_DTYPE)
        dphi = np.abs(np.angle((ra["probe_re"] + 1j * ra["probe_im"]) * (rb["probe_re"] - 1j * rb["probe_im"])))
        return {"byte_identical": False,
                "doppler_or_code_phase_mismatches": int(np.count_nonzero((ra["doppler"] != rb["doppler"]) |
                                                                         (ra["code_phase"] != rb["code_phase"]))),
                "max_strength_rel_diff": float(np.max(np.abs(ra["strength"] - rb["strength"]) / ra["strength"])),
                "max_carrier_phase_diff_rad": float(np.max(dphi))}
    ra, rb = a.view(_native.RECORD_DTYPE), b.view(_native.RECORD_DTYPE)
    scale = float(np.max(ra["peak"]))
    return {"byte_identical": False,
            "max_peak_diff_over_max_peak": float(np.max(np.abs(ra["peak"] - rb["peak"]))) / scale,
            "max_sum_diff_over_max_peak": float(np.max(np.abs(ra["sum"] - rb["sum"]))) / scale,
            "max_probe_diff_over_max_peak": float(np.max(np.abs((ra["probe_re"] - rb["probe_re"]) +
                                                                1j * (ra["probe_im"] - rb["probe_im"])))) / scale,
            "argmax_mismatches": int(np.count_nonzero(ra["argmax"] != rb["argmax"])),
            "count_mismatches": int(np.count_nonzero(ra["count"] != rb["count"]))}


def run(workload: str, libs: list[str], rounds: int, calls: int) -> dict:
    children = []
    for lib in libs:
        env = dict(os.environ, GB200_LIB=lib)
        children.append(subprocess.Popen([sys.executable, os.path.abspath(__file__), "--worker", workload, str(calls)], env=env,
                                         text=True, stdin=subprocess.PIPE, stdout=subprocess.PIPE))

    def ask(child, line: str) -> dict:
        child.stdin.write(line + "\n")
        child.stdin.flush()
        return json.loads(child.stdout.readline())

    try:
        for c in children:
            if not json.loads(c.stdout.readline()).get("ready"):
                raise RuntimeError("a worker did not start")
        info = card()
        sampler = ClockSampler()
        runs: list[list[dict]] = [[] for _ in libs]
        for _ in range(rounds):
            for i, c in enumerate(children):
                runs[i].append(ask(c, "round"))
        mhz = sampler.stop()
        with tempfile.TemporaryDirectory() as tmp:
            outs = []
            for i, c in enumerate(children):
                path = os.path.join(tmp, f"out{i}.npy")
                ask(c, f"output {path}")
                outs.append(np.load(path))
        result = {"workload": workload, "card": info, "sm_mhz_during_rounds": spread([float(m) for m in mhz]) if mhz else None,
                  "rounds": rounds, "calls_per_round": calls, "builds": []}
        kind = "acquisition" if workload == "detect" else "profile" if workload.startswith("profile-") else "records"
        for i, lib in enumerate(libs):
            r = runs[i]
            b = {"lib": os.path.relpath(lib, ROOT), "call_ms": spread([x["call_ms"] for x in r]),
                 "spectra_ms": spread([x["spectra_ms"] for x in r]), "correlate_ms": spread([x["correlate_ms"] for x in r])}
            if i:
                first = result["builds"][0]
                b["call_change_vs_first"] = b["call_ms"]["median"] / first["call_ms"]["median"] - 1
                b["correlate_change_vs_first"] = b["correlate_ms"]["median"] / first["correlate_ms"]["median"] - 1
                b["output_vs_first"] = compare(outs[0], outs[i], kind)
            result["builds"].append(b)
    finally:
        for c in children:
            if c.poll() is None:
                try:
                    c.stdin.write("quit\n")
                    c.stdin.flush()
                except BrokenPipeError:
                    pass
        for c in children:
            try:
                c.wait(timeout=60)
            except subprocess.TimeoutExpired:
                c.kill()
                c.wait()
    return result


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+")
    ap.add_argument("--workload", default="config2", help="comma-separated workloads (see the module docstring)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=24)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if len(args.libs) < 2:
        ap.error("give at least two library builds")
    libs = [os.path.abspath(p) for p in args.libs]
    lines = []
    for w in args.workload.split(","):
        lines.append(json.dumps(run(w, libs, args.rounds, args.calls)))
        print(lines[-1], flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ab_correlate.json"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    if sys.argv[1:2] == ["--worker"]:
        worker(sys.argv[2], int(sys.argv[3]))
    else:
        main()
