"""A/B timing of library builds on bench.py's config-2 call: 256 blocks x 32 PRN x 41 Doppler, 1 ms, from a device-resident IQ
ring larger than L2 (bench.make_ring, seed 1000).  Every build runs in its own child process (GB200_LIB selects the library);
the builds take turns for --rounds rounds, so clock and neighbour drift spread over all of them.

usage: python tools/ab_correlate.py LIB_A LIB_B [LIB ...] [--rounds 5] [--calls 24] [--out DIR]

Prints one JSON line: per build the per-launch ms of doppler_spectra and correlate (enable_kernel_timing; median, min, max over
rounds) and the call time (CUDA events), the card's name, power limit and SM clock (sampled during the rounds), and, for every
build after the first, whether its records on the first ring slot are byte-identical to LIB_A's -- or else the largest
|peak| and |sum| difference over max(peak).  --out also writes that line to DIR/ab_correlate.json."""
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


def worker(calls: int) -> None:
    """Child: one library build, `calls` calls per round.  Reads 'round' / 'records PATH' / 'quit' lines on stdin and
    answers each with one JSON line."""
    import torch

    import bench
    from gypsum_b200 import _native
    from gypsum_b200.gps_ca_prn_codes import ca_code_chips

    B = 256
    block_bytes = bench.N * 8
    ring_blocks = (bench.L2_BYTES // block_bytes // B + 2) * B  # bench.py's ring: larger than L2
    ring = torch.from_numpy(bench.make_ring(ring_blocks, seed=1000)).cuda()
    n_slots = ring_blocks // B
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    eng = _native.Engine(bench.FS, bench.N)
    eng.set_replicas(np.stack([ca_code_chips(sv) for sv in range(1, 33)]).astype(np.uint8))
    eng.set_stream(stream.cuda_stream)
    prn = np.arange(bench.N_PRN, dtype=np.int32)
    dop = np.ascontiguousarray(bench.DOPPLERS, dtype=np.float64)
    rec = torch.empty(B * bench.N_PRN * dop.size * 32, dtype=torch.uint8, device="cuda")

    def call(j: int) -> None:
        eng.bind_iq_device(ring.data_ptr() + (j % n_slots) * B * block_bytes, B * bench.N)
        eng.acquire_grid_device(B, 1, prn, dop, _native.NON_COHERENT, rec.data_ptr())

    for j in range(2 * n_slots):  # warm-up: every slot once, twice
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
        elif cmd[0] == "records":
            call(0)
            torch.cuda.synchronize()
            np.save(cmd[1], rec.cpu().numpy())
            print(json.dumps({"saved": cmd[1]}), flush=True)
        else:
            break
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


def compare(a: np.ndarray, b: np.ndarray) -> dict:
    if a.tobytes() == b.tobytes():
        return {"byte_identical": True}
    from gypsum_b200 import _native

    ra, rb = a.view(_native.RECORD_DTYPE), b.view(_native.RECORD_DTYPE)
    scale = float(np.max(ra["peak"]))
    return {"byte_identical": False,
            "max_peak_diff_over_max_peak": float(np.max(np.abs(ra["peak"] - rb["peak"]))) / scale,
            "max_sum_diff_over_max_peak": float(np.max(np.abs(ra["sum"] - rb["sum"]))) / scale,
            "argmax_mismatches": int(np.count_nonzero(ra["argmax"] != rb["argmax"]))}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="+")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=24)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if len(args.libs) < 2:
        ap.error("give at least two library builds")
    libs = [os.path.abspath(p) for p in args.libs]
    children = []
    for lib in libs:
        env = dict(os.environ, GB200_LIB=lib)
        children.append(subprocess.Popen([sys.executable, os.path.abspath(__file__), "--worker", str(args.calls)], env=env, text=True,
                                         stdin=subprocess.PIPE, stdout=subprocess.PIPE))

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
        for _ in range(args.rounds):
            for i, c in enumerate(children):
                runs[i].append(ask(c, "round"))
        mhz = sampler.stop()
        with tempfile.TemporaryDirectory() as tmp:
            recs = []
            for i, c in enumerate(children):
                path = os.path.join(tmp, f"rec{i}.npy")
                ask(c, f"records {path}")
                recs.append(np.load(path))
        result = {"card": info, "sm_mhz_during_rounds": spread([float(m) for m in mhz]) if mhz else None,
                  "rounds": args.rounds, "calls_per_round": args.calls, "builds": []}
        for i, lib in enumerate(libs):
            r = runs[i]
            b = {"lib": os.path.relpath(lib, ROOT), "call_ms": spread([x["call_ms"] for x in r]),
                 "spectra_ms": spread([x["spectra_ms"] for x in r]), "correlate_ms": spread([x["correlate_ms"] for x in r])}
            if i:
                b["correlate_change_vs_first"] = b["correlate_ms"]["median"] / result["builds"][0]["correlate_ms"]["median"] - 1
                b["records_vs_first"] = compare(recs[0], recs[i])
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
    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ab_correlate.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    if sys.argv[1:2] == ["--worker"]:
        worker(int(sys.argv[2]))
    else:
        main()
