"""Builds the in-tree CUDA shared library (sm_90a only) with nvcc.  Used by __graft_entry__.build()."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libgypsum_b200.so")
SOURCES = ["kernels.cu", "tracker.cu", "bits.cu", "nav.cu", "orbit.cu", "fix.cu", "velocity.cu", "signal.cu", "fused.cu", "engine.cu", "receiver.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "-shared", "-cudart", "static",
]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libgypsum_b200.so")


def is_stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "gypsum_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps if os.path.isfile(d))


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return LIB
    cmd = [_nvcc(), *NVCC_FLAGS, "-o", LIB, *[os.path.join(CSRC, s) for s in SOURCES]]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + proc.stdout + proc.stderr)
    if verbose:
        print(proc.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
