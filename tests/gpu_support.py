"""What the GPU test modules share: the acquisition, tracking and position-fix modules build their engines here, and the
host-side modules their stream attributes.  gypsum_b200 is imported inside, so collection works without the library."""
import os
import subprocess
import sys

import numpy as np

from oracle import gypsum_oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def all_chips():
    """The C/A codes of PRN 1 to 32, one row of chips per satellite: row a holds SV a + 1."""
    return np.stack([o.ca_code(sv) for sv in range(1, 33)]).astype(np.uint8)


def make_engine(fs, n):
    """An engine at fs samples per second and n samples per millisecond, holding the C/A codes of PRN 1 to 32."""
    from gypsum_b200 import _native

    e = _native.Engine(fs, n)
    e.set_replicas(all_chips())
    return e


class Attrs:
    """The stream attributes the drop-in classes read from a sample provider."""

    def __init__(self, fs, n):
        self.samples_per_second = fs
        self.samples_per_prn_transmission = n


class EngineCache:
    """One engine per n samples per millisecond (fs = 1000 n), made by make_engine on first use and kept until close()."""

    def __init__(self):
        self._engines = {}

    def __call__(self, n):
        if n not in self._engines:
            self._engines[n] = make_engine(1000 * n, n)
        return self._engines[n]

    def close(self):
        for e in self._engines.values():
            e.close()
        self._engines.clear()


def run_child(script, *args, ok=None, timeout=600):
    """Runs `python -c script ROOT *args` in a process of its own and asserts that it exits with 0 and, if ok is given,
    that it printed ok.  A child keeps a fault on a path no other test has run out of the CUDA context of the tests
    after it, and reads the library's environment knobs afresh."""
    proc = subprocess.run([sys.executable, "-c", script, ROOT, *map(str, args)], capture_output=True, text=True,
                          timeout=timeout)
    assert proc.returncode == 0, proc.stderr[-2000:]
    if ok is not None:
        assert ok in proc.stdout, proc.stderr[-2000:]
