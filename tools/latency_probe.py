"""Single-block host-to-host latency of the config-2 grid, by entry point."""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from gypsum_b200 import _native  # noqa: E402
from gypsum_b200.gps_ca_prn_codes import ca_code_chips  # noqa: E402

N, FS = 2046, 2046000
eng = _native.Engine(FS, N)
eng.set_replicas(np.stack([ca_code_chips(sv) for sv in range(1, 33)]).astype(np.uint8))
x = torch.randn(64, N * 2).pin_memory()
prn = np.arange(32, dtype=np.int32)
dop = np.arange(-10000.0, 10001.0, 500.0)
out = np.empty((1, 32, 41), dtype=_native.RECORD_DTYPE)


def med(fn, n=600):
    ts = []
    for k in range(n):
        t0 = time.perf_counter()
        fn(k)
        ts.append(time.perf_counter() - t0)
    return 1e6 * float(np.median(ts[50:]))


def host_call(k):
    eng.acquire_grid_host(x.data_ptr() + (k % 64) * N * 8, 1, 1, prn, dop, 2, out=out)


out_pinned = torch.empty(out.nbytes, dtype=torch.uint8).pin_memory().numpy().view(_native.RECORD_DTYPE).reshape(out.shape)


def host_call_pinned(k):
    eng.acquire_grid_host(x.data_ptr() + (k % 64) * N * 8, 1, 1, prn, dop, 2, out=out_pinned)


def two_calls(k):
    eng.upload_iq_ptr(x.data_ptr() + (k % 64) * N * 8, N)
    eng.acquire_grid(1, 1, prn, dop, 2, out=out)


print("acquire_grid_host us", med(host_call), "with a pinned record buffer us", med(host_call_pinned),
      "upload+acquire_grid us", med(two_calls))
host_call(0)
assert out_pinned.tobytes() != out.tobytes() or True
host_call_pinned(0)
assert np.array_equal(out_pinned["argmax"], out["argmax"]) and np.array_equal(out_pinned["peak"], out["peak"])
eng.enable_kernel_timing(True)
for k in range(100):
    two_calls(k)
a, na = eng.kernel_timing(0)
b, nb = eng.kernel_timing(1)
print("kernels: doppler_spectra us", 1e3 * a / na, "correlate us", 1e3 * b / nb)
