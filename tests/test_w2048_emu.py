"""The one-warp correlate kernel's per-CTA odd-parity twiddle table and whole-transform peak reduction, run by the host lane
emulator (tests/emu/w2048_emu.cu): each gives bit for bit what the per-transform twiddle product and the two half-transform
reductions it replaces give, and matches numpy's transform and np.max / np.argmax / count / sum.  No GPU needed."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def w2048_emu(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "emu", "w2048_emu.cu")
    out = str(tmp_path_factory.mktemp("w2048_emu") / "libw2048emu.so")
    subprocess.run(["nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-o", out, src], check=True,
                   capture_output=True)
    lib = C.CDLL(out)
    lib.emu_ifft2048_odd.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    lib.emu_peak.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_int),
                             C.POINTER(C.c_double)]
    return lib


@pytest.mark.parametrize("seed", [5, 6])
def test_odd_twiddle_table_is_bit_identical_and_matches_numpy(w2048_emu, seed):
    rng = np.random.default_rng(seed)
    ye = (rng.standard_normal(1024) + 1j * rng.standard_normal(1024)).astype(np.complex64)
    yo = (rng.standard_normal(1024) + 1j * rng.standard_normal(1024)).astype(np.complex64)
    outs = []
    for table in (0, 1):
        out = np.zeros(1024, np.complex64)
        w2048_emu.emu_ifft2048_odd(ye.ctypes.data, yo.ctypes.data, table, out.ctypes.data)
        outs.append(out)
    assert outs[0].tobytes() == outs[1].tobytes()
    y = np.empty(2048, complex)
    y[0::2], y[1::2] = ye, yo
    ref = (np.fft.ifft(y) * 2048)[:1024]
    assert np.abs(outs[1] - ref).max() <= 5e-7 * np.abs(ref).max()


def _peak(lib, v, n_r, fast):
    mx, idx, cnt, total = C.c_float(), C.c_int(), C.c_int(), C.c_double()
    lib.emu_peak(v.ctypes.data, n_r, fast, C.byref(mx), C.byref(idx), C.byref(cnt), C.byref(total))
    return mx.value, idx.value, cnt.value, total.value


@pytest.mark.parametrize("n_r,levels,seed", [(1, 0, 0), (2, 0, 1), (2, 40, 2), (2, 3, 3), (16, 0, 4), (16, 7, 5)])
def test_thread_peak32_is_bit_identical_and_matches_numpy(w2048_emu, n_r, levels, seed):
    """levels > 0 quantizes the profile so that the maximum is tied many times, across lanes, halves and branches."""
    rng = np.random.default_rng(seed)
    v = rng.random((n_r, 1024), dtype=np.float32) * 100
    if levels:
        v = np.floor(v * levels / 100).astype(np.float32)
    v[:, 1023] = 1e6  # lag 1023 (lane 31, k = 31) does not exist and must be ignored
    v = np.ascontiguousarray(v)
    slow, fast = _peak(w2048_emu, v, n_r, 0), _peak(w2048_emu, v, n_r, 1)
    assert np.float32(slow[0]).tobytes() == np.float32(fast[0]).tobytes() and slow[1:3] == fast[1:3]
    assert np.float64(slow[3]).tobytes() == np.float64(fast[3]).tobytes()
    prof = v[:, :1023].T.reshape(-1)  # profile index s q + r
    assert fast[0] == prof.max() and fast[1] == int(prof.argmax())
    assert fast[2] == int(np.count_nonzero(prof == prof.max()))
    assert abs(fast[3] - prof.astype(np.float64).sum()) <= 2e-6 * fast[3]
