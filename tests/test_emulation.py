"""The product's lane-level device functions (warp FFT-1024, polyphase split, padded-FFT correlation, replica
spectra) executed on the CPU by the lane emulator and compared with the oracle.  No GPU needed."""
import ctypes

import numpy as np
import pytest

from oracle import gypsum_oracle as o


@pytest.mark.parametrize("inverse", [0, 1])
def test_warp_fft1024(emu_lib, inverse):
    rng = np.random.default_rng(inverse)
    x = (rng.standard_normal(1024) + 1j * rng.standard_normal(1024)).astype(np.complex64)
    y = x.copy()
    emu_lib.emu_fft1024(y.ctypes.data_as(ctypes.c_void_p), inverse)
    ref = np.fft.ifft(x.astype(complex)) * 1024 if inverse else np.fft.fft(x.astype(complex))
    assert np.abs(y - ref).max() <= 5e-7 * np.abs(ref).max()


@pytest.mark.parametrize("n,n_ms,sv,f", [(2046, 1, 25, 1500.0), (2046, 3, 7, -3250.0), (4092, 2, 11, 4875.5),
                                         (16368, 1, 32, -250.0), (1023, 2, 1, 700.0), (3069, 1, 19, 10000.0),
                                         (5115, 2, 14, 2345.0), (6138, 1, 7, -4250.0), (8184, 3, 21, 6500.0),
                                         (10230, 1, 30, -1250.0), (12276, 2, 2, 9000.0)])
def test_polyphase_correlation_matches_oracle(emu_lib, n, n_ms, sv, f):
    emu_lib.emu_cell_profile.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.c_double,
                                         ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    rec = np.zeros(1, dtype=[("peak", "<f4"), ("argmax", "<i4"), ("sum", "<f8"), ("count", "<i4"), ("pr", "<f4"),
                             ("pi", "<f4"), ("pad", "<i4")])
    fs = n * 1000
    iq = o.synth_iq(1, n, n_ms, fs, [(sv, f + 3, n - 7, 0.3, 0.3)])
    chips = o.ca_code(sv).astype(np.uint8)
    prn = o.replica(sv, n)
    nc = np.zeros(n, np.float32)
    emu_lib.emu_cell_profile(iq.ctypes.data, n, n_ms, float(fs), float(f), chips.ctypes.data, 2, nc.ctypes.data, rec.ctypes.data)
    ref = o.integrate(o.NON_COHERENT, iq, fs, n, f, prn)
    assert np.abs(nc - ref).max() <= 1e-6 * ref.max()
    assert nc.argmax() == ref.argmax() == n - 7
    # the branch-free per-thread reduction + merges reproduce np.max / np.argmax / count / sum of the profile
    assert rec["peak"][0] == nc.max() and rec["argmax"][0] == int(nc.argmax())
    assert rec["count"][0] == int(np.count_nonzero(nc == nc.max()))
    assert abs(rec["sum"][0] - nc.astype(np.float64).sum()) <= 2e-6 * rec["sum"][0]
    co = np.zeros(n, np.complex64)
    emu_lib.emu_cell_profile(iq.ctypes.data, n, n_ms, float(fs), float(f), chips.ctypes.data, 1, co.ctypes.data, None)
    refc = o.integrate(o.COHERENT, iq, fs, n, f, prn)
    assert np.abs(co - refc).max() <= 1e-6 * np.abs(refc).max()


def test_one_warp_pruned_ifft2048(emu_lib):
    """w2048_phase1/2: out[k] = sum_g Y[g] exp(+2 pi i g k / 2048) for k < 1024, Y[2f+h] = Y_h[f]."""
    rng = np.random.default_rng(5)
    ye = (rng.standard_normal(1024) + 1j * rng.standard_normal(1024)).astype(np.complex64)
    yo = (rng.standard_normal(1024) + 1j * rng.standard_normal(1024)).astype(np.complex64)
    out = np.zeros(1024, np.complex64)
    emu_lib.emu_ifft2048_pruned(ye.ctypes.data_as(ctypes.c_void_p), yo.ctypes.data_as(ctypes.c_void_p),
                                out.ctypes.data_as(ctypes.c_void_p))
    y = np.empty(2048, complex)
    y[0::2], y[1::2] = ye, yo
    ref = (np.fft.ifft(y) * 2048)[:1024]
    assert np.abs(out - ref).max() <= 5e-7 * np.abs(ref).max()
