"""The one-warp correlate kernel's exact 1023-point transforms and peak reduction (warp_pfa.cuh), run by the host lane emulator
(tests/emu/pfa_emu.cu): forward and inverse DFT-1023 in the permuted bin order against numpy, the polyphase correlation they
carry at N = 1023 s against a float64 circular correlation, and the record of permuted lags against np.max / first argmax /
count / sum.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

from hostbuild import host_library

K1, K2 = np.meshgrid(np.arange(32), np.arange(33), indexing="ij")
# pidx(k2, k1) of every (k1, k2) and the DFT bin stored there
PIDX = ((((K2 >> 1) * 32 + K1) << 1) | (K2 & 1)).ravel()
BIN = ((528 * K1 + 496 * K2) % 1023).ravel()
VALID = (K1 < 31).ravel()


@pytest.fixture(scope="module")
def pfa_emu():
    lib = host_library("pfa_emu")
    lib.emu_dft1023_fwd.argtypes = [C.c_void_p, C.c_void_p]
    lib.emu_dft1023_inv.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.emu_peak.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_int),
                             C.POINTER(C.c_double)]
    return lib


def _fwd(lib, z):
    z = np.ascontiguousarray(z, np.complex64)
    spec = np.full(1088, np.nan, np.complex64)
    lib.emu_dft1023_fwd(z.ctypes.data, spec.ctypes.data)
    return spec


def _inv(lib, spec, rep):
    out = np.zeros(1023, np.complex64)
    lib.emu_dft1023_inv(np.ascontiguousarray(spec).ctypes.data, np.ascontiguousarray(rep, np.complex64).ctypes.data,
                        out.ctypes.data)
    return out


def _permuted(x):
    """A length-1023 spectrum in the kernel's storage order (zero in the unused slots)."""
    out = np.zeros(1088, np.complex64)
    out[PIDX[VALID]] = x[BIN[VALID]]
    return out


@pytest.mark.parametrize("seed", [1, 2])
def test_forward_and_inverse_dft1023_match_numpy(pfa_emu, seed):
    rng = np.random.default_rng(seed)
    z = (rng.standard_normal(1023) + 1j * rng.standard_normal(1023)).astype(np.complex64)
    spec = _fwd(pfa_emu, z)
    ref = np.fft.fft(z.astype(complex))
    assert np.abs(spec[PIDX[VALID]] - ref[BIN[VALID]]).max() <= 5e-7 * np.abs(ref).max()
    assert (spec[PIDX[~VALID]] == 0).all()  # every slot the inverse reads is written
    x = (rng.standard_normal(1023) + 1j * rng.standard_normal(1023)).astype(np.complex64)
    ones = _permuted(np.ones(1023, np.complex64))
    out = _inv(pfa_emu, _permuted(x), ones)
    ref = np.fft.ifft(x.astype(complex)) * 1023
    assert np.abs(out - ref).max() <= 5e-7 * np.abs(ref).max()


@pytest.mark.parametrize("s", [1, 2, 3, 16])
def test_polyphase_correlation_matches_float64(pfa_emu, s):
    """|corr| of a millisecond against a chip replica at N = 1023 s: polyphase boxcar, forward, replica product, inverse."""
    rng = np.random.default_rng(100 + s)
    n = 1023 * s
    chips = rng.integers(0, 2, 1023)
    c = np.where(chips == 1, 1.0, -1.0)
    y = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    rep = _permuted(np.conj(np.fft.fft(c)) / 1023)
    got = np.zeros(n)
    for r in range(s):
        z = np.array([y[(s * m + r + np.arange(s)) % n].astype(complex).sum() for m in range(1023)])
        got[r::s] = np.abs(_inv(pfa_emu, _fwd(pfa_emu, z), rep))
    p = np.repeat(c, s)
    ref = np.abs(np.fft.ifft(np.fft.fft(y.astype(complex)) * np.conj(np.fft.fft(p))))
    assert np.abs(got - ref).max() <= 1e-6 * ref.max()


@pytest.mark.parametrize("n_r,levels", [(1, 0), (1, 5), (2, 3), (16, 4), (16, 0)])
@pytest.mark.parametrize("seed", [3, 4])
def test_peak_of_permuted_lags_matches_numpy(pfa_emu, n_r, levels, seed):
    """Max, first profile index s q + r of the max, count of the max and sum; levels > 0 draws from few values, so the max
    is tied at many lags and branches."""
    rng = np.random.default_rng(seed)
    v = rng.integers(0, levels, (n_r, 1023)).astype(np.float32) if levels else rng.random((n_r, 1023), np.float32)
    mx, idx, cnt, total = C.c_float(), C.c_int(), C.c_int(), C.c_double()
    pfa_emu.emu_peak(np.ascontiguousarray(v).ctypes.data, n_r, C.byref(mx), C.byref(idx), C.byref(cnt), C.byref(total))
    prof = v.T.ravel()  # profile index s q + r
    assert mx.value == prof.max()
    assert idx.value == int(np.argmax(prof))
    assert cnt.value == int((prof == prof.max()).sum())
    assert abs(total.value - prof.astype(np.float64).sum()) <= 1e-6 * prof.astype(np.float64).sum()
