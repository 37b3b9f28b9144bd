"""The float64 oracle of the semi-coherent grid and what its tests share.

integrate_semicoherent restates gb200_acquire_grid_semicoherent's profile on the oracle's own integrate: segment k's
coherent sum is integrate(COHERENT, ...) over a window whose milliseconds before the segment are zero, so each of its
milliseconds is wiped off at its place in the window (the carrier phase is continuous, as on the device) and the zero
milliseconds add exact zeros.  vector_semicoherent is the same arithmetic batched for grids, in the manner of
acq_support.vector_grid: per (Doppler, segment) the wiped-off milliseconds' forward FFTs are summed and one batched inverse
FFT runs over every SV."""
import math

import numpy as np

from acq_support import _replica_spectrum, by_doppler_column, check_records
from oracle import gypsum_oracle as o


def integrate_semicoherent(data, fs, n, doppler, prn, coherent_ms):
    """sum_k |integrate(COHERENT, segment k of coherent_ms milliseconds)|.  The window must be a whole number of
    segments."""
    n_ms = len(data) // n
    if coherent_ms < 1 or n_ms % coherent_ms:
        raise ValueError("the window must be a whole number of coherent_ms-ms segments")
    out = np.zeros(n, dtype=np.float64)
    seg = coherent_ms * n
    for k in range(n_ms // coherent_ms):
        window = np.zeros((k + 1) * seg, dtype=data.dtype)
        window[k * seg:] = data[k * seg:(k + 1) * seg]
        out += np.abs(o.integrate(o.COHERENT, window, fs, n, doppler, prn))
    return out


def _semi_cols(x, fs, n, svs, dop, coherent_ms):
    uniq = sorted(set(svs))
    rows = [uniq.index(sv) for sv in svs]
    rep = np.stack([_replica_spectrum(sv, n) for sv in uniq])
    shape = (len(svs), len(dop))
    peak, arg, total, count = (np.zeros(shape), np.zeros(shape, np.int64), np.zeros(shape), np.zeros(shape, np.int64))
    n_ms = len(x) // n
    for b, f in enumerate(dop):
        acc = np.zeros((len(uniq), n))
        for k in range(n_ms // coherent_ms):
            spec = np.zeros(n, dtype=complex)
            for i in range(k * coherent_ms, (k + 1) * coherent_ms):
                t = (np.arange(n) / fs) + ((i * n) / fs)
                spec += np.fft.fft(x[i * n:(i + 1) * n] * np.exp(-1j * math.tau * f * t))
            acc += np.abs(np.fft.ifft(spec[None, :] * rep, axis=-1))
        mx = acc.max(axis=1)
        peak[:, b], arg[:, b], total[:, b] = mx[rows], acc.argmax(axis=1)[rows], acc.sum(axis=1)[rows]
        count[:, b] = np.count_nonzero(acc == mx[:, None], axis=1)[rows]
    return peak, arg, total, count


def vector_semicoherent(x, fs, n, svs, dop, coherent_ms):
    """(peak, argmax, sum, count) of every (SV, Doppler) cell of one block's semi-coherent grid, each [len(svs),
    len(dop)].  Large grids are spread over the host's cores by Doppler column."""
    dop = np.asarray(dop, dtype=np.float64)
    return by_doppler_column(_semi_cols, dop.size, len(set(svs)) * dop.size * len(x),
                             lambda p: (x, fs, n, list(svs), dop[p], coherent_ms))


def check_semicoherent(rec, x, fs, n, svs, dop, coherent_ms, what, ref=None):
    """acq_support.check_records for one block of a semi-coherent grid.  Returns the near-tie proofs."""
    ref = ref if ref is not None else vector_semicoherent(x, fs, n, svs, dop, coherent_ms)
    return check_records(rec, ref, n, lambda i: integrate_semicoherent(x, fs, n, dop[i[1]], o.replica(svs[i[0]], n),
                                                                       coherent_ms), what)


def best_bins(peak):
    """k_best_bins' choice per row: the first bin with the largest peak."""
    return np.argmax(peak, axis=-1)


# The sensitivity case: one satellite at C/N0 = a^2 * fs for noise of unit variance (sigma = 1), data bits every 20 ms
# from the first sample (so aligned to 10-ms segments), searched among noise-only PRNs over a 50-Hz grid.
SENS_FS, SENS_N = 2046000, 2046
SENS_SEED, SENS_AMP = 5, 0.023  # C/N0 = 0.023^2 * 2.046e6 = 1082 Hz = 30.3 dB-Hz
SENS_SV, SENS_DOPPLER, SENS_CODE_PHASE = 12, 1234.0, 1501
SENS_SVS = [SENS_SV, 3, 8, 17, 22, 30]
SENS_BINS = np.arange(750.0, 1751.0, 50.0)


def sensitivity_iq():
    return o.synth_iq(SENS_SEED, SENS_N, 20, SENS_FS, [(SENS_SV, SENS_DOPPLER, SENS_CODE_PHASE, 0.4, SENS_AMP)],
                      nav_bits=True)


def search_decision(peak, arg):
    """(planted SV's best bin, its code phase there, whether its best peak ranks above every noise PRN's)."""
    b = int(np.argmax(peak[0]))
    return b, int(arg[0, b]), bool(peak[0].max() > peak[1:].max())
