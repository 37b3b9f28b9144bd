"""The float64 oracle of the weak grid and what its tests share.

integrate_weak restates gb200_acquire_grid_weak's profile with the oracle's own arithmetic: each millisecond m is wiped
off at its place in the block exactly as gypsum_oracle.integrate does, its samples are rolled by the code-Doppler shift
s_m = rint(m * N * f / f_L1), and bit phase j sums |coherent sum of segment k| over the segments starting at millisecond
j * T / B + k * T.  vector_weak is the same arithmetic batched for grids, in the manner of
semicoherent_support.vector_semicoherent.  synth_weak_iq plants satellites whose code runs at (1 + f / f_L1) * 1.023 MHz
and whose +-1 data bits change at their own code epochs."""
import math

import numpy as np

from acq_support import _replica_spectrum, by_doppler_column, check_records
from oracle import gypsum_oracle as o

F_L1 = 1575.42e6


def shift(m, n, f):
    """s_m, evaluated in the engine's order."""
    return np.rint(float(m) * n * f / 1575.42e6)


def weak_shape(n_ms, coherent_ms, bit_phases):
    """(phase step, K) of a window of n_ms milliseconds; ValueError when it breaks a rule of the weak grid."""
    if coherent_ms < 1 or bit_phases < 1 or coherent_ms % bit_phases:
        raise ValueError("bit_phases must divide coherent_ms")
    step = coherent_ms // bit_phases
    span = (bit_phases - 1) * step
    if n_ms < coherent_ms + span or (n_ms - span) % coherent_ms:
        raise ValueError("the window is not the phases' span plus whole segments")
    return step, (n_ms - span) // coherent_ms


def _wiped(data, fs, n, f, m):
    """Millisecond m wiped off at its place in the block (gypsum_oracle.integrate's carrier), rolled by s_m."""
    t = (np.arange(n) / fs) + ((m * n) / fs)
    return np.roll(data[m * n:(m + 1) * n] * np.exp(-1j * math.tau * f * t), int(shift(m, n, f)))


def integrate_weak(data, fs, n, doppler, prn, coherent_ms, bit_phases):
    """[bit_phases, n]: per bit phase j, sum_k |sum_t corr(aligned millisecond j * step + k * T + t)|."""
    step, k_count = weak_shape(len(data) // n, coherent_ms, bit_phases)
    out = np.zeros((bit_phases, n), dtype=np.float64)
    for j in range(bit_phases):
        for k in range(k_count):
            coh = np.zeros(n, dtype=complex)
            for t in range(coherent_ms):
                coh += o.correlate_1ms(_wiped(data, fs, n, doppler, j * step + k * coherent_ms + t), prn)
            out[j] += np.abs(coh)
    return out


def _weak_cols(x, fs, n, svs, dop, coherent_ms, bit_phases):
    uniq = sorted(set(svs))
    rows = [uniq.index(sv) for sv in svs]
    rep = np.stack([_replica_spectrum(sv, n) for sv in uniq])
    shape = (len(svs), bit_phases, len(dop))
    peak, arg, total, count = (np.zeros(shape), np.zeros(shape, np.int64), np.zeros(shape), np.zeros(shape, np.int64))
    step, k_count = weak_shape(len(x) // n, coherent_ms, bit_phases)
    for b, f in enumerate(dop):
        ffts = {}  # a millisecond's aligned spectrum is shared by the phases that overlap on it
        for j in range(bit_phases):
            acc = np.zeros((len(uniq), n))
            for k in range(k_count):
                spec = np.zeros(n, dtype=complex)
                for m in range(j * step + k * coherent_ms, j * step + (k + 1) * coherent_ms):
                    if m not in ffts:
                        ffts[m] = np.fft.fft(_wiped(x, fs, n, f, m))
                    spec += ffts[m]
                acc += np.abs(np.fft.ifft(spec[None, :] * rep, axis=-1))
            mx = acc.max(axis=1)
            peak[:, j, b], arg[:, j, b], total[:, j, b] = mx[rows], acc.argmax(axis=1)[rows], acc.sum(axis=1)[rows]
            count[:, j, b] = np.count_nonzero(acc == mx[:, None], axis=1)[rows]
    return peak, arg, total, count


def vector_weak(x, fs, n, svs, dop, coherent_ms, bit_phases):
    """(peak, argmax, sum, count) of every (SV, bit phase, Doppler) cell of one block's weak grid, each [len(svs),
    bit_phases, len(dop)].  Large grids are spread over the host's cores by Doppler column."""
    dop = np.asarray(dop, dtype=np.float64)
    return by_doppler_column(_weak_cols, dop.size, len(set(svs)) * dop.size * len(x) * bit_phases,
                             lambda p: (x, fs, n, list(svs), dop[p], coherent_ms, bit_phases))


def check_weak(rec, x, fs, n, svs, dop, coherent_ms, bit_phases, what, ref=None):
    """acq_support.check_records on one block's weak records [n_svs, B, D].  Returns the number of near-tie proofs."""
    ref = ref if ref is not None else vector_weak(x, fs, n, svs, dop, coherent_ms, bit_phases)
    return check_records(rec, ref, n, lambda i: integrate_weak(x, fs, n, dop[i[2]], o.replica(svs[i[0]], n), coherent_ms,
                                                               bit_phases)[i[1]], what)


def best_folded(peak):
    """k_best_bins' choice per row over the folded B * D axis: (bin, phase j, Doppler index d)."""
    flat = peak.reshape(peak.shape[:-2] + (-1,))
    b = np.argmax(flat, axis=-1)
    return b, b // peak.shape[-1], b % peak.shape[-1]


def synth_weak_iq(seed, n, n_ms, fs, planted, sigma=1.0):
    """complex64[n_ms * n]: complex gaussian noise * sigma plus, per planted (sv, doppler_hz, code_phase_samples,
    carrier_phase_rad, amplitude, bit_phase_ms, bits), a satellite whose code runs at (1 + f / f_L1) * 1.023 MHz (chip
    index ((1 + f / f_L1) * k - code_phase + 1/2) * 1023 / N at sample k, so its lag at the first sample is code_phase), times
    +-1 data bits that change at the code epochs e with (e - bit_phase_ms) % 20 == 0, on the carrier exp(+j(2 pi f t +
    phi)).  bits: None (random from the seed), "alternate" (+1, -1, ... from the first whole bit), or the signs
    themselves, one per bit from the one holding sample 0."""
    rng = np.random.default_rng(seed)
    total = n * n_ms
    x = (rng.standard_normal(total) + 1j * rng.standard_normal(total)) * (sigma / math.sqrt(2.0))
    k = np.arange(total, dtype=np.float64)
    for sv, f, tau, phi, amp, bit_phase, bits in planted:
        # chip edges half a sample before the samples, so that a small code Doppler of either sign keeps the sampled lag
        chip_pos = ((1.0 + f / F_L1) * k - tau + 0.5) * (o.PRN_CHIP_COUNT / n)
        chip = np.floor(chip_pos).astype(np.int64)
        code = 2.0 * o.ca_code(sv)[chip % o.PRN_CHIP_COUNT] - 1.0
        bit = np.floor_divide(np.floor_divide(chip, o.PRN_CHIP_COUNT) - bit_phase, 20)
        bit -= bit[0]
        n_bits = int(bit[-1]) + 1
        if bits is None:
            signs = rng.integers(0, 2, size=n_bits) * 2.0 - 1.0
        elif isinstance(bits, str) and bits == "alternate":
            signs = np.where(np.arange(n_bits) % 2 == 0, 1.0, -1.0)
        else:
            signs = np.asarray(bits, dtype=np.float64)[:n_bits]
        x = x + amp * code * signs[bit] * np.exp(1j * (math.tau * f * k / fs + phi))
    return x.astype(np.complex64)


def search_decision(peak, arg, dop):
    """(planted SV's best folded bin as (phase, Doppler Hz), its code phase there, whether its best peak ranks above every
    noise PRN's) -- the planted SV in row 0."""
    b, j, d = best_folded(peak[0])
    return (int(j), float(dop[d])), int(arg[0, j, d]), bool(peak[0].max() > peak[1:].max())


# The bit-phase case: a strong satellite whose bits alternate every 20 ms with edges at epochs 10, 30, 50, ... -- in the
# middle of every 20-ms segment of bit phase 0, which then cancels, and on the boundaries of phase 1 of B = 2 (phase 2 of
# B = 4).
BIT_FS, BIT_N = 2046000, 2046
BIT_SV, BIT_DOPPLER, BIT_CODE_PHASE, BIT_AMP = 7, 1000.0, 2, 0.05
BIT_SVS = [BIT_SV, 4, 15, 21]
BIT_BINS = np.arange(850.0, 1151.0, 25.0)
BIT_MS = 100  # T = 20: K = 5 at B = 1, 4 at B = 2 and 4


def bit_phase_iq(n_ms=BIT_MS):
    return synth_weak_iq(11, BIT_N, n_ms, BIT_FS, [(BIT_SV, BIT_DOPPLER, BIT_CODE_PHASE, 0.3, BIT_AMP, 10, "alternate")])
