"""ctypes binding of include/gypsum_b200.h.  The product path: if the shared library is missing this raises --
there is no numpy/CPU route behind it."""
from __future__ import annotations

import ctypes as C
import os
import weakref

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("GB200_LIB") or os.path.join(_HERE, "libgypsum_b200.so")  # GB200_LIB: experiment builds

OK, EINVAL, ECUDA, ESTATE = 0, 1, 2, 3
COHERENT, NON_COHERENT = 1, 2

RECORD_DTYPE = np.dtype(
    [("peak", "<f4"), ("argmax", "<i4"), ("sum", "<f8"), ("count", "<i4"), ("probe_re", "<f4"), ("probe_im", "<f4"),
     ("reserved", "<i4")]
)
assert RECORD_DTYPE.itemsize == 32
TRACK_DTYPE = np.dtype(
    [("doppler", "<f8"), ("carrier_phase", "<f8"), ("error", "<f8"), ("disc", "<f8"), ("phase_acc", "<f8"),
     ("doppler_hist", "<f8"), ("carrier_phase_hist", "<f8"), ("peak_re", "<f4"), ("peak_im", "<f4"), ("strength", "<f4"), ("early_re", "<f4"), ("early_im", "<f4"),
     ("late_re", "<f4"), ("late_im", "<f4"), ("code_phase", "<i4"), ("symbol", "<i4"), ("locked", "<i4"), ("lost", "<i4"),
     ("peak_offset", "<i4"), ("reserved0", "<i4"), ("reserved1", "<i4")]
)
assert TRACK_DTYPE.itemsize == 112
ACQ_DTYPE = np.dtype([("doppler", "<f8"), ("strength", "<f8"), ("probe_re", "<f4"), ("probe_im", "<f4"),
                      ("code_phase", "<i4"), ("reserved", "<i4")])
assert ACQ_DTYPE.itemsize == 32
BEST_DTYPE = np.dtype([("doppler", "<f8"), ("strength", "<f8"), ("peak", "<f4"), ("code_phase", "<i4"), ("bin", "<i4"),
                       ("reserved", "<i4")])  # gb200_best_record
assert BEST_DTYPE.itemsize == 32

# every symbol include/gypsum_b200.h declares: name -> (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    "gb200_abi_version": (C.c_int, []),
    "gb200_create": (C.c_int, [C.c_int, C.c_int, C.c_int, C.POINTER(_P)]),
    "gb200_destroy": (C.c_int, [_P]),
    "gb200_last_error": (C.c_char_p, [_P]),
    "gb200_set_stream": (C.c_int, [_P, _P]),
    "gb200_set_replicas": (C.c_int, [_P, _P, C.c_int]),
    "gb200_upload_iq": (C.c_int, [_P, _P, C.c_int64]),
    "gb200_bind_iq_device": (C.c_int, [_P, _P, C.c_int64]),
    "gb200_acquire_grid": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, _P]),
    "gb200_acquire_grid_device": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, _P]),
    "gb200_acquire_grid_host": (C.c_int, [_P, _P, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, _P]),
    "gb200_acquire_grid_best": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, _P]),
    "gb200_acquire_grid_best_device": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, _P]),
    "gb200_acquire_grid_semicoherent": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, _P]),
    "gb200_acquire_grid_semicoherent_device": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, _P]),
    "gb200_acquire_grid_semicoherent_best": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, _P]),
    "gb200_acquire_grid_semicoherent_best_device": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, _P]),
    "gb200_acquire_grid_weak": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, _P]),
    "gb200_acquire_grid_weak_device": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, _P]),
    "gb200_acquire_grid_weak_best": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, _P]),
    "gb200_acquire_grid_weak_best_device": (C.c_int, [_P, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, _P]),
    "gb200_ring_create": (C.c_int, [_P, C.c_int, C.POINTER(_P)]),
    "gb200_ring_destroy": (C.c_int, [_P]),
    "gb200_ring_append": (C.c_int, [_P, _P, C.c_int]),
    "gb200_ring_bind_newest": (C.c_int, [_P, C.c_int]),
    "gb200_ring_appended": (C.c_int, [_P, C.POINTER(C.c_int64)]),
    "gb200_acquire_cells": (C.c_int, [_P, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P]),
    "gb200_detect": (C.c_int, [_P, C.c_int, _P, C.c_int, _P]),
    "gb200_correlation_profile": (C.c_int, [_P, C.c_int, C.c_double, C.c_int, C.c_int, _P]),
    "gb200_correlation_profile_replica": (C.c_int, [_P, _P, C.c_double, C.c_int, C.c_int, _P]),
    "gb200_tracker_create": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, C.POINTER(_P)]),
    "gb200_tracker_destroy": (C.c_int, [_P]),
    "gb200_tracker_process": (C.c_int, [_P, C.c_int, _P, _P, _P]),
    "gb200_tracker_process_device": (C.c_int, [_P, C.c_int, _P, _P]),
    "gb200_tracker_get_state": (C.c_int, [_P, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double),
                                          C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "gb200_tracker_set_state": (C.c_int, [_P, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int32]),
    "gb200_tracker_create_pool": (C.c_int, [_P, C.c_int, C.POINTER(_P)]),
    "gb200_tracker_reset_channel": (C.c_int, [_P, C.c_int, C.c_int32, C.c_double, C.c_double, C.c_int32]),
    "gb200_tracker_process_channels": (C.c_int, [_P, C.c_int, _P, C.c_int, _P, C.c_int, _P, _P]),
    "gb200_tracker_undo_channel": (C.c_int, [_P, C.c_int]),
    "gb200_grid_stream_create": (C.c_int, [_P, C.c_int, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, C.c_int, C.POINTER(_P)]),
    "gb200_grid_stream_submit": (C.c_int, [_P, _P, _P]),
    "gb200_grid_stream_collect": (C.c_int, [_P]),
    "gb200_grid_stream_destroy": (C.c_int, [_P]),
    "gb200_tracker_integrate_bits": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, C.c_int32, _P]),
    "gb200_tracker_bit_state": (C.c_int, [_P, C.c_int, _P]),
    "gb200_tracker_decode_subframes": (C.c_int, [_P, _P, _P, C.c_int32, _P, C.c_int32, _P]),
    "gb200_tracker_subframe_state": (C.c_int, [_P, C.c_int, _P]),
    "gb200_tracker_parse_subframes": (C.c_int, [_P, _P, _P, C.c_int32, _P, _P, C.c_int32, _P, C.c_int32, _P]),
    "gb200_tracker_orbit_state": (C.c_int, [_P, C.c_int, _P, C.POINTER(C.c_uint32), C.POINTER(C.c_int64),
                                            C.POINTER(C.c_int32)]),
    "gb200_tracker_observations": (C.c_int, [_P, _P]),
    "gb200_tracker_observations_device": (C.c_int, [_P, _P]),
    "gb200_tracker_position_fixes": (C.c_int, [_P, _P, _P]),
    "gb200_tracker_position_fixes_device": (C.c_int, [_P, _P, _P]),
    "gb200_tracker_receiver_state": (C.c_int, [_P, C.POINTER(C.c_double), C.POINTER(C.c_int32), _P]),
    "gb200_tracker_fix_repairs": (C.c_int, [_P, C.POINTER(C.c_int64)]),
    "gb200_tracker_set_fix_solver": (C.c_int, [_P, C.c_int]),
    "gb200_tracker_set_code_phase_mode": (C.c_int, [_P, C.c_int]),
    "gb200_tracker_velocity_fixes": (C.c_int, [_P, _P, _P, _P]),
    "gb200_tracker_velocity_fixes_device": (C.c_int, [_P, _P, _P, _P]),
    "gb200_tracker_signal_windows": (C.c_int, [_P, C.c_int, _P, C.c_int32, _P, _P, C.c_int32, _P]),
    "gb200_tracker_chain_sizes": (C.c_int, [_P, _P]),
    "gb200_set_fused": (C.c_int, [_P, C.c_int]),
    "gb200_launch_count": (C.c_int, [_P, C.POINTER(C.c_int64)]),
    "gb200_enable_kernel_timing": (C.c_int, [_P, C.c_int]),
    "gb200_kernel_timing": (C.c_int, [_P, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_int64)]),
}

_lib = None


class NativeLibraryMissing(ImportError):
    pass


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeLibraryMissing(
                f"{LIB_PATH} is not built. Run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(needs nvcc). gypsum_b200 has no CPU fallback."
            )
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        if lib.gb200_abi_version() != 2:
            raise ImportError("libgypsum_b200.so ABI version mismatch; rebuild")
        _lib = lib
    return _lib


def _ptr(a: np.ndarray) -> int:
    return a.ctypes.data


def _records_out(out: np.ndarray | None, shape: tuple) -> np.ndarray:
    """A grid's record buffer: out, which must be a C-contiguous RECORD_DTYPE array of that shape, or a new one."""
    if out is None:
        return np.empty(shape, dtype=RECORD_DTYPE)
    if out.dtype != RECORD_DTYPE or out.shape != shape or not out.flags["C_CONTIGUOUS"]:
        raise ValueError("out must be a C-contiguous RECORD_DTYPE array of shape [n_blocks, n_prn, n_doppler]")
    return out


class Engine:
    """One engine per (device, sample rate).  Thin, exception-raising wrapper over the C ABI."""

    def __init__(self, samples_per_second: int, samples_per_ms: int, device: int = 0):
        self._lib = load()
        self._h = _P()
        self._host_call_cache = None
        rc = self._lib.gb200_create(int(device), int(samples_per_second), int(samples_per_ms), C.byref(self._h))
        if rc != OK:
            msg = (self._lib.gb200_last_error(None) or b"").decode()
            raise (ValueError if rc == EINVAL else RuntimeError)(f"gb200_create: {msg}")
        self.samples_per_second = int(samples_per_second)
        self.samples_per_ms = int(samples_per_ms)
        self.device = int(device)
        self.n_prn = 0
        # What the engine's single IQ binding currently holds: a caller-chosen tag (e.g. the chunk key the trackers use to
        # share one upload), cleared by EVERY call that rebinds the IQ -- so no caller can mistake another caller's samples
        # for its own.
        self.iq_tag = None
        self._children = weakref.WeakSet()  # trackers / grid streams: they hold device memory tied to this engine

    # -- plumbing ------------------------------------------------------------------------------------------
    def _check(self, rc: int, what: str) -> None:
        if rc == OK:
            return
        msg = (self._lib.gb200_last_error(self._h) or b"").decode()
        raise (ValueError if rc == EINVAL else RuntimeError)(f"{what}: {msg}")

    def close(self) -> None:
        if getattr(self, "_h", None):
            for child in list(getattr(self, "_children", ())):
                child.close()  # before the engine goes: their buffers live behind its handle's device
            self._lib.gb200_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_stream(self, cuda_stream_ptr: int) -> None:
        self._check(self._lib.gb200_set_stream(self._h, _P(cuda_stream_ptr or 0)), "gb200_set_stream")

    @property
    def launch_count(self) -> int:
        n = C.c_int64()
        self._check(self._lib.gb200_launch_count(self._h, C.byref(n)), "gb200_launch_count")
        return n.value

    def set_fused(self, mode) -> None:
        """acquire_cells kernel choice: True / 1 = fused block-per-(PRN, Doppler) kernel, False / 0 = doppler_spectra +
        correlate_cells, None / -1 = automatic (default)."""
        m = -1 if mode is None else int(mode)
        self._check(self._lib.gb200_set_fused(self._h, m), "gb200_set_fused")

    def enable_kernel_timing(self, on: bool) -> None:
        self._check(self._lib.gb200_enable_kernel_timing(self._h, int(bool(on))), "gb200_enable_kernel_timing")

    def kernel_timing(self, which: int) -> tuple[float, int]:
        """(total device ms, launches) of doppler_spectra (0) / correlate_cells (1) since timing was enabled."""
        ms, n = C.c_double(), C.c_int64()
        self._check(self._lib.gb200_kernel_timing(self._h, which, C.byref(ms), C.byref(n)), "gb200_kernel_timing")
        return ms.value, n.value

    # -- inputs --------------------------------------------------------------------------------------------
    def set_replicas(self, chips: np.ndarray) -> None:
        chips = np.ascontiguousarray(chips, dtype=np.uint8)
        if chips.ndim != 2 or chips.shape[1] != 1023:
            raise ValueError("chips must be [n_prn, 1023]")
        self._check(self._lib.gb200_set_replicas(self._h, _ptr(chips), chips.shape[0]), "gb200_set_replicas")
        self.n_prn = chips.shape[0]

    def upload_iq(self, samples: np.ndarray, tag=None) -> None:
        """tag: optional hashable naming these samples; `iq_tag` holds it until the next call that rebinds the IQ."""
        x = np.ascontiguousarray(samples, dtype=np.complex64)
        self._iq_keepalive = x
        self.iq_tag = None
        self._check(self._lib.gb200_upload_iq(self._h, _ptr(x), x.size), "gb200_upload_iq")
        self.iq_tag = tag

    def upload_iq_ptr(self, host_ptr: int, n_samples: int) -> None:
        self.iq_tag = None
        self._check(self._lib.gb200_upload_iq(self._h, _P(host_ptr), n_samples), "gb200_upload_iq")

    def bind_iq_device(self, device_ptr: int, n_samples: int, tag=None) -> None:
        self.iq_tag = None
        self._check(self._lib.gb200_bind_iq_device(self._h, _P(device_ptr), n_samples), "gb200_bind_iq_device")
        self.iq_tag = tag

    # -- the hot path --------------------------------------------------------------------------------------
    def _grid(self, name: str, n_blocks: int, ms_per_block: int, prn_idx, doppler_hz, out, segments: tuple = (),
              kind: int | None = None):
        """Every grid method but acquire_grid_host: gb200_<name> over int32 PRN rows and float64 Dopplers with the family's
        arguments (kind, or segments: (coherent_ms,) or (coherent_ms, bit_phases)).  out: a _device call's device address
        (returns None), else the records, RECORD_DTYPE [n_blocks, n_prn, (bit_phases,) n_doppler] or (0,) for a grid with no
        cells, made when None; best records (BEST_DTYPE [n_blocks, n_prn]) are always made.  Returns them."""
        prn = np.ascontiguousarray(prn_idx, dtype=np.int32)
        dop = np.ascontiguousarray(doppler_hz, dtype=np.float64)
        ret = None
        if name.endswith("_best"):
            ret = np.empty((max(n_blocks, 0), prn.size), dtype=BEST_DTYPE)
        elif not name.endswith("_device"):
            shape = (n_blocks, prn.size, *segments[1:], dop.size)  # a weak grid's bit phases fold into the bins
            ret = _records_out(out, shape if min(shape) > 0 else (0,))
        tail = () if kind is None else (kind,)
        rc = getattr(self._lib, "gb200_" + name)(self._h, n_blocks, ms_per_block, *segments, _ptr(prn), prn.size, _ptr(dop),
                                                 dop.size, *tail, _P(out) if ret is None else _ptr(ret))
        self._check(rc, "gb200_" + name)
        return ret

    def acquire_grid(self, n_blocks: int, ms_per_block: int, prn_idx, doppler_hz, kind: int = NON_COHERENT,
                     out: np.ndarray | None = None) -> np.ndarray:
        """out: optional preallocated RECORD_DTYPE array [n_blocks, n_prn, n_doppler]; if it lives in pinned memory
        (e.g. a view of a torch pinned tensor) the records are DMA'd straight into it."""
        return self._grid("acquire_grid", n_blocks, ms_per_block, prn_idx, doppler_hz, out, kind=kind)

    def acquire_grid_host(self, iq, n_blocks: int, ms_per_block: int, prn_idx, doppler_hz, kind: int = NON_COHERENT,
                          out: np.ndarray | None = None) -> np.ndarray:
        """upload + grid + records back in ONE call, replayed as a CUDA graph per shape (latency-bound callers).
        iq: complex64 array of n_blocks * ms_per_block * N samples, or an int host address of such a buffer."""
        # latency path: numpy's .ctypes costs ~1 us per array, so the addresses of the axes and of the record buffer are kept
        # for as long as the caller passes the very same array objects (their data cannot move while we hold them)
        c = self._host_call_cache
        if c is not None and c[0] is prn_idx and c[1] is doppler_hz and c[2] is out:
            prn, dop, p_prn, p_dop, p_out = c[3:]
            _records_out(out, (n_blocks, prn.size, dop.size))
        else:
            prn = np.ascontiguousarray(prn_idx, dtype=np.int32)
            dop = np.ascontiguousarray(doppler_hz, dtype=np.float64)
            cacheable = out is not None and prn is prn_idx and dop is doppler_hz  # no converted copies that could go stale
            out = _records_out(out, (n_blocks, prn.size, dop.size))
            p_prn, p_dop, p_out = _ptr(prn), _ptr(dop), _ptr(out)
            self._host_call_cache = (prn_idx, doppler_hz, out, prn, dop, p_prn, p_dop, p_out) if cacheable else None
        if isinstance(iq, int):
            keep, ptr = None, iq
        elif isinstance(iq, np.integer):
            keep, ptr = None, int(iq)
        else:
            keep = np.ascontiguousarray(iq, dtype=np.complex64)
            if keep.size < n_blocks * ms_per_block * self.samples_per_ms:
                raise ValueError("not enough samples for the grid")
            ptr = _ptr(keep)
        self.iq_tag = None
        rc = self._lib.gb200_acquire_grid_host(self._h, ptr, n_blocks, ms_per_block, p_prn, prn.size, p_dop, dop.size, kind, p_out)
        if rc:
            self._check(rc, "gb200_acquire_grid_host")
        return out

    def acquire_grid_best(self, n_blocks: int, ms_per_block: int, prn_idx, doppler_hz, kind: int = NON_COHERENT) -> np.ndarray:
        """acquisition.py:179-189 per (block, prn) row: BEST_DTYPE [n_blocks, n_prn]."""
        return self._grid("acquire_grid_best", n_blocks, ms_per_block, prn_idx, doppler_hz, None, kind=kind)

    def acquire_grid_best_device(self, n_blocks, ms_per_block, prn: np.ndarray, dop: np.ndarray, kind: int, out_device_ptr: int):
        self._grid("acquire_grid_best_device", n_blocks, ms_per_block, prn, dop, out_device_ptr, kind=kind)

    def acquire_grid_device(self, n_blocks, ms_per_block, prn: np.ndarray, dop: np.ndarray, kind: int, out_device_ptr: int):
        """Enqueue only: the records reach out_device_ptr in the engine's stream order."""
        self._grid("acquire_grid_device", n_blocks, ms_per_block, prn, dop, out_device_ptr, kind=kind)

    def acquire_grid_semicoherent(self, n_blocks: int, ms_per_block: int, coherent_ms: int, prn_idx, doppler_hz,
                                  out: np.ndarray | None = None) -> np.ndarray:
        """Semi-coherent grid (gb200_acquire_grid_semicoherent): per cell the profile sum_k |coherent sum of milliseconds
        k*coherent_ms .. (k+1)*coherent_ms - 1|, reduced to RECORD_DTYPE [n_blocks, n_prn, n_doppler]."""
        return self._grid("acquire_grid_semicoherent", n_blocks, ms_per_block, prn_idx, doppler_hz, out, (coherent_ms,))

    def acquire_grid_semicoherent_device(self, n_blocks, ms_per_block, coherent_ms, prn: np.ndarray, dop: np.ndarray,
                                         out_device_ptr: int):
        """Enqueue only: the records reach out_device_ptr in the engine's stream order."""
        self._grid("acquire_grid_semicoherent_device", n_blocks, ms_per_block, prn, dop, out_device_ptr, (coherent_ms,))

    def acquire_grid_semicoherent_best(self, n_blocks: int, ms_per_block: int, coherent_ms: int, prn_idx,
                                       doppler_hz) -> np.ndarray:
        """The semi-coherent grid's best bin per (block, prn) row: BEST_DTYPE [n_blocks, n_prn]."""
        return self._grid("acquire_grid_semicoherent_best", n_blocks, ms_per_block, prn_idx, doppler_hz, None, (coherent_ms,))

    def acquire_grid_semicoherent_best_device(self, n_blocks, ms_per_block, coherent_ms, prn: np.ndarray, dop: np.ndarray,
                                              out_device_ptr: int):
        self._grid("acquire_grid_semicoherent_best_device", n_blocks, ms_per_block, prn, dop, out_device_ptr, (coherent_ms,))

    def acquire_grid_weak(self, n_blocks: int, ms_per_block: int, coherent_ms: int, bit_phases: int, prn_idx, doppler_hz,
                          out: np.ndarray | None = None) -> np.ndarray:
        """Weak grid (gb200_acquire_grid_weak): per cell and bit phase j the semi-coherent profile of the segments starting
        at millisecond j * coherent_ms / bit_phases, every millisecond realigned by its code Doppler, reduced to
        RECORD_DTYPE [n_blocks, n_prn, bit_phases, n_doppler]."""
        return self._grid("acquire_grid_weak", n_blocks, ms_per_block, prn_idx, doppler_hz, out, (coherent_ms, bit_phases))

    def acquire_grid_weak_device(self, n_blocks, ms_per_block, coherent_ms, bit_phases, prn: np.ndarray, dop: np.ndarray,
                                 out_device_ptr: int):
        """Enqueue only: the records reach out_device_ptr in the engine's stream order."""
        self._grid("acquire_grid_weak_device", n_blocks, ms_per_block, prn, dop, out_device_ptr, (coherent_ms, bit_phases))

    def acquire_grid_weak_best(self, n_blocks: int, ms_per_block: int, coherent_ms: int, bit_phases: int, prn_idx,
                               doppler_hz) -> np.ndarray:
        """The weak grid's best folded bin per (block, prn) row: BEST_DTYPE [n_blocks, n_prn], bin = j * n_doppler + d."""
        return self._grid("acquire_grid_weak_best", n_blocks, ms_per_block, prn_idx, doppler_hz, None, (coherent_ms, bit_phases))

    def acquire_grid_weak_best_device(self, n_blocks, ms_per_block, coherent_ms, bit_phases, prn: np.ndarray, dop: np.ndarray,
                                      out_device_ptr: int):
        self._grid("acquire_grid_weak_best_device", n_blocks, ms_per_block, prn, dop, out_device_ptr,
                   (coherent_ms, bit_phases))

    def acquire_cells(self, prn_idx, doppler_hz, n_ms: int, kind: int = NON_COHERENT, probe_idx=None) -> np.ndarray:
        prn = np.ascontiguousarray(prn_idx, dtype=np.int32)
        dop = np.ascontiguousarray(doppler_hz, dtype=np.float64)
        if prn.shape != dop.shape or prn.ndim != 1:
            raise ValueError("prn_idx and doppler_hz must be 1-D and the same length")
        probe = None if probe_idx is None else np.ascontiguousarray(probe_idx, dtype=np.int32)
        out = np.empty(prn.size, dtype=RECORD_DTYPE)
        self._check(
            self._lib.gb200_acquire_cells(self._h, prn.size, _ptr(prn), _ptr(dop), None if probe is None else _ptr(probe),
                                          n_ms, kind, _ptr(out)),
            "gb200_acquire_cells",
        )
        return out

    def detect(self, prn_idx, n_ms: int) -> np.ndarray:
        """acquisition.py:70-152 for every listed replica row, all ten passes + the coherent pass on the device."""
        prn = np.ascontiguousarray(prn_idx, dtype=np.int32)
        out = np.empty(prn.size, dtype=ACQ_DTYPE)
        self._check(self._lib.gb200_detect(self._h, prn.size, _ptr(prn), int(n_ms), _ptr(out)), "gb200_detect")
        return out

    def correlation_profile(self, prn_idx: int, doppler_hz: float, n_ms: int, kind: int) -> np.ndarray:
        n = self.samples_per_ms
        out = np.empty(n * (2 if kind == COHERENT else 1), dtype=np.float32)
        self._check(
            self._lib.gb200_correlation_profile(self._h, int(prn_idx), float(doppler_hz), int(n_ms), int(kind), _ptr(out)),
            "gb200_correlation_profile",
        )
        return out.view(np.complex64) if kind == COHERENT else out

    def correlation_profile_replica(self, replica: np.ndarray, doppler_hz: float, n_ms: int, kind: int) -> np.ndarray:
        """utils.py:77-108 against an ARBITRARY complex replica of samples_per_ms samples (direct evaluation)."""
        n = self.samples_per_ms
        rep = np.ascontiguousarray(replica, dtype=np.complex64)
        if rep.shape != (n,):
            raise ValueError(f"replica must have {n} samples")
        out = np.empty(n * (2 if kind == COHERENT else 1), dtype=np.float32)
        self._check(
            self._lib.gb200_correlation_profile_replica(self._h, _ptr(rep), float(doppler_hz), int(n_ms), int(kind), _ptr(out)),
            "gb200_correlation_profile_replica",
        )
        return out.view(np.complex64) if kind == COHERENT else out


class GridStream:
    """Pipelined stream of equally shaped grid batches (gb200_grid_stream_*): `submit` enqueues copy-in, the grid and
    copy-out of one batch, `collect` waits for the oldest batch in flight and returns its record array.  With depth >= 2
    the transfers of neighbouring batches run under the kernels of the current one."""

    def __init__(self, engine: Engine, n_blocks: int, ms_per_block: int, prn_idx, doppler_hz, kind: int = NON_COHERENT,
                 depth: int = 2):
        self._engine = engine
        self._lib = engine._lib
        prn = np.ascontiguousarray(prn_idx, dtype=np.int32)
        dop = np.ascontiguousarray(doppler_hz, dtype=np.float64)
        self.shape = (n_blocks, prn.size, dop.size)
        self.samples_per_batch = n_blocks * ms_per_block * engine.samples_per_ms
        self.depth = depth
        self._pending: list = []  # (iq keep-alive, out array) per batch in flight
        self._h = _P()
        engine._check(self._lib.gb200_grid_stream_create(engine._h, n_blocks, ms_per_block, _ptr(prn), prn.size, _ptr(dop),
                                                         dop.size, kind, depth, C.byref(self._h)), "gb200_grid_stream_create")
        engine._children.add(self)

    @property
    def in_flight(self) -> int:
        return len(self._pending)

    def submit(self, iq, out: np.ndarray | None = None) -> None:
        """iq: complex64 array of samples_per_batch samples, or an int host address of such a buffer.  out: optional
        RECORD_DTYPE array [n_blocks, n_prn, n_doppler] (pinned memory = direct DMA)."""
        if isinstance(iq, (int, np.integer)):
            keep, ptr = None, _P(int(iq))
        else:
            keep = np.ascontiguousarray(iq, dtype=np.complex64)
            if keep.size != self.samples_per_batch:
                raise ValueError(f"a batch is {self.samples_per_batch} samples, got {keep.size}")
            ptr = _ptr(keep)
        out = _records_out(out, self.shape)
        self._engine.iq_tag = None  # the stream rebinds the engine's IQ to its own slot buffer
        self._engine._check(self._lib.gb200_grid_stream_submit(self._h, ptr, _ptr(out)), "gb200_grid_stream_submit")
        self._pending.append((keep, out))

    def collect(self) -> np.ndarray:
        self._engine._check(self._lib.gb200_grid_stream_collect(self._h), "gb200_grid_stream_collect")
        return self._pending.pop(0)[1]

    def close(self) -> None:
        if getattr(self, "_h", None) and getattr(self._engine, "_h", None):
            self._lib.gb200_grid_stream_destroy(self._h)
        self._h = None
        self._pending = []

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Ring:
    """Device-resident rolling window of the newest milliseconds (gb200_ring_*; receiver.py:68,100,219)."""

    def __init__(self, engine: Engine, capacity_ms: int):
        self._engine = engine
        self._lib = engine._lib
        self.capacity_ms = int(capacity_ms)
        self._h = _P()
        engine._check(self._lib.gb200_ring_create(engine._h, self.capacity_ms, C.byref(self._h)), "gb200_ring_create")
        engine._children.add(self)

    def append(self, samples) -> None:
        """samples: complex64[n_ms * N] (whole milliseconds)."""
        x = np.ascontiguousarray(samples, dtype=np.complex64)
        n = self._engine.samples_per_ms
        if x.size == 0 or x.size % n:
            raise ValueError("append whole milliseconds")
        self._engine._check(self._lib.gb200_ring_append(self._h, _ptr(x), x.size // n), "gb200_ring_append")
        if isinstance(self._engine.iq_tag, tuple) and self._engine.iq_tag[:1] == ("ring",):
            self._engine.iq_tag = None  # a binding into this ring no longer names the newest samples

    @property
    def appended_ms(self) -> int:
        n = C.c_int64()
        self._engine._check(self._lib.gb200_ring_appended(self._h, C.byref(n)), "gb200_ring_appended")
        return n.value

    def bind_newest(self, n_ms: int) -> None:
        """The engine's IQ := the newest n_ms milliseconds, in place."""
        tag = ("ring", id(self), self.appended_ms, int(n_ms))
        if self._engine.iq_tag == tag:
            return
        self._engine.iq_tag = None
        self._engine._check(self._lib.gb200_ring_bind_newest(self._h, int(n_ms)), "gb200_ring_bind_newest")
        self._engine.iq_tag = tag

    def close(self) -> None:
        if getattr(self, "_h", None) and getattr(self._engine, "_h", None):
            self._lib.gb200_ring_destroy(self._h)
            self._engine.iq_tag = None
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Tracker:
    """A bank of tracking channels on one engine (gb200_tracker_*).  Channels consume the engine's loaded IQ."""

    @classmethod
    def pool(cls, engine: Engine, capacity: int) -> "Tracker":
        """`capacity` idle channel slots (gb200_tracker_create_pool); seed them with reset_channel."""
        self = cls.__new__(cls)
        self._engine = engine
        self._lib = engine._lib
        self.n_channels = int(capacity)
        self._h = _P()
        engine._check(self._lib.gb200_tracker_create_pool(engine._h, int(capacity), C.byref(self._h)), "gb200_tracker_create_pool")
        engine._children.add(self)
        return self

    def reset_channel(self, channel: int, prn_idx: int, doppler: float, carrier_phase: float, code_phase: int) -> None:
        self._engine._check(self._lib.gb200_tracker_reset_channel(self._h, int(channel), int(prn_idx), float(doppler),
                                                                  float(carrier_phase), int(code_phase)),
                            "gb200_tracker_reset_channel")

    def process_channels(self, channels, n_ms: int, start_times, want_profiles: bool = False, keep_undo: bool = False):
        """gb200_tracker_process for a subset, one launch: records [len(channels), n_ms] (and profiles)."""
        sel = np.ascontiguousarray(channels, dtype=np.int32)
        ts = np.ascontiguousarray(start_times, dtype=np.float64)
        if ts.shape != (n_ms,):
            raise ValueError("start_times must hold one timestamp per millisecond")
        out = np.empty((sel.size, n_ms), dtype=TRACK_DTYPE)
        prof = np.empty((sel.size, n_ms, self._engine.samples_per_ms), dtype=np.float32) if want_profiles else None
        self._engine._check(
            self._lib.gb200_tracker_process_channels(self._h, sel.size, _ptr(sel), n_ms, _ptr(ts), int(bool(keep_undo)),
                                                     _ptr(out), None if prof is None else _ptr(prof)),
            "gb200_tracker_process_channels")
        return (out, prof) if want_profiles else out

    def undo_channel(self, channel: int) -> None:
        self._engine._check(self._lib.gb200_tracker_undo_channel(self._h, int(channel)), "gb200_tracker_undo_channel")

    def __init__(self, engine: Engine, prn_idx, doppler_hz, carrier_phase, code_phase):
        self._engine = engine
        self._lib = engine._lib
        prn = np.ascontiguousarray(prn_idx, dtype=np.int32)
        dop = np.ascontiguousarray(doppler_hz, dtype=np.float64)
        cph = np.ascontiguousarray(carrier_phase, dtype=np.float64)
        code = np.ascontiguousarray(code_phase, dtype=np.int32)
        if not (prn.shape == dop.shape == cph.shape == code.shape) or prn.ndim != 1:
            raise ValueError("per-channel arrays must be 1-D and the same length")
        self.n_channels = prn.size
        self._h = _P()
        engine._check(self._lib.gb200_tracker_create(engine._h, prn.size, _ptr(prn), _ptr(dop), _ptr(cph), _ptr(code),
                                                     C.byref(self._h)), "gb200_tracker_create")
        engine._children.add(self)

    def close(self) -> None:
        if getattr(self, "_h", None) and getattr(self._engine, "_h", None):
            self._lib.gb200_tracker_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def process(self, n_ms: int, start_times, want_profiles: bool = False):
        """Records [n_channels, n_ms] (TRACK_DTYPE) and, optionally, |prompt profile| [n_channels, n_ms, N]."""
        ts = np.ascontiguousarray(start_times, dtype=np.float64)
        if ts.shape != (n_ms,):
            raise ValueError("start_times must hold one timestamp per millisecond")
        out = np.empty((self.n_channels, n_ms), dtype=TRACK_DTYPE)
        prof = np.empty((self.n_channels, n_ms, self._engine.samples_per_ms), dtype=np.float32) if want_profiles else None
        self._engine._check(
            self._lib.gb200_tracker_process(self._h, n_ms, _ptr(ts), _ptr(out), None if prof is None else _ptr(prof)),
            "gb200_tracker_process")
        return (out, prof) if want_profiles else out

    def process_device(self, n_ms: int, start_times: np.ndarray, out_device_ptr: int) -> None:
        self._engine._check(self._lib.gb200_tracker_process_device(self._h, n_ms, _ptr(start_times), _P(out_device_ptr)),
                            "gb200_tracker_process_device")

    def integrate_bits(self, n_ms: int, start_times, end_times, records_device_ptr: int | None = None) -> list:
        """navigation_bit_intergrator.py:278-288 for every channel over records in device memory (default: the ones the
        last `process` call left there).  Returns one BIT_DTYPE array per channel."""
        t0 = np.ascontiguousarray(start_times, dtype=np.float64)
        t1 = np.ascontiguousarray(end_times, dtype=np.float64)
        if t0.shape != (n_ms,) or t1.shape != (n_ms,):
            raise ValueError("start_times / end_times must hold one timestamp per millisecond")
        cap = n_ms // 20 + 8  # whole bits in the call + the backlog a first phase decision releases (<= 81 symbols)
        records = None if records_device_ptr is None else _P(records_device_ptr)
        return self._per_channel("gb200_tracker_integrate_bits", BIT_DTYPE, cap, "bit event",  # cannot truncate: see `cap`
                                 n_ms, _ptr(t0), _ptr(t1), records)

    def _per_channel(self, name: str, dtype, cap: int, what: str, *args) -> list:
        """Calls the C function `name` with (handle, *args, out, cap, counts), out being [n_channels, cap] of dtype, and
        returns the events of each channel."""
        out = np.empty((self.n_channels, cap), dtype=dtype)
        cnt = np.empty(self.n_channels, dtype=np.int32)
        self._engine._check(getattr(self._lib, name)(self._h, *args, _ptr(out), cap, _ptr(cnt)), name)
        if (cnt > cap).any():
            raise RuntimeError(f"{what} buffer too small")
        return [out[c, : cnt[c]].copy() for c in range(self.n_channels)]

    def _chain_sizes(self) -> list[int]:
        """Bit events per channel the last integrate_bits call kept, subframe events per channel the last
        decode_subframes call kept, and the milliseconds of the last parse_subframes call (gb200_tracker_chain_sizes)."""
        out = np.zeros(3, dtype=np.int32)
        self._engine._check(self._lib.gb200_tracker_chain_sizes(self._h, _ptr(out)), "gb200_tracker_chain_sizes")
        return [int(v) for v in out]

    def bit_state(self, channel: int) -> dict:
        out = np.zeros(8, dtype=np.int64)
        self._engine._check(self._lib.gb200_tracker_bit_state(self._h, channel, _ptr(out)), "gb200_tracker_bit_state")
        keys = ("emitted_bit_count", "failed_bit_count", "processed_pseudosymbol_count", "slide", "determined_bit_phase",
                "previous_bit_phase_decision", "pseudosymbol_cursor_within_queue", "stopped")
        d = dict(zip(keys, (int(v) for v in out)))
        for k in ("determined_bit_phase", "previous_bit_phase_decision"):
            d[k] = None if d[k] < 0 else d[k]
        return d

    def decode_subframes(self, bits_device_ptr: int | None = None, counts=None, stride: int | None = None) -> list:
        """navigation_message_decoder.py:173-196 for every channel over bit events in device memory: by default the
        ones the last `integrate_bits` call left there; else a device array [n_channels][stride] of BIT_DTYPE with
        counts[c] events in row c.  Returns one SUBFRAME_DTYPE array per channel (kinds: 0 subframe, 1 determined
        phase, 2 cannot determine phase, 3 the reference raises; see include/gypsum_b200.h)."""
        if bits_device_ptr is None:
            if counts is not None or stride is not None:
                raise ValueError("counts / stride describe a caller's device array only")
            n_bits = self._chain_sizes()[0]
            args = (None, None, 0)
        else:
            cnt_in = np.ascontiguousarray(counts, dtype=np.int32)
            if cnt_in.shape != (self.n_channels,) or stride is None:
                raise ValueError("a device bit array needs one count per channel and its stride")
            n_bits = int(cnt_in.max(initial=0))
            args = (_P(bits_device_ptr), _ptr(cnt_in), int(stride))
        return self._per_channel("gb200_tracker_decode_subframes", SUBFRAME_DTYPE, subframe_event_capacity(n_bits),
                                 "subframe event", *args)  # cannot truncate: see subframe_event_capacity

    def parse_subframes(self, events_device_ptr: int | None = None, counts=None, stride: int | None = None,
                        event_ms=None, drop_ms=None, n_ms: int | None = None) -> list:
        """Subframe fields and the world model's per-satellite state (gb200_tracker_parse_subframes).  By default over
        the events the last `decode_subframes` call left on the device (the process -> integrate_bits ->
        decode_subframes chain); else over a device array [n_channels][stride] of SUBFRAME_DTYPE with counts[c] events
        in row c, their milliseconds event_ms [n_channels, stride], drop_ms [n_channels] (-1 = none) and n_ms.
        Returns one FIELDS_DTYPE array per channel."""
        if events_device_ptr is None:
            if any(v is not None for v in (counts, stride, event_ms, drop_ms, n_ms)):
                raise ValueError("counts / stride / event_ms / drop_ms / n_ms describe a caller's device array only")
            cap = self._chain_sizes()[1]
            args = (None, None, 0, None, None, 0)
        else:
            cnt_in = np.ascontiguousarray(counts, dtype=np.int32)
            ems = np.ascontiguousarray(event_ms, dtype=np.int32)
            drop = np.ascontiguousarray(drop_ms, dtype=np.int32)
            if cnt_in.shape != (self.n_channels,) or drop.shape != (self.n_channels,) or stride is None or n_ms is None:
                raise ValueError("a device event array needs one count and one drop per channel, its stride and n_ms")
            if ems.shape != (self.n_channels, int(stride)):
                raise ValueError("event_ms must be [n_channels, stride]")
            cap = int(cnt_in.max(initial=0))
            args = (_P(events_device_ptr), _ptr(cnt_in), int(stride), _ptr(ems), _ptr(drop), int(n_ms))
        # a channel's fields are at most its events
        return self._per_channel("gb200_tracker_parse_subframes", FIELDS_DTYPE, max(1, cap), "field", *args)

    def orbit_state(self, channel: int) -> dict:
        """One channel's world-model entry: params (float64[26], OrbitalParameterType order), set_mask, prn_count,
        counting."""
        p = np.zeros(ORBIT_PARAMS, dtype=np.float64)
        mask, count, counting = C.c_uint32(), C.c_int64(), C.c_int32()
        self._engine._check(self._lib.gb200_tracker_orbit_state(self._h, channel, _ptr(p), C.byref(mask), C.byref(count),
                                                                C.byref(counting)), "gb200_tracker_orbit_state")
        return {"params": p, "set_mask": mask.value, "prn_count": count.value, "counting": bool(counting.value)}

    def observations(self) -> np.ndarray:
        """OBSERVATION_DTYPE [n_channels, n_ms] over the milliseconds of the last parse_subframes call."""
        out = np.empty((self.n_channels, self._chain_sizes()[2]), dtype=OBSERVATION_DTYPE)
        self._engine._check(self._lib.gb200_tracker_observations(self._h, _ptr(out)), "gb200_tracker_observations")
        return out

    def observations_device(self, out_device_ptr: int) -> None:
        """Enqueue only: n_channels * n_ms OBSERVATION_DTYPE records to device memory."""
        self._engine._check(self._lib.gb200_tracker_observations_device(self._h, _P(out_device_ptr)),
                            "gb200_tracker_observations_device")

    def _fix_times(self, receiver_timestamps) -> np.ndarray:
        rx = np.ascontiguousarray(receiver_timestamps, dtype=np.float64)
        n_ms = self._chain_sizes()[2]
        if rx.shape != (n_ms,):
            raise ValueError(f"receiver_timestamps must hold one start time per millisecond of the last parse_subframes "
                             f"call ({n_ms})")
        return rx

    def position_fixes(self, receiver_timestamps) -> np.ndarray:
        """FIX_DTYPE [n_ms]: the world model's position fix (world_model.py:567-633) for every millisecond of the last
        parse_subframes call, receiver_timestamps being the chunk start times.  The receiver's clock slide, world-model
        order and stop carry from call to call (gb200_tracker_position_fixes)."""
        rx = self._fix_times(receiver_timestamps)
        out = np.empty(rx.size, dtype=FIX_DTYPE)
        self._engine._check(self._lib.gb200_tracker_position_fixes(self._h, _ptr(rx), _ptr(out)),
                            "gb200_tracker_position_fixes")
        return out

    def set_fix_solver(self, solver: str) -> None:
        """Which fix a millisecond with five or more ready satellites gets (gb200_tracker_set_fix_solver): "reference"
        (the default) raises there as the reference does and stops the receiver; "least_squares" solves by least
        squares over all of them.  Only before the first fix call (RuntimeError after it); ValueError for another
        name."""
        if solver not in FIX_SOLVERS:
            raise ValueError(f"fix solver must be one of {sorted(FIX_SOLVERS)}, not {solver!r}")
        self._engine._check(self._lib.gb200_tracker_set_fix_solver(self._h, FIX_SOLVERS[solver]),
                            "gb200_tracker_set_fix_solver")

    def set_code_phase_mode(self, mode: str) -> None:
        """How the channels count code phase (gb200_tracker_set_code_phase_mode): "reference" (the default) wraps the DLL
        accumulator at 2046 and delays each pseudosymbol by code phase / 2046 ms at every rate, as the reference does;
        "samples" wraps at the engine's samples per millisecond N and delays by code phase / N ms, so that every code
        phase in [0, N) stays tracked.  Only before the first tracking or bit-integration call (RuntimeError after it);
        ValueError for another name."""
        if mode not in CODE_PHASE_MODES:
            raise ValueError(f"code-phase mode must be one of {sorted(CODE_PHASE_MODES)}, not {mode!r}")
        self._engine._check(self._lib.gb200_tracker_set_code_phase_mode(self._h, CODE_PHASE_MODES[mode]),
                            "gb200_tracker_set_code_phase_mode")

    def position_fixes_device(self, receiver_timestamps, out_device_ptr: int) -> None:
        """Enqueue only: n_ms FIX_DTYPE records to device memory."""
        rx = self._fix_times(receiver_timestamps)
        self._engine._check(self._lib.gb200_tracker_position_fixes_device(self._h, _ptr(rx), _P(out_device_ptr)),
                            "gb200_tracker_position_fixes_device")

    def velocity_fixes(self, doppler_device_ptr=None, fixes_device_ptr=None) -> np.ndarray:
        """VELOCITY_DTYPE [n_ms]: velocity, clock drift, geodetic position and DOP of every millisecond of the last
        parse_subframes call with a solved position fix (gb200_tracker_velocity_fixes).  doppler_device_ptr: a device
        float64 [n_channels, n_ms] Doppler in Hz, or None for the tracking records of the process call behind that parse
        call; fixes_device_ptr: the fix records on the device, or None for those the last position_fixes call kept."""
        out = np.empty(self._chain_sizes()[2], dtype=VELOCITY_DTYPE)
        self._engine._check(self._lib.gb200_tracker_velocity_fixes(self._h, _P(doppler_device_ptr), _P(fixes_device_ptr),
                                                                   _ptr(out)), "gb200_tracker_velocity_fixes")
        return out

    def velocity_fixes_device(self, out_device_ptr: int, doppler_device_ptr=None, fixes_device_ptr=None) -> None:
        """Enqueue only: n_ms VELOCITY_DTYPE records to device memory."""
        self._engine._check(self._lib.gb200_tracker_velocity_fixes_device(self._h, _P(doppler_device_ptr),
                                                                          _P(fixes_device_ptr), _P(out_device_ptr)),
                            "gb200_tracker_velocity_fixes_device")

    def signal_windows(self, n_ms: int, start_times, window_ms: int, records_device_ptr: int | None = None,
                       max_windows: int | None = None) -> list:
        """Carrier-to-noise density and phase-lock indicator of every channel over windows of window_ms consecutive
        milliseconds of its tracking records (gb200_tracker_signal_windows): records in device memory, by default the
        ones the last `process` call left there.  Each channel's open window carries into the next call; window_ms is
        fixed by the first call.  Returns one SIGNAL_DTYPE array per channel.  max_windows (default: the most one call
        touches) caps the windows kept per channel; RuntimeError if a channel produced more."""
        ts = np.ascontiguousarray(start_times, dtype=np.float64)
        if ts.shape != (n_ms,):
            raise ValueError("start_times must hold one timestamp per millisecond")
        # the window the last call left open, then one every window_ms: at most n_ms // window_ms + 2 (valid W only)
        cap = int(n_ms) // max(int(window_ms), 1) + 2 if max_windows is None else int(max_windows)
        records = None if records_device_ptr is None else _P(records_device_ptr)
        return self._per_channel("gb200_tracker_signal_windows", SIGNAL_DTYPE, cap, "signal window",
                                 int(n_ms), _ptr(ts), int(window_ms), records)

    def receiver_state(self) -> dict:
        """After the last fix call: slide (receiver_clock_slide, None before any), stopped, order: the channels in
        the world model's order, and repaired: the fixes the serial chain recomputed where the parallel passes' chain
        check failed (gb200_tracker_fix_repairs)."""
        slide, stopped, repaired = C.c_double(), C.c_int32(), C.c_int64()
        order = np.empty(self.n_channels, dtype=np.int32)
        self._engine._check(self._lib.gb200_tracker_receiver_state(self._h, C.byref(slide), C.byref(stopped), _ptr(order)),
                            "gb200_tracker_receiver_state")
        self._engine._check(self._lib.gb200_tracker_fix_repairs(self._h, C.byref(repaired)), "gb200_tracker_fix_repairs")
        return {"slide": None if np.isnan(slide.value) else slide.value, "stopped": bool(stopped.value),
                "order": [int(c) for c in order if c >= 0], "repaired": int(repaired.value)}

    def subframe_state(self, channel: int) -> dict:
        out = np.zeros(6, dtype=np.int64)
        self._engine._check(self._lib.gb200_tracker_subframe_state(self._h, channel, _ptr(out)), "gb200_tracker_subframe_state")
        keys = ("determined_subframe_phase", "emitted_subframe_count", "polarity", "queued_bit_count", "stopped",
                "processed_bit_count")
        d = dict(zip(keys, (int(v) for v in out)))
        if d["determined_subframe_phase"] < 0:
            d["determined_subframe_phase"] = None
        return d

    def get_state(self, channel: int) -> dict:
        d, c, a = C.c_double(), C.c_double(), C.c_double()
        p, lost = C.c_int32(), C.c_int32()
        self._engine._check(self._lib.gb200_tracker_get_state(self._h, channel, C.byref(d), C.byref(c), C.byref(a), C.byref(p),
                                                              C.byref(lost)), "gb200_tracker_get_state")
        return {"doppler": d.value, "carrier_phase": c.value, "phase_acc": a.value, "code_phase": p.value, "lost": lost.value}

    def set_state(self, channel: int, doppler: float, carrier_phase: float, phase_acc: float, code_phase: int) -> None:
        self._engine._check(self._lib.gb200_tracker_set_state(self._h, channel, float(doppler), float(carrier_phase),
                                                              float(phase_acc), int(code_phase)), "gb200_tracker_set_state")


BIT_DTYPE = np.dtype([  # gb200_bit_event
    ("receiver_timestamp", "<f8"), ("trailing_edge_receiver_timestamp", "<f8"), ("ms_index", "<i4"), ("bit_value", "<i4"),
    ("slide", "<i4"), ("pad_", "<i4")])
assert BIT_DTYPE.itemsize == 32

SUBFRAME_DTYPE = np.dtype([  # gb200_subframe_event
    ("receiver_timestamp", "<f8"), ("trailing_edge_receiver_timestamp", "<f8"), ("words", "<u4", (10,)), ("kind", "<i4"),
    ("bit_index", "<i4"), ("subframe_id", "<i4"), ("tow", "<i4"), ("phase", "<i4"), ("polarity", "<i4"),
    ("parity_ok", "<i4"), ("pad_", "<i4", (3,))])
assert SUBFRAME_DTYPE.itemsize == 96
SUBFRAME, DETERMINED_PHASE, CANNOT_DETERMINE_PHASE, RAISED = 0, 1, 2, 3  # SUBFRAME_DTYPE["kind"]
STOP_RAISED, STOP_OVERFLOW, STOP_LOST_LOCK = 1, 2, 3  # Tracker.subframe_state()["stopped"]

FIELDS_DTYPE = np.dtype([  # gb200_subframe_fields
    ("event_index", "<i4"), ("ms", "<i4"), ("subframe_id", "<i4"), ("reserved", "<i4"), ("tow_seconds", "<f8"),
    ("ints", "<i4", (2,)), ("bits", "<u4", (4,)), ("bit_widths", "<i4", (4,)), ("values", "<f8", (10,))])
assert FIELDS_DTYPE.itemsize == 144
OBSERVATION_DTYPE = np.dtype([  # gb200_sv_observation
    ("tow", "<f8"), ("dsv", "<f8"), ("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("prn_count", "<i8"), ("flags", "<i4"),
    ("reserved", "<i4")])
assert OBSERVATION_DTYPE.itemsize == 56
ORBIT_PARAMS = 26
OBS_TIMING, OBS_COMPLETE, OBS_FIX_GATE, OBS_COUNTING, OBS_FROZEN = 1, 2, 4, 8, 16  # OBSERVATION_DTYPE["flags"]
FIX_DTYPE = np.dtype([  # gb200_position_fix
    ("receiver_timestamp", "<f8"), ("slide_in", "<f8"), ("slide_out", "<f8"), ("clock_bias", "<f8"), ("x", "<f8"),
    ("y", "<f8"), ("z", "<f8"), ("pseudorange", "<f8", (4,)), ("status", "<i4"), ("n_ready", "<i4"),
    ("channel", "<i4", (4,))])
assert FIX_DTYPE.itemsize == 112
FIX_NONE, FIX_SOLVED, FIX_RAISED, FIX_STOPPED = 0, 1, 2, 3  # FIX_DTYPE["status"]
FIX_SOLVERS = {"reference": 0, "least_squares": 1}  # GB200_FIX_SOLVER_*
CODE_PHASE_MODES = {"reference": 0, "samples": 1}  # GB200_CODE_PHASE_*
REFERENCE_CODE_WRAP = 2046  # where the reference's DLL accumulator wraps at every rate (tracker.py:301-303, :319)
VELOCITY_DTYPE = np.dtype([  # gb200_velocity_fix
    ("receiver_timestamp", "<f8"), ("vx", "<f8"), ("vy", "<f8"), ("vz", "<f8"), ("clock_drift", "<f8"),
    ("latitude_deg", "<f8"), ("longitude_deg", "<f8"), ("height", "<f8"), ("gdop", "<f8"), ("pdop", "<f8"),
    ("hdop", "<f8"), ("vdop", "<f8"), ("tdop", "<f8"), ("residual_rms", "<f8"), ("status", "<i4"), ("n_rows", "<i4"),
    ("reserved", "<i4", (2,))])
assert VELOCITY_DTYPE.itemsize == 128
VEL_NONE, VEL_SOLVED, VEL_UNSOLVABLE = 0, 1, 2  # VELOCITY_DTYPE["status"]
SIGNAL_DTYPE = np.dtype([  # gb200_signal_window
    ("receiver_timestamp", "<f8"), ("cn0_dbhz", "<f8"), ("prompt_power", "<f8"), ("noise_power", "<f8"),
    ("pll_lock", "<f8"), ("first_ms", "<i8"), ("ms_index", "<i4"), ("n_ms", "<i4"), ("locked_ms", "<i4"),
    ("status", "<i4")])
assert SIGNAL_DTYPE.itemsize == 64
SIGNAL_NONE, SIGNAL_FOUND, SIGNAL_NOISE = 0, 1, 2  # SIGNAL_DTYPE["status"]


def subframe_event_capacity(n_bits: int) -> int:
    """Most events one channel's decoder can produce from n_bits bit events: one phase event per bit at most, where a
    run of CannotDetermine events spans at most 497 bits (3600..4096 queued) and runs are >= 3300 bits apart, a
    determined phase needs >= 300 new bits, and the subframes drained come from the queue (<= 4096 bits) plus the new
    bits."""
    n = int(n_bits)
    return min(n, 497 * (1 + n // 3300)) + (1 + n // 300) + (4096 + n) // 300 + 1


def subframe_bits(event) -> list[int]:
    """The 300 upright bits of a SUBFRAME_DTYPE event, IS-GPS-200 bit 1 of word 1 first: the list the reference's
    NavigationMessageSubframeParser takes."""
    return [int(w >> (29 - i)) & 1 for w in event["words"] for i in range(30)]


def strength_from_records(rec: np.ndarray, n: int) -> np.ndarray:
    """utils.py:111-116 on the reduced record: peak / mean(profile[profile != peak])."""
    peak = rec["peak"].astype(np.float64)
    cnt = rec["count"].astype(np.float64)
    return peak / ((rec["sum"] - cnt * peak) / (n - cnt))
