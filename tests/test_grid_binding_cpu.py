"""How the Engine's twelve grid methods -- acquire_grid, acquire_grid_semicoherent and acquire_grid_weak, each with its
_device, _best and _best_device variant -- call the library, checked without a GPU against a stand-in library that
records every call: the symbol, the arguments after the engine handle (pointers as integers), the PRN and Doppler axes as
the library reads them during the call, and the output buffer it is handed."""
import ctypes as C
from unittest.mock import ANY

import numpy as np
import pytest

from gypsum_b200 import _native

NB, M = 2, 8
PRN = np.array([3, 0, 7], np.int32)
DOP = np.array([-500.0, 0.0, 250.0, 1000.0])
DEV = 0x7F0000001000  # a device address: handed over, never dereferenced here
EXTRA = {"plain": (_native.COHERENT,), "semicoherent": (4,), "weak": (4, 2)}  # kind / coherent_ms / coherent_ms, bit_phases
PHASES = {"plain": 1, "semicoherent": 1, "weak": 2}
VARIANTS = ["", "_device", "_best", "_best_device"]
METHODS = [(f, v) for f in EXTRA for v in VARIANTS]


class _Lib:
    """Stands in for the library: records each grid call and returns rc, with last_error as the message."""

    def __init__(self, rc=_native.OK, last_error=b""):
        self.calls, self.rc, self.last_error = [], rc, last_error

    def gb200_last_error(self, h):
        return self.last_error

    def __getattr__(self, name):
        if not name.startswith("gb200_acquire_grid"):
            raise AttributeError(name)
        skip = 2 if "weak" in name else 1 if "semicoherent" in name else 0  # arguments between ms_per_block and prn_idx

        def call(h, *args):
            args = tuple(a.value if isinstance(a, C.c_void_p) else a for a in args)
            p_prn, n_prn, p_dop, n_dop = args[2 + skip:6 + skip]
            prn = np.frombuffer((C.c_int32 * n_prn).from_address(p_prn), np.int32).copy() if n_prn > 0 else None
            dop = np.frombuffer((C.c_double * n_dop).from_address(p_dop), np.float64).copy() if n_dop > 0 else None
            self.calls.append((name, args, prn, dop))
            return self.rc

        return call


def _engine(lib=None):
    eng = object.__new__(_native.Engine)
    eng._lib, eng._h = lib or _Lib(), None
    return eng


def _name(family, variant):
    return "acquire_grid" + ("" if family == "plain" else "_" + family) + variant


def _call(eng, family, variant, nb=NB, prn=PRN, dop=DOP, **kw):
    """The method's positional call (kind passed explicitly for the plain family)."""
    args = (nb, M, prn, dop) + EXTRA[family] if family == "plain" else (nb, M) + EXTRA[family] + (prn, dop)
    return getattr(eng, _name(family, variant))(*args, *((DEV,) if variant.endswith("_device") else ()), **kw)


def _c_args(family, nb, p_prn, n_prn, p_dop, n_dop, p_out):
    """The arguments the symbol is called with, after the engine handle."""
    if family == "plain":
        return (nb, M, p_prn, n_prn, p_dop, n_dop) + EXTRA[family] + (p_out,)
    return (nb, M) + EXTRA[family] + (p_prn, n_prn, p_dop, n_dop, p_out)


def _out_shape(family, variant, nb=NB, n_prn=PRN.size, n_dop=DOP.size):
    if variant == "_best":
        return (nb, n_prn)
    return (nb, n_prn, PHASES[family], n_dop) if family == "weak" else (nb, n_prn, n_dop)


@pytest.mark.parametrize("family,variant", METHODS)
def test_each_method_calls_its_symbol_with_the_callers_arrays(family, variant):
    """Conforming axes are passed in place; the host variants return a new buffer of their layout and hand over its
    address, the device variants hand over the caller's address and return None."""
    eng = _engine()
    got = _call(eng, family, variant)
    [(name, args, prn, dop)] = eng._lib.calls
    assert name == "gb200_" + _name(family, variant)
    if variant.endswith("_device"):
        assert got is None
        p_out = DEV
    else:
        assert got.dtype == (_native.BEST_DTYPE if variant == "_best" else _native.RECORD_DTYPE)
        assert got.shape == _out_shape(family, variant) and got.flags["C_CONTIGUOUS"]
        p_out = got.ctypes.data
    assert args == _c_args(family, NB, PRN.ctypes.data, PRN.size, DOP.ctypes.data, DOP.size, p_out)
    assert np.array_equal(prn, PRN) and np.array_equal(dop, DOP)


@pytest.mark.parametrize("family,variant", [(f, v) for f, v in METHODS if not v.endswith("_device")])
def test_host_methods_convert_the_axes(family, variant):
    """Lists and other dtypes reach the library as int32 PRN rows and float64 Dopplers."""
    eng = _engine()
    got = _call(eng, family, variant, prn=[3, 0, 7], dop=[-500, 0, 250, 1000])
    [(_, args, prn, dop)] = eng._lib.calls
    assert args == _c_args(family, NB, ANY, 3, ANY, 4, got.ctypes.data)
    assert np.array_equal(prn, PRN) and np.array_equal(dop, DOP)


def test_plain_kind_defaults_to_non_coherent():
    eng = _engine()
    eng.acquire_grid(NB, M, PRN, DOP)
    eng.acquire_grid_best(NB, M, PRN, DOP)
    assert [c[1][6] for c in eng._lib.calls] == [_native.NON_COHERENT] * 2


@pytest.mark.parametrize("family", list(EXTRA))
def test_given_out_is_filled_in_place(family):
    eng = _engine()
    out = np.empty(_out_shape(family, ""), _native.RECORD_DTYPE)
    assert _call(eng, family, "", out=out) is out
    assert eng._lib.calls[0][1][-1] == out.ctypes.data


@pytest.mark.parametrize("family", list(EXTRA))
@pytest.mark.parametrize("bad", ["shape", "dtype", "strided"])
def test_wrong_out_raises_before_any_call(family, bad):
    shape = _out_shape(family, "")
    out = {"shape": np.empty((NB + 1,) + shape[1:], _native.RECORD_DTYPE),
           "dtype": np.empty(shape, _native.BEST_DTYPE),
           "strided": np.empty(shape[:-1] + (2 * shape[-1],), _native.RECORD_DTYPE)[..., ::2]}[bad]
    eng = _engine()
    with pytest.raises(ValueError, match="out must be"):
        _call(eng, family, "", out=out)
    assert eng._lib.calls == []


@pytest.mark.parametrize("nb,bit_phases", [(0, 2), (NB, 0), (-1, 2), (-3, 0)])
def test_empty_weak_shape(nb, bit_phases):
    """A weak grid with no cells gets a (0,) record buffer, and a best buffer with no rows, and still reaches the library,
    whose rules name the fault."""
    eng = _engine()
    rec = eng.acquire_grid_weak(nb, M, 4, bit_phases, PRN, DOP)
    best = eng.acquire_grid_weak_best(nb, M, 4, bit_phases, PRN, DOP)
    assert rec.shape == (0,) and best.shape == (max(nb, 0), PRN.size)
    assert [c[1][:4] for c in eng._lib.calls] == [(nb, M, 4, bit_phases)] * 2
    assert [c[1][-1] for c in eng._lib.calls] == [rec.ctypes.data, best.ctypes.data]
    assert eng.acquire_grid_weak(nb, M, 4, bit_phases, PRN, DOP, out=np.empty((0,), _native.RECORD_DTYPE)).shape == (0,)


@pytest.mark.parametrize("family,variant", METHODS)
@pytest.mark.parametrize("rc,exc", [(_native.EINVAL, ValueError), (_native.ESTATE, RuntimeError), (_native.ECUDA, RuntimeError)])
def test_an_error_raises_with_the_symbol_and_message(family, variant, rc, exc):
    eng = _engine(_Lib(rc, b"the library's message"))
    with pytest.raises(exc, match=f"^gb200_{_name(family, variant)}: the library's message$"):
        _call(eng, family, variant)
    assert len(eng._lib.calls) == 1


@pytest.mark.parametrize("family,variant", METHODS)
def test_negative_blocks_reach_the_engine(family, variant):
    """A negative n_blocks is the library's "empty grid" in every family, never a numpy error on the way."""
    eng = _engine()
    got = _call(eng, family, variant, nb=-1)
    [(_, args, _, _)] = eng._lib.calls
    assert args[0] == -1
    if not variant.endswith("_device"):
        assert got.shape == ((0, PRN.size) if variant == "_best" else (0,))


@pytest.mark.parametrize("family", list(EXTRA))
@pytest.mark.parametrize("variant", ["_device", "_best_device"])
def test_device_methods_convert_the_axes(family, variant):
    """The device variants take lists and other dtypes as the host variants do."""
    eng = _engine()
    _call(eng, family, variant, prn=[3, 0, 7], dop=[-500, 0, 250, 1000])
    [(_, args, prn, dop)] = eng._lib.calls
    assert args[-1] == DEV and np.array_equal(prn, PRN) and np.array_equal(dop, DOP)
