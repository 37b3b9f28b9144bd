"""The argument rules of the twelve grid entry points -- gb200_acquire_grid, _semicoherent and _weak, each with its
_device, _best and _best_device variant -- broken one at a time, and two at a time where an argument rule meets an
engine-state rule.  Every entry point of a family raises the same exception with the same message, families raise the
same one for the rules they share, and none launches a kernel or writes to its device output.  The header states the
order in which the rules are checked; the families' own argument tables (test_gpu_semicoherent.py, test_gpu_weak.py)
cover the rest of each segment rule."""
import numpy as np
import pytest

from gpu_support import all_chips
from gypsum_b200 import _native
from oracle import gypsum_oracle as o

pytestmark = pytest.mark.gpu

N, FS, M = 2046, 2046000, 4
BASE = dict(nb=1, m=M, t=2, b=1, kind=_native.NON_COHERENT, prn=np.array([0, 3], np.int32), dop=np.array([0.0, 500.0]))
VARIANTS = ["", "_device", "_best", "_best_device"]
ALL = ("plain", "semicoherent", "weak")
SEGMENTED = ("semicoherent", "weak")
NO_IQ = (RuntimeError, "no IQ loaded (gb200_upload_iq / gb200_bind_iq_device)")
EMPTY = (ValueError, "empty grid")
PARTIAL = {"semicoherent": (ValueError, "ms_per_block (4) is not a whole number of 3-ms coherent segments"),
           "weak": (ValueError, "ms_per_block (4) is not 0 ms plus a whole number (>= 1) of 3-ms coherent segments")}

# rule: (families it applies to, arguments changed from BASE, engine, (exception, message) or one per family)
RULES = {
    "null_output": (ALL, {}, "ready", (ValueError, "null output")),
    "kind": (("plain",), dict(kind=7), "ready", (ValueError, "Unexpected integration type")),
    "no_replicas": (ALL, {}, "no_replicas", (RuntimeError, "no PRN replicas loaded (gb200_set_replicas)")),
    "no_iq": (ALL, {}, "no_iq", NO_IQ),
    "blocks0": (ALL, dict(nb=0), "ready", EMPTY),
    "prn0": (ALL, dict(prn=np.zeros(0, np.int32)), "ready", EMPTY),
    "dop0": (ALL, dict(dop=np.zeros(0)), "ready", EMPTY),
    "nan": (ALL, dict(dop=np.array([0.0, np.nan])), "ready", (ValueError, "Doppler 1 is not finite (nan Hz)")),
    "inf": (ALL, dict(dop=np.array([-np.inf, 0.0])), "ready", (ValueError, "Doppler 0 is not finite (-inf Hz)")),
    "prn_range": (ALL, dict(prn=np.array([0, 32], np.int32)), "ready", (ValueError, "prn index 32 out of range")),
    "samples": (ALL, dict(nb=2), "ready", (ValueError, f"grid needs {2 * M * N} samples, {M * N} loaded")),
    "t0": (SEGMENTED, dict(t=0), "ready", (ValueError, "coherent_ms must be at least 1 (got 0)")),
    "partial": (SEGMENTED, dict(t=3), "ready", PARTIAL),
    "b0": (("weak",), dict(b=0), "ready", (ValueError, "bit_phases (0) must be at least 1 and divide coherent_ms (2)")),
    "b3": (("weak",), dict(b=3), "ready", (ValueError, "bit_phases (3) must be at least 1 and divide coherent_ms (2)")),
    # two rules broken: the argument rule is reported
    "no_iq_and_empty": (ALL, dict(nb=0), "no_iq", EMPTY),
    "no_iq_and_partial": (SEGMENTED, dict(t=3), "no_iq", PARTIAL),
    "kind_and_empty": (("plain",), dict(kind=7, nb=0), "ready", EMPTY),
}


@pytest.fixture(scope="module")
def engines(native_lib):
    x = o.synth_iq(3, N, M, FS, [])
    engs = {k: _native.Engine(FS, N) for k in ("ready", "no_replicas", "no_iq")}
    for k, e in engs.items():
        if k != "no_replicas":
            e.set_replicas(all_chips())
        if k != "no_iq":
            e.upload_iq(x)
    yield engs
    for e in engs.values():
        e.close()


def _call(eng, family, variant, a, null, dev):
    """One entry point with the arguments a; a _device call writes to dev.  null: the output is null -- on a host call
    passed to the library directly, as the Engine methods never do."""
    name = "acquire_grid" + ("" if family == "plain" else "_" + family) + variant
    mid = {"plain": (), "semicoherent": (a["t"],), "weak": (a["t"], a["b"])}[family]
    tail = (a["kind"],) if family == "plain" else ()
    if variant.endswith("_device"):
        return getattr(eng, name)(a["nb"], a["m"], *mid, a["prn"], a["dop"], *tail, 0 if null else dev)
    if null:
        prn, dop = a["prn"], a["dop"]
        rc = getattr(eng._lib, "gb200_" + name)(eng._h, a["nb"], a["m"], *mid, prn.ctypes.data, prn.size, dop.ctypes.data,
                                                 dop.size, *tail, None)
        return eng._check(rc, "gb200_" + name)
    return getattr(eng, name)(a["nb"], a["m"], *mid, a["prn"], a["dop"], *tail)


@pytest.mark.parametrize("rule", list(RULES))
def test_every_entry_point_reports_the_same_rule_and_launches_nothing(engines, rule):
    import torch

    families, change, which, want = RULES[rule]
    eng = engines[which]
    a = dict(BASE, **change)
    guard = {v: torch.full((4096,), 0xFF, dtype=torch.uint8, device="cuda") for v in ("_device", "_best_device")}
    before = eng.launch_count
    got = {}
    for family in families:
        for variant in VARIANTS:
            name = "gb200_acquire_grid" + ("" if family == "plain" else "_" + family) + variant
            with pytest.raises((ValueError, RuntimeError)) as err:
                _call(eng, family, variant, a, rule == "null_output", guard[variant].data_ptr() if variant in guard else 0)
            assert str(err.value).startswith(name + ": "), (rule, str(err.value))
            got[family, variant] = (err.type, str(err.value)[len(name) + 2:])
    for family in families:
        expect = want[family] if isinstance(want, dict) else want
        assert {got[family, v] for v in VARIANTS} == {expect}, (rule, family, {v: got[family, v] for v in VARIANTS})
    assert eng.launch_count == before, rule
    torch.cuda.synchronize()
    for v, buf in guard.items():
        assert (buf.cpu().numpy() == 0xFF).all(), (rule, v, "device output written")
