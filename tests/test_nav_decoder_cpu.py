"""Navigation-message subframe decoding on the CPU: the oracle and the device state machine (nav_core.cuh compiled for
the host) against event streams recorded from the live reference decoder (tests/golden/nav_decoder.npz), the LNAV
generator against the IS-GPS-200 parity equations, and the gb200_subframe_event layout."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import nav_oracle as nav

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "nav_decoder.npz")
STREAMS = ["clean", "negated", "unknown", "bad_tlm_how", "false_pair", "no_preamble", "raise", "parity"]


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def nav_emu(tmp_path_factory):
    src = os.path.join(ROOT, "tests", "emu", "nav_emu.cu")
    out = str(tmp_path_factory.mktemp("nav_emu") / "libnavemu.so")
    subprocess.run(["nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-o", out, src], check=True,
                   capture_output=True)
    lib = C.CDLL(out)
    lib.nav_emu_run.restype = C.c_int
    return lib


def _rows(events):
    """SUBFRAME_DTYPE events (bit_index within the call) -> the golden's rows and words."""
    rows = np.array([[e["bit_index"], e["kind"], e["subframe_id"], e["tow"], e["phase"], e["polarity"], e["parity_ok"],
                      e["receiver_timestamp"], e["trailing_edge_receiver_timestamp"]] for e in events],
                    dtype=np.float64).reshape(-1, 9)
    words = np.array([e["words"] for e in events], dtype=np.int64).reshape(-1, 10)
    return rows, words


def _emu_run(lib, bits, t0, t1, splits):
    from gypsum_b200._native import SUBFRAME_DTYPE, subframe_event_capacity

    st = (C.c_char * lib.nav_emu_state_size())()
    lib.nav_emu_init(st)
    rows, words = [], []
    edges = [0, *splits, len(bits)]
    for a, b in zip(edges[:-1], edges[1:]):
        x = np.ascontiguousarray(bits[a:b], dtype=np.int32)
        u0, u1 = np.ascontiguousarray(t0[a:b]), np.ascontiguousarray(t1[a:b])
        cap = subframe_event_capacity(b - a)
        ev = np.zeros(cap, dtype=SUBFRAME_DTYPE)
        n = lib.nav_emu_run(st, b - a, x.ctypes.data_as(C.c_void_p), u0.ctypes.data_as(C.c_void_p),
                            u1.ctypes.data_as(C.c_void_p), ev.ctypes.data_as(C.c_void_p), cap)
        assert n <= cap
        r, w = _rows(ev[:n])
        r[:, 0] += a
        rows.append(r)
        words.append(w)
    summary = np.zeros(6, dtype=np.int64)
    lib.nav_emu_summary(st, summary.ctypes.data_as(C.c_void_p))
    return np.concatenate(rows), np.concatenate(words), list(summary)


@pytest.mark.parametrize("stream", STREAMS)
def test_oracle_equals_reference(golden, stream):
    z = golden
    events, final = nav.decode(z[f"{stream}_bits"], z[f"{stream}_t0"], z[f"{stream}_t1"])
    rows, words = nav.events_to_arrays(events)
    assert np.array_equal(rows, z[f"{stream}_events"])
    assert np.array_equal(words, z[f"{stream}_words"])
    assert final == list(z[f"{stream}_final"])


def test_golden_streams_cover_every_path(golden):
    z = golden
    kinds = {s: set(z[f"{s}_events"][:, 1].astype(int)) for s in STREAMS}
    assert kinds["raise"] == {nav.KIND_RAISED} and nav.KIND_CANNOT in kinds["no_preamble"]
    assert (z["negated_events"][:, 5] == -1).all()
    # subframes emitted with no polarity after a reset inside the drain loop
    assert ((z["unknown_events"][:, 1] == 0) & (z["unknown_events"][:, 5] == 0)).any()
    assert ((z["no_preamble_events"][:, 1] == 0) & (z["no_preamble_events"][:, 4] == -1)).any()
    # the first phase of the false-pair stream is the planted pair at 50, and the real one follows
    ph = z["false_pair_events"][z["false_pair_events"][:, 1] == 1]
    assert ph[0, 4] == 50 and len(ph) >= 2
    par = z["parity_events"]
    assert sorted(set(par[par[:, 1] == 0, 6].astype(int))) == sorted({0x3FF, 0x3FF & ~(1 << 3), 0x3FF & ~(3 << 4)})


@pytest.mark.parametrize("stream", STREAMS)
@pytest.mark.parametrize("cut", ["whole", "ragged", "every_bit_near_sync"])
def test_device_state_machine_on_host(golden, nav_emu, stream, cut):
    """The golden streams through the state machine the GPU runs, in one call and cut into calls so that the state
    carries across them."""
    z = golden
    bits = z[f"{stream}_bits"]
    n = bits.size
    splits = {"whole": [], "ragged": list(range(997, n, 997)) + [1, 599, 600, 601],
              "every_bit_near_sync": list(range(590, 620)) + list(range(3595, 3610))}[cut]
    splits = sorted(s for s in set(splits) if 0 < s < n)
    rows, words, final = _emu_run(nav_emu, bits, z[f"{stream}_t0"], z[f"{stream}_t1"], splits)
    assert np.array_equal(rows, z[f"{stream}_events"])
    assert np.array_equal(words, z[f"{stream}_words"])
    assert final == list(z[f"{stream}_final"])


def test_queue_overflow_latches_at_the_documented_bit(nav_emu):
    """No preamble ever: CannotDetermine from 3600 queued bits, and the bit that arrives with 4096 queued stops the
    decoder without being taken."""
    bits = nav.no_preamble_noise(11, 4300)
    bits[1000:1003] = -1
    t0, t1 = nav.bit_times(bits.size)
    rows, _, final = _emu_run(nav_emu, bits, t0, t1, [2000, 4095, 4096, 4097])
    assert final == [-1, 0, 0, 4096, 2, 4096]
    assert np.array_equal(rows[:, 0], np.arange(3599, 4096)) and (rows[:, 1] == nav.KIND_CANNOT).all()
    events, state = nav.decode(bits, t0, t1)
    assert state == final and np.array_equal(nav.events_to_arrays(events)[0], rows)


def test_lnav_generator_parity():
    for seed in range(3):
        sfs = nav.lnav_frames(seed, 10, first_id=2, tow0=777)
        prev30 = 0
        for k, sf in enumerate(sfs):
            assert len(sf) == 300
            assert nav.check_parity(sf) == 0x3FF  # word 1 may start from 00: the previous word 10 ends in 00
            assert sf[58:60] == [0, 0] and sf[298:300] == [0, 0]  # words 2 and 10: D29 = D30 = 0
            assert tuple(sf[:8]) == nav.PREAMBLE and prev30 == 0
            how = [v ^ sf[29] for v in sf[30:54]]
            assert nav.word_value(how[:17]) == 777 + k and nav.word_value(how[19:22]) == (1 + k) % 5 + 1
            prev30 = sf[-1]
        bad = [list(sf) for sf in sfs]
        bad[3][30 * 6 + 2] ^= 1  # a data bit: word 7 only
        assert nav.check_parity(bad[3]) == 0x3FF & ~(1 << 6)
        bad[4][30 * 2 + 29] ^= 1  # D30: words 3 and 4
        assert nav.check_parity(bad[4]) == 0x3FF & ~(3 << 2)


def test_subframe_bits_helper():
    from gypsum_b200._native import SUBFRAME_DTYPE, subframe_bits

    sf = nav.lnav_frames(2, 1)[0]
    ev = np.zeros(1, dtype=SUBFRAME_DTYPE)[0]
    ev["words"] = [nav.word_value(sf[30 * k: 30 * k + 30]) for k in range(10)]
    assert subframe_bits(ev) == list(sf)


def test_event_layout_python_c_and_cpp(nav_emu, tmp_path):
    from gypsum_b200._native import SUBFRAME_DTYPE

    names = ["receiver_timestamp", "trailing_edge_receiver_timestamp", "words", "kind", "bit_index", "subframe_id", "tow",
             "phase", "polarity", "parity_ok"]
    py = [SUBFRAME_DTYPE.fields[k][1] for k in names] + [SUBFRAME_DTYPE.itemsize]
    assert py == [0, 8, 16, 56, 60, 64, 68, 72, 76, 80, 96]
    cpp = np.zeros(11, dtype=np.int64)
    nav_emu.nav_emu_layout(cpp.ctypes.data_as(C.c_void_p))
    assert list(cpp) == py
    src = tmp_path / "layout.c"
    src.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"gypsum_b200.h\"\nint main(void) {\n"
                   + "".join(f'    printf("%d\\n", (int)offsetof(gb200_subframe_event, {k}));\n' for k in names)
                   + '    printf("%d\\n", (int)sizeof(gb200_subframe_event));\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", f"-I{os.path.join(ROOT, 'include')}", str(src),
                    "-o", str(exe)], check=True, capture_output=True)
    c = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert c == py


def test_event_capacity_bounds_every_golden_call(golden):
    from gypsum_b200._native import subframe_event_capacity

    for s in STREAMS:
        ev = golden[f"{s}_events"]
        for chunk in (97, 997, 4001):
            idx = ev[:, 0].astype(int) // chunk
            worst = np.bincount(idx).max() if idx.size else 0
            assert worst <= subframe_event_capacity(chunk)
