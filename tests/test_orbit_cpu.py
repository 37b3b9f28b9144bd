"""Subframe fields, the per-satellite world-model state and the per-millisecond satellite time and position on the CPU:
the oracle and the device code (orbit_core.cuh compiled for the host) against timelines recorded from the live
reference's parser and GpsWorldModel (tests/golden/orbit.npz), the LNAV encoder, and the struct layouts."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from hostbuild import host_library
from oracle import nav_oracle as nav
from oracle import orbit_oracle as orb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "orbit.npz")
TIMELINES = ["realistic", "extreme", "week_edge", "order", "mixing", "lost"]


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def orbit_emu():
    lib = host_library("orbit_emu")
    lib.orbit_emu_call.restype = C.c_int
    return lib


def _fields_rows(recs) -> np.ndarray:
    """FIELDS_DTYPE records -> the golden's field rows (id, tow, ints[2], bits[4], values[10])."""
    return np.array([[r["subframe_id"], r["tow_seconds"], *r["ints"], *r["bits"], *r["values"]] for r in recs],
                    dtype=np.float64).reshape(-1, 18)


def _oracle_fields_row(f) -> list:
    return [f["subframe_id"], f["tow_seconds"], *f["ints"], *f["bits"], *f["values"]]


def _want_obs(z, name, c, ch):
    o = z[f"{name}_obs"]
    sel = (o[:, 0] == c) & (o[:, 1] == ch)
    return o[sel, 2].astype(int), o[sel][:, [3, 4, 5, 6, 7, 8]]


def _obs_rows(obs) -> np.ndarray:
    return np.array([[o[0], o[2], o[3], o[4], o[5], o[6] & ~orb.OBS_FROZEN] for o in obs], dtype=np.float64).reshape(-1, 6)


@pytest.mark.parametrize("name", TIMELINES)
def test_oracle_equals_reference(golden, name):
    """Fields, observations and parameter sets of the oracle equal the reference's bit for bit."""
    z = golden
    calls = orb.golden_calls(z, name)
    n_ch = len(calls[0][1])
    svs = [orb.OrbitOracle() for _ in range(n_ch)]
    fields = []
    for c, (n_ms, chans) in enumerate(calls):
        for ch, (events, drop) in enumerate(chans):
            f, obs = orb.run_call(svs[ch], [(k, w, te, m) for k, w, _, te, m in events], drop, n_ms)
            fields += [_oracle_fields_row(x[2]) for x in f]
            ms, want = _want_obs(z, name, c, ch)
            orb.compare_observations(_obs_rows(obs)[ms], want, exact=True)
            p, mask = svs[ch].params()
            assert mask == z[f"{name}_mask"][c, ch]
            assert np.array_equal(p, z[f"{name}_params"][c, ch])
    # the golden lists events by call, then channel: the same order as here
    assert np.array_equal(np.array(fields), z[f"{name}_fields"])


def test_golden_covers_every_case(golden):
    z = golden
    f = z["extreme_fields"]
    assert f[:, 8:].min() < -1e-3 and f[:, 8:].max() > 1e-3  # both ends of the signed ranges
    wk = z["week_edge_obs"]
    assert (wk[:, 8].astype(int) & orb.OBS_COMPLETE).any()
    order = z["order_obs"]
    first_complete = order[(order[:, 8].astype(int) & orb.OBS_COMPLETE) > 0, 2].min()
    assert first_complete == z["order_events"][4, 2]  # after the fifth event (subframe 3), not before
    real = z["realistic_obs"]
    gate = real[(real[:, 0] == 1) & (real[:, 8].astype(int) & orb.OBS_COUNTING > 0)]
    assert (gate[:, 7] > 6000).any() and not (gate[gate[:, 7] > 6000, 8].astype(int) & orb.OBS_FIX_GATE).any()
    lost = z["lost_obs"]
    assert ((lost[:, 0] == 0) & (lost[:, 7] == -1)).any() and (z["lost_mask"][0, 0] >> orb.TOW_LAST) & 1 == 0
    mix = z["mixing_fields"]
    assert mix[0, 7] != mix[3, 7] and mix[0, 0] == mix[3, 0] == 1  # the two subframes 1 carry different IODCs


def _emu_call(lib, st, events, drop, n_ms):
    from gypsum_b200._native import FIELDS_DTYPE, OBSERVATION_DTYPE, SUBFRAME_DTYPE

    ev = np.zeros(max(1, len(events)), dtype=SUBFRAME_DTYPE)
    ms = np.zeros(max(1, len(events)), dtype=np.int32)
    for j, (kind, w, t0, t1, m) in enumerate(events):
        ev[j]["kind"], ev[j]["words"], ev[j]["receiver_timestamp"], ev[j]["trailing_edge_receiver_timestamp"] = kind, w, t0, t1
        ms[j] = m
    fields = np.zeros(max(1, len(events)), dtype=FIELDS_DTYPE)
    obs = np.zeros(n_ms, dtype=OBSERVATION_DTYPE)
    nf = lib.orbit_emu_call(st, len(events), ev.ctypes.data_as(C.c_void_p), ms.ctypes.data_as(C.c_void_p), drop, n_ms,
                            fields.ctypes.data_as(C.c_void_p), obs.ctypes.data_as(C.c_void_p))
    return fields[:nf], obs


def obs_rows(obs) -> np.ndarray:
    """OBSERVATION_DTYPE -> rows of tow, x, y, z, prn count, flags (the frozen flag left out, as the golden has none)."""
    return np.stack([obs["tow"], obs["x"], obs["y"], obs["z"], obs["prn_count"].astype(np.float64),
                     (obs["flags"] & ~orb.OBS_FROZEN).astype(np.float64)], axis=1)


@pytest.mark.parametrize("name", TIMELINES)
def test_device_code_on_host(golden, orbit_emu, name):
    """orbit_core.cuh compiled for the host: fields exact, time of week within 1 ulp, ECEF within 1e-4 m."""
    z = golden
    calls = orb.golden_calls(z, name)
    n_ch = len(calls[0][1])
    states = [(C.c_char * orbit_emu.orbit_emu_state_size())() for _ in range(n_ch)]
    for st in states:
        orbit_emu.orbit_emu_init(st)
    fields = []
    for c, (n_ms, chans) in enumerate(calls):
        for ch, (events, drop) in enumerate(chans):
            f, obs = _emu_call(orbit_emu, states[ch], events, drop, n_ms)
            fields.append(_fields_rows(f))
            assert list(f["ms"]) == [e[4] for e in events if e[0] == 0]
            ms, want = _want_obs(z, name, c, ch)
            orb.compare_observations(obs_rows(obs)[ms], want)
            p = np.zeros(26)
            out = np.zeros(3, dtype=np.int64)
            orbit_emu.orbit_emu_params(states[ch], p.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
            assert out[0] == z[f"{name}_mask"][c, ch]
            assert np.array_equal(p, z[f"{name}_params"][c, ch])
    assert np.array_equal(np.concatenate(fields), z[f"{name}_fields"])


def test_frozen_channel_on_host(orbit_emu):
    """A kind-3 event freezes the channel at the millisecond before it, as the oracle does."""
    rng = np.random.default_rng(5)
    eph = orb.realistic_ephemeris(rng, 7)
    sfs = orb.ephemeris_subframes(eph, 3, tow0=500)
    events = [(0, orb.words_of(sf), 0.0, 1.0 + k, 100 + 100 * k) for k, sf in enumerate(sfs)]
    events.append((nav.KIND_RAISED, orb.words_of(sfs[0]), 0.0, 9.0, 700))
    st = (C.c_char * orbit_emu.orbit_emu_state_size())()
    orbit_emu.orbit_emu_init(st)
    _, obs = _emu_call(orbit_emu, st, events, -1, 1000)
    sv = orb.OrbitOracle()
    _, want = orb.run_call(sv, [(k, w, te, m) for k, w, _, te, m in events], -1, 1000)
    want = np.array([[o[0], o[2], o[3], o[4], o[5], o[6]] for o in want])
    got = np.stack([obs["tow"], obs["x"], obs["y"], obs["z"], obs["prn_count"].astype(float), obs["flags"].astype(float)], 1)
    orb.compare_observations(got, want)
    assert (obs["flags"][700:] & orb.OBS_FROZEN).all() and (obs["prn_count"][699:] == 399).all()


def test_encoder_round_trips_through_the_reference_parser_fields(golden):
    """The encoder's subframes have valid parity, and the oracle parser returns the planted values exactly (the
    reference parser itself reads the same subframes in the golden, see test_oracle_equals_reference)."""
    rng = np.random.default_rng(8)
    for sv in (1, 14, 32):
        eph = orb.realistic_ephemeris(rng, sv)
        for k, sf in enumerate(orb.ephemeris_subframes(eph, 5, tow0=1234, seed=sv)):
            assert nav.check_parity(sf) == 0x3FF
            f = orb.parse(orb.words_of(sf))
            assert f["subframe_id"] == k + 1 and f["tow_seconds"] == 6.0 * (1234 + k)
            want = orb.planted_values(k + 1, eph)
            assert f["values"][:len(want)] == want
            if k == 0:
                assert f["ints"][0] == eph["wn"] and f["bits"][3] == eph["iodc"]
            if k == 4:
                assert f["bits"][:2] == [1, sv]
    # the encoder wrote the golden's subframes: the reference parsed them into exactly the values it planted
    assert len(golden["realistic_fields"]) == 24


def test_layouts_python_c_and_cpp(orbit_emu, tmp_path):
    from gypsum_b200._native import FIELDS_DTYPE, OBSERVATION_DTYPE

    fnames = ["event_index", "ms", "subframe_id", "tow_seconds", "ints", "bits", "bit_widths", "values"]
    onames = ["tow", "dsv", "x", "y", "z", "prn_count", "flags"]
    py = ([FIELDS_DTYPE.fields[k][1] for k in fnames] + [FIELDS_DTYPE.itemsize]
          + [OBSERVATION_DTYPE.fields[k][1] for k in onames] + [OBSERVATION_DTYPE.itemsize])
    assert py == [0, 4, 8, 16, 24, 32, 48, 64, 144, 0, 8, 16, 24, 32, 40, 48, 56]
    cpp = np.zeros(17, dtype=np.int64)
    orbit_emu.orbit_emu_layout(cpp.ctypes.data_as(C.c_void_p))
    assert list(cpp) == py
    src = tmp_path / "layout.c"
    src.write_text("#include <stdio.h>\n#include <stddef.h>\n#include \"gypsum_b200.h\"\nint main(void) {\n"
                   + "".join(f'    printf("%d\\n", (int)offsetof(gb200_subframe_fields, {k}));\n' for k in fnames)
                   + '    printf("%d\\n", (int)sizeof(gb200_subframe_fields));\n'
                   + "".join(f'    printf("%d\\n", (int)offsetof(gb200_sv_observation, {k}));\n' for k in onames)
                   + '    printf("%d\\n", (int)sizeof(gb200_sv_observation));\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", f"-I{os.path.join(ROOT, 'include')}", str(src),
                    "-o", str(exe)], check=True, capture_output=True)
    c = [int(v) for v in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    assert c == py


def test_python_subframe_types():
    from gypsum_b200._native import FIELDS_DTYPE
    from gypsum_b200.navigation_message_parser import GpsSubframeId, subframe_from_fields

    rng = np.random.default_rng(3)
    eph = orb.realistic_ephemeris(rng, 9)
    for k, sf in enumerate(orb.ephemeris_subframes(eph, 5, tow0=77)):
        f = orb.parse(orb.words_of(sf))
        rec = np.zeros(1, dtype=FIELDS_DTYPE)[0]
        rec["subframe_id"], rec["tow_seconds"], rec["ints"], rec["bits"], rec["bit_widths"] = (
            f["subframe_id"], f["tow_seconds"], f["ints"], f["bits"], f["widths"])
        rec["values"] = f["values"]
        s = subframe_from_fields(rec)
        assert s.subframe_id == list(GpsSubframeId)[k]
        if k == 0:
            assert s.week_num == eph["wn"] + 2048 and len(s.issue_of_data_clock) == 10
            assert s.issue_of_data_clock == [(eph["iodc"] >> (9 - i)) & 1 for i in range(10)]
        if k == 1:
            assert s.sqrt_semi_major_axis == orb.planted_values(2, eph)[6] and isinstance(s.reference_time_ephemeris, int)
