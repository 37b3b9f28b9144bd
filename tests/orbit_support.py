"""What the orbit edge tests share, on the CPU and the GPU: seeded per-channel scenarios for the explicit-event path of
gb200_tracker_parse_subframes, each placing one decision of orbit_walk / orbit_change_at at a block, call or table
edge, the oracle run over them and the host build of the same core (tests/emu/orbit_emu.cu)."""
import ctypes as C

import numpy as np

from hostbuild import host_library
from oracle import nav_oracle as nav
from oracle import orbit_oracle as orb

SUB, PHASE, CANNOT, RAISED = nav.KIND_SUBFRAME, nav.KIND_PHASE, nav.KIND_CANNOT, nav.KIND_RAISED
# channels and call lengths of the grid: partial and whole 4-warp blocks of k_parse_subframes, idle warps, and the
# 128-thread blocks of k_sv_observations around their edges
CHANNELS = (1, 3, 4, 5, 8, 31, 32)
CALL_MS = (1, 127, 128, 129, 256, 257)
# every scenario but the capacity trio, which a case with three or more channels puts first
SCENARIOS = ("placed", "stacked", "raise_first", "raise_last", "raise_shared", "raise_before", "drop_first",
             "drop_1", "drop_127", "drop_128", "drop_last", "empty")
CALLS = 3  # two calls of the scenario, then one with no events and no drops


class Pool:
    """One channel's subframes (ids cycling 1..5, TOW counts rising), handed out in turn."""

    def __init__(self, seed, sv):
        rng = np.random.default_rng(seed)
        self.words = [orb.words_of(sf) for sf in orb.ephemeris_subframes(orb.realistic_ephemeris(rng, sv), 25,
                                                                         tow0=int(rng.integers(1000, 90000)), seed=seed)]
        self.k = 0
        self.t = float(rng.uniform(0.0, 100.0))

    def next(self):
        w = self.words[self.k % len(self.words)]
        self.k += 1
        self.t += 0.25
        return w, self.t


def _ev(pool, kind, m):
    w, te = pool.next()
    return (kind, w, 0.0, te, m)


def scenario(name, n_ms, call, pool, stride=None):
    """(events [(kind, words, receiver_timestamp, trailing_edge, ms)], drop_ms) of one channel's call."""
    last = n_ms - 1
    sub = lambda m: _ev(pool, SUB, m)  # noqa: E731
    if name == "placed":  # subframes at ms 0, 127, 128 and n_ms - 1, kinds 1 and 2 between them
        ms = sorted({m for m in (0, 127, 128, last) if m < n_ms})
        ev = []
        for m in ms:
            ev += [sub(m), _ev(pool, PHASE, m)]
        return ev, -1
    if name == "stacked":  # two subframes in one millisecond, then three in the last, kinds 1 and 2 interleaved
        a = min(64, last)
        return [_ev(pool, PHASE, a), sub(a), _ev(pool, CANNOT, a), sub(a), sub(last), _ev(pool, PHASE, last), sub(last),
                _ev(pool, CANNOT, last), sub(last)], -1
    if name == "raise_first":  # a raise at ms 0, a subframe after it in that millisecond and later
        return [_ev(pool, RAISED, 0), sub(0), sub(min(5, last))], -1
    if name == "raise_last":  # subframes in earlier milliseconds, the raise at n_ms - 1
        return [sub(0), sub(last // 2), _ev(pool, RAISED, last)], -1
    if name == "raise_shared":  # a subframe, then the raise, in one millisecond: the subframe holds there
        m = last // 2
        return [sub(0), sub(m), _ev(pool, RAISED, m), sub(m)] + ([sub(last)] if last > m else []), -1
    if name == "raise_before":  # the raise first in a millisecond with subframes: none of them holds
        m = last // 2
        return [sub(0)] * (m > 0) + [_ev(pool, RAISED, m), sub(m), sub(m)], -1
    if name.startswith("drop_"):  # dropped at d, with events at and after it, which are ignored
        d = {"first": 0, "1": 1, "127": 127, "128": 128, "last": last}[name[5:]]
        d = min(d, last)
        if name == "drop_first" and call == 0:  # counting when the next call drops it at its ms 0
            return [sub(0), sub(last)], -1
        ev = [sub(m) for m in sorted({0, d // 2, d - 1}) if 0 <= m < d]
        ev += [sub(d), _ev(pool, RAISED, d)] + [sub(m) for m in range(d + 1, min(d + 3, n_ms))]
        return ev, d
    if name == "capacity":  # stride subframes before a drop at n_ms - 1: the change table's stride + 2 entries
        if n_ms == 1:
            return [sub(0) for _ in range(stride)], -1
        return [sub(int(m)) for m in np.linspace(0, last - 1, stride).astype(int)], last
    if name == "short":  # stride - 1 subframes
        return [sub(int(m)) for m in np.linspace(0, last, stride - 1).astype(int)], -1
    if name == "none":
        return [], -1
    if name == "empty":  # no events: counts from 1 in its first call, on from the carried count after
        return [], -1
    raise ValueError(name)


def case_names(n_ch, n_ms):
    """The scenario of every channel of a grid case: the capacity trio first when there are three channels or more,
    then the others in turn from an offset that moves with the case, so that one-channel cases differ."""
    head = ["capacity", "none", "short"] if n_ch >= 3 else []
    off = CHANNELS.index(n_ch) * len(CALL_MS) + CALL_MS.index(n_ms) if n_ch in CHANNELS and n_ms in CALL_MS else 0
    rest = [SCENARIOS[(off + k) % len(SCENARIOS)] for k in range(n_ch - len(head))]
    return head + rest


def case_calls(n_ch, n_ms, seed=0):
    """[(n_ms, [per channel: (events, drop_ms)])] of a grid case, and the channels' scenario names."""
    names = case_names(n_ch, n_ms)
    pools = [Pool(1000 * seed + 37 * n_ms + c, 1 + c) for c in range(n_ch)]
    calls = []
    for call in range(CALLS):
        if call == CALLS - 1:
            calls.append((n_ms, [([], -1) for _ in range(n_ch)]))
            continue
        chans = [None] * n_ch
        for c, name in enumerate(names):
            if name not in ("capacity", "none", "short"):
                chans[c] = scenario(name, n_ms, call, pools[c])
        stride = max([4] + [len(ch[0]) for ch in chans if ch is not None]) + 1
        for c, name in enumerate(names):
            if chans[c] is None:
                chans[c] = scenario(name, n_ms, call, pools[c], stride)
        calls.append((n_ms, chans))
    return calls, names


# the 6000-count fix gate: per channel of gate_calls, the (call, in-call index) of its first millisecond past the gate
GATE_LEFT = ((0, 6003), (0, 6000), (1, 101), (2, 10), (1, 2901))


def gate_calls(seed=7):
    """Five channels in calls of 6100, 5990 and 100 ms around the 6000-count gate: two leave it inside the first call
    (after subframes at ms 0..2, and counting from the call's start), three with a count carried across a call boundary
    (subframes at ms 198..200, at the last ms and at 3000 of the first call).  GATE_LEFT says where."""
    pools = [Pool(5000 + seed * 10 + c, 20 + c) for c in range(5)]
    first = [(0, 1, 2), (), (198, 199, 200), (6099,), (3000,)]
    calls = [(6100, [([_ev(pools[c], SUB, m) for m in ms], -1) for c, ms in enumerate(first)])]
    calls.append((5990, [([_ev(pools[0], SUB, 0)] if c == 0 else [], -1) for c in range(5)]))
    calls.append((100, [([], -1)] * 5))
    return calls


def oracle_events(events):
    """The oracle's (kind, words, trailing_edge, ms) of events (kind, words, receiver_timestamp, trailing_edge, ms)."""
    return [(k, w, te, m) for k, w, _, te, m in events]


def obs_rows(o) -> np.ndarray:
    """Oracle observations [(tow, dsv, x, y, z, prn_count, flags)] or OBSERVATION_DTYPE records -> rows of tow, x, y,
    z, prn count, flags (the frozen flag kept)."""
    if isinstance(o, np.ndarray) and o.dtype.names:
        return np.stack([o["tow"], o["x"], o["y"], o["z"], o["prn_count"].astype(np.float64),
                         o["flags"].astype(np.float64)], axis=1)
    return np.array([[r[0], r[2], r[3], r[4], r[5], r[6]] for r in o], dtype=np.float64).reshape(-1, 6)


def fields_rows(recs) -> np.ndarray:
    """FIELDS_DTYPE records -> rows (event_index, ms, id, tow, ints[2], bits[4], widths[4], values[10])."""
    return np.array([[r["event_index"], r["ms"], r["subframe_id"], r["tow_seconds"], *r["ints"], *r["bits"],
                      *r["bit_widths"], *r["values"]] for r in recs], dtype=np.float64).reshape(-1, 24)


def oracle_fields_rows(fields) -> np.ndarray:
    return np.array([[j, m, f["subframe_id"], f["tow_seconds"], *f["ints"], *f["bits"], *f["widths"], *f["values"]]
                     for j, m, f in fields], dtype=np.float64).reshape(-1, 24)


class OracleRun:
    """The oracle over a case's calls, one OrbitOracle per channel: per call and channel the field rows, observation
    rows and (params, set mask, prn count, counting) after the call."""

    def __init__(self, calls):
        n_ch = len(calls[0][1])
        svs = [orb.OrbitOracle() for _ in range(n_ch)]
        self.fields, self.obs, self.state = [], [], []
        for n_ms, chans in calls:
            f, o, s = [], [], []
            for c, (events, drop) in enumerate(chans):
                fc, oc = orb.run_call(svs[c], oracle_events(events), drop, n_ms)
                p, mask = svs[c].params()
                f.append(oracle_fields_rows(fc))
                o.append(obs_rows(oc))
                s.append((p, mask, svs[c].count, svs[c].counting))
            self.fields.append(f)
            self.obs.append(o)
            self.state.append(s)


class OrbitEmulator:
    """The host build of orbit_core.cuh, one state per channel, run as k_parse_subframes and k_sv_observations run it."""

    def __init__(self, n_ch):
        self.lib = host_library("orbit_emu")
        self.lib.orbit_emu_call.restype = C.c_int
        self.states = [(C.c_char * self.lib.orbit_emu_state_size())() for _ in range(n_ch)]
        for st in self.states:
            self.lib.orbit_emu_init(st)

    def call(self, c, events, drop, n_ms):
        """FIELDS_DTYPE [fields], OBSERVATION_DTYPE [n_ms] and (params, mask, count, counting) after the call."""
        from gypsum_b200._native import FIELDS_DTYPE, OBSERVATION_DTYPE, SUBFRAME_DTYPE

        n = max(1, len(events))
        ev, ms = np.zeros(n, dtype=SUBFRAME_DTYPE), np.zeros(n, dtype=np.int32)
        for j, (kind, w, t0, t1, m) in enumerate(events):
            ev[j]["kind"], ev[j]["words"], ev[j]["receiver_timestamp"], ev[j]["trailing_edge_receiver_timestamp"] = \
                kind, w, t0, t1
            ms[j] = m
        fields, obs = np.zeros(n, dtype=FIELDS_DTYPE), np.zeros(n_ms, dtype=OBSERVATION_DTYPE)
        nf = self.lib.orbit_emu_call(self.states[c], len(events), ev.ctypes.data_as(C.c_void_p),
                                     ms.ctypes.data_as(C.c_void_p), drop, n_ms, fields.ctypes.data_as(C.c_void_p),
                                     obs.ctypes.data_as(C.c_void_p))
        p, out = np.zeros(orb.N_PARAMS), np.zeros(3, dtype=np.int64)
        self.lib.orbit_emu_params(self.states[c], p.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
        return fields[:nf], obs, (p, int(out[0]), int(out[1]), bool(out[2]))


def assert_state(got, want, what=""):
    """(params, set mask, prn count, counting) exact."""
    assert np.array_equal(got[0], want[0]) and got[1] == want[1], what
    assert got[2] == want[2] and got[3] == want[3], (what, got[2:], want[2:])


def assert_edge(name, events, drop, n_ms, call, obs, state, prev):
    """The edge scenario `name` is named for, on one call's oracle rows (obs_rows) and state after it; prev: the
    channel's (prn count, frozen) at the end of the call before (None in the first call).  Returns the edges shown."""
    cnt, flags = obs[:, 4].astype(int), obs[:, 5].astype(int)
    frozen = (flags & orb.OBS_FROZEN) > 0
    sub_ms = [m for k, _, _, _, m in events if k == SUB]
    last = n_ms - 1
    before = prev[0] if prev is not None else -1
    if prev is not None and prev[1]:  # frozen in an earlier call: nothing changes any more
        assert frozen.all() and (cnt == before).all()
        return ["stays frozen"]
    if name == "placed":
        assert sorted(set(sub_ms)) == sorted({m for m in (0, 127, 128, last) if m < n_ms})
        assert set(np.flatnonzero(cnt == 0)) == set(sub_ms)  # each subframe holds from its own millisecond
        assert any(k != SUB for k, *_ in events)
        return [f"subframe at {m}" for m in sorted(set(sub_ms))]
    if name == "stacked":
        at_last = [orb.parse(w)["tow_seconds"] for k, w, _, _, m in events if k == SUB and m == last]
        assert len(at_last) >= 3 and len(set(at_last)) == len(at_last)
        assert state[0][orb.TOW_LAST] == at_last[-1] and cnt[last] == 0  # the last of the millisecond holds
        return [f"{len(at_last)} subframes at {last}"]
    if name == "raise_first":
        assert frozen.all() and (cnt == before).all()
        return ["raise at 0"]
    if name == "raise_last":
        assert frozen[last] and not frozen[:last].any()
        assert n_ms == 1 or cnt[last] == cnt[last - 1]  # the raising millisecond is not counted
        return [f"raise at {last}"]
    if name in ("raise_shared", "raise_before"):
        m = last // 2
        assert frozen[m:].all() and not frozen[:m].any()
        at_m = [(k, orb.parse(w)["tow_seconds"]) for k, w, _, _, e in events if e == m]
        r = [k for k, _ in at_m].index(RAISED)
        tows_before = [t for k, t in at_m[:r] if k == SUB]
        tows_after = [t for k, t in at_m[r + 1:] if k == SUB]
        assert tows_after and not set(tows_after) & set(tows_before)
        if name == "raise_shared":  # the subframes before the raise hold, the ones after it do not
            assert tows_before and cnt[m] == 0 and state[0][orb.TOW_LAST] == tows_before[-1]
        else:  # the raise first: nothing of its millisecond holds or counts
            assert not tows_before and state[0][orb.TOW_LAST] not in tows_after
            assert cnt[m] == (cnt[m - 1] if m > 0 else before)
        return [f"{name} at {m}"]
    if name.startswith("drop_"):
        if drop < 0:
            assert name == "drop_first" and call == 0
            return []
        assert (cnt[drop:] == -1).all() and not state[3] and not (state[1] >> orb.TOW_LAST) & 1
        assert any(m >= drop for m in sub_ms) and not frozen.any()  # events at and after it ignored
        if drop > 0:
            assert cnt[drop - 1] >= 0
        elif name == "drop_first":
            assert before >= 0  # counting when the call drops it at its ms 0
        return [f"drop at {drop}"]
    if name == "capacity" and n_ms > 1:
        assert drop == last and all(k == SUB for k, *_ in events) and max(sub_ms) < drop and not frozen.any()
        assert (cnt[drop:] == -1).all()
        return [f"{len(events) + 2} change entries"]
    return []
