"""What the position-fix tests share, on the CPU and the GPU: the parity bounds, the host build of the fix core
(tests/emu/fix_emu.cu) and the way a scripted timeline reaches the device.  torch and gypsum_b200 are imported inside the
functions that need them, so the CPU tests collect and run without the library."""
import ctypes as C

import numpy as np

from hostbuild import host_library
from oracle import fix_oracle as fx

# parity bounds of the host and device core against the reference's numpy (DESIGN.md §6), a small multiple of the
# spread measured on the recorded timelines (clock bias 1.2e-15 s, position 2.7e-7 m, slides identical)
POS_M, BIAS_S, SLIDE_ULPS = 2e-6, 1e-14, 4
# the least-squares mode on five or more rows of the recorded and scripted timelines (DESIGN.md §8c).  The golden rows
# are 1e4 km off any common solution, and Gauss-Newton on the squared ranges does not converge there (numpy's last step
# is up to 1.4e7 m in `five`): host and numpy follow the same cycle apart by rounding, measured up to 1.3 m, 2.7e-9 s and
# 34 ulp of the slide.  tests/test_gpu_fix_lsq.py's scripted six rows converge, on a poorer geometry: 5.6e-4 m,
# 6.1e-13 s, 0 ulp.
MANY_POS_M, MANY_BIAS_S, MANY_SLIDE_ULPS = 4.0, 1e-8, 100


def slide_tol(s):
    """SLIDE_ULPS units in the last place of a slide (about 3e5 s on the recorded timelines)."""
    return SLIDE_ULPS * 2.0 ** -52 * np.abs(s)


def fix_emulator():
    """compute(rows, rx, slide) -> one fx.FIX_DTYPE record: fix_core.cuh on the host, as the device computes the fix of
    one millisecond from rows [n][4] of (tow, x, y, z), n >= 4 (more than four rows: the least-squares mode)."""
    lib = host_library("fix_emu")
    lib.fix_emu_compute_n.restype = C.c_int
    lib.fix_emu_compute_n.argtypes = [C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_void_p]

    def compute(rows, rx, slide):
        r = np.ascontiguousarray(rows, dtype=np.float64).reshape(-1, 4)
        out = np.zeros(1, dtype=fx.FIX_DTYPE)
        lib.fix_emu_compute_n(r.ctypes.data, len(r), float(rx), float(slide), out.ctypes.data)
        return out[0]

    return compute


def parse_events(trk, chans, n_ms):
    """chans: [(events [(kind, words, trailing_edge, ms)], drop_ms)] through device event arrays."""
    import torch

    from gypsum_b200._native import SUBFRAME_DTYPE

    n_ch = len(chans)
    stride = max(1, max(len(ev) for ev, _ in chans))
    host = np.zeros((n_ch, stride), dtype=SUBFRAME_DTYPE)
    ems = np.zeros((n_ch, stride), dtype=np.int32)
    counts = np.array([len(ev) for ev, _ in chans], dtype=np.int32)
    for c, (events, _) in enumerate(chans):
        for j, (kind, w, te, m) in enumerate(events):
            host[c, j]["kind"], host[c, j]["words"], host[c, j]["trailing_edge_receiver_timestamp"] = kind, w, te
            ems[c, j] = m
    dev = torch.from_numpy(host.view(np.uint8).reshape(n_ch, -1)).cuda()
    trk.parse_subframes(dev.data_ptr(), counts, stride, ems, np.array([d for _, d in chans], dtype=np.int32), n_ms)


def rows_at(obs, channels, m):
    """The rows (tow, x, y, z) of the given channels at millisecond m, from the device's observations."""
    return [(obs[ch, m]["tow"], obs[ch, m]["x"], obs[ch, m]["y"], obs[ch, m]["z"]) for ch in channels]


def run_calls(engine, calls, device_out=False, solver=None):
    """A timeline ([(rx, chans)], the layout of fx.golden_calls) through one tracker, call after call; per call the
    records (read back from a device buffer if device_out), the device's observations and receiver_state().  A solver
    is set before the first call; None leaves the tracker's own."""
    import torch

    from gypsum_b200 import _native

    n_ch = len(calls[0][1])
    trk = _native.Tracker(engine, list(range(n_ch)), [0.0] * n_ch, [0.0] * n_ch, [0] * n_ch)
    if solver is not None:
        trk.set_fix_solver(solver)
    out = []
    for rx, chans in calls:
        parse_events(trk, chans, len(rx))
        if device_out:
            dev = torch.empty(len(rx) * _native.FIX_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
            trk.position_fixes_device(rx, dev.data_ptr())
            torch.cuda.synchronize()
            rec = dev.cpu().numpy().view(_native.FIX_DTYPE).copy()
        else:
            rec = trk.position_fixes(rx)
        out.append((rec, trk.observations(), trk.receiver_state()))
    trk.close()
    return out


def run_golden(engine, golden_path, name, device_out=False, solver=None):
    """run_calls on a recorded timeline: the golden file, its calls and what run_calls returns."""
    z = np.load(golden_path)
    calls = fx.golden_calls(z, name)
    return z, calls, run_calls(engine, calls, device_out, solver)


def scripted_timeline():
    """Six channels with their own planted ephemerides and the same TOW counts, in two calls (the layout of
    fx.golden_calls), built as tools/make_golden_fix.py builds its timelines:
      call 0  subframes 1-3 on all six at ms 100 / 200 / 300: six ready from 300; channel 4 loses lock at 600 and
              channel 5 at 700 (6 -> 5 -> 4 inside the segment); subframe 4 on channels 0-3 at 900 resets the slide
      call 1  subframe 5 on all six at ms 200: channels 4 and 5 return, six ready again; a receiver-clock jump of
              -0.2 s at ms 600 inside that segment, so the chain check misses and the repair solves six rows"""
    from oracle import nav_oracle as nav
    from oracle import orbit_oracle as orb

    rng = np.random.default_rng(2031)
    svs = (2, 6, 11, 17, 24, 29)
    words = [[orb.words_of(sf) for sf in orb.ephemeris_subframes(orb.realistic_ephemeris(rng, sv), 5, tow0=50000,
                                                                  seed=100 + c)] for c, sv in enumerate(svs)]
    sched = [[[(0, 100), (1, 200), (2, 300), (3, 900)], [(4, 200)]] for _ in range(4)]
    sched += [[[(0, 100), (1, 200), (2, 300)], [(4, 200)]] for _ in range(2)]
    drops = [[-1, -1, -1, -1, 600, 700], [-1] * 6]
    calls_ms, jumps = [1500, 1200], [(1, 600, -0.2)]
    out, t0 = [], 0.0
    for c, n_ms in enumerate(calls_ms):
        def offset(m, c=c):
            return sum(j for jc, jm, j in jumps if (jc, jm) <= (c, m))

        rx = np.array([t0 + 0.001 * m + offset(m) for m in range(n_ms)])
        chans = [([(nav.KIND_SUBFRAME, words[ch][k], round(t0 + 0.001 * m - 0.0003 * ch + offset(m), 7), m)
                   for k, m in sched[ch][c]], drops[c][ch]) for ch in range(len(svs))]
        out.append((rx, chans))
        t0 += 0.001 * n_ms
    return out


def ready_rows(obs, order, m):
    """The ready rows (flags 2 and 4) of millisecond m in the world model's order, from the device's observations."""
    return [(obs[ch, m]["tow"], obs[ch, m]["x"], obs[ch, m]["y"], obs[ch, m]["z"]) for ch in order
            if (obs[ch, m]["flags"] & 6) == 6]


def call_starts(calls):
    """The global millisecond each call of a timeline starts at, and the timeline's length."""
    starts = np.cumsum([0] + [len(rx) for rx, _ in calls])
    return [int(s) for s in starts[:-1]], int(starts[-1])


def resplit(calls, cuts):
    """A timeline (the layout of fx.golden_calls) cut into more calls: its own call boundaries are kept and one is added
    at every global millisecond in `cuts`.  Events and drops move to the call that holds them, their milliseconds
    relative to it, and the receiver timestamps are the concatenated ones, sliced.  A drop holds for its call only (the
    header comment of gb200_tracker_parse_subframes), so each piece of a call that starts after one of its channels'
    drop drops that channel again at its millisecond 0: the receiver then sees what it saw in the one call."""
    bounds, total = call_starts(calls)
    rx_all = np.concatenate([rx for rx, _ in calls])
    starts = sorted(set(bounds) | {int(c) for c in cuts if 0 < c < total})
    out = []
    for s, e in zip(starts, starts[1:] + [total]):
        ci = max(i for i, b in enumerate(bounds) if b <= s)
        b = bounds[ci]
        chans = []
        for events, drop in calls[ci][1]:
            ev = [(k, w, te, m + b - s) for k, w, te, m in events if s <= m + b < e]
            if drop < 0 or drop + b >= e:
                d = -1
            else:
                d = max(drop + b - s, 0)
            chans.append((ev, d))
        out.append((rx_all[s:e], chans))
    return out


class OracleTimeline:
    """A receiver oracle (fx or fix_lsq_oracle) run once over a timeline's calls, in global milliseconds: the records
    concatenated, {ms: slide} of every reset, {ms: rows} of every fix and [(ms, channel)] of the world model's order as it
    grows.  The oracle does not depend on where the calls are cut (tests/test_fix_splits_cpu.py shows it byte for byte),
    so call() slices what the oracle says of any call [s, e) of a re-split timeline."""

    def __init__(self, oracle, calls):
        self.oracle = oracle
        touches, at = [], [0]

        class Clock:  # the receiver timestamps of one call: which millisecond the oracle reads is the one it is at
            def __init__(self, rx, off):
                self.rx, self.off = rx, off

            def __len__(self):
                return len(self.rx)

            def __getitem__(self, m):
                at[0] = self.off + m
                return self.rx[m]

        class Traced(oracle.ReceiverOracle):
            def _touch(self, ch):
                if ch not in self.order:
                    touches.append((at[0], ch))
                super()._touch(ch)

        rcv = Traced(len(calls[0][1]))
        recs, self.resets, self.rows, off = [], {}, {}, 0
        for rx, chans in calls:
            recs.append(rcv.call(chans, Clock(rx, off)))
            self.resets.update({off + m: v for m, v in rcv.resets.items()})
            self.rows.update({off + m: v for m, v in rcv.rows.items()})
            off += len(rx)
        self.records = np.concatenate(recs)
        self.touches = touches
        assert [ch for _, ch in touches] == rcv.order
        self.order, self.stopped, self.slide = rcv.order, rcv.stopped, rcv.slide

    def call(self, s, e):
        """(records, call-relative resets, order, stopped) of the oracle for the call [s, e), as ReceiverOracle.call,
        .resets, .order and .stopped would give them after it."""
        resets = {m - s: v for m, v in self.resets.items() if s <= m < e}
        order = [ch for m, ch in self.touches if m < e]
        stopped = bool(np.isin(self.records["status"][:e], [fx.FIX_RAISED, fx.FIX_STOPPED]).any())
        return self.records[s:e], resets, order, stopped

    def model(self, compute, calls):
        """device_passes on the oracle's rows over the calls of a split of this timeline (compute: the host core), the
        slide carried across: per call its result."""
        bounds, _ = call_starts(calls)
        carried, out = None, []
        for s, (rx, _) in zip(bounds, calls):
            rec, resets, _, _ = self.call(s, s + len(rx))
            rows = {m - s: r for m, r in self.rows.items() if s <= m < s + len(rx)}
            d = self.oracle.device_passes(compute, rec, rows, resets, carried)
            carried = d["slide"]
            out.append(d)
        return out


FIXING = (fx.FIX_SOLVED, fx.FIX_RAISED)


def edge_ms(calls, tl, misses=()):
    """The global milliseconds where k_fix_plan decides something in a timeline (calls, its OracleTimeline tl): every
    reset, drop and decoder raise; every millisecond whose (status, n_ready, rows) differ from the one before; the first
    fixing millisecond at and after each reset; the given misses of the model; the first and last millisecond."""
    from oracle import nav_oracle as nav

    bounds, total = call_starts(calls)
    out = {0, total - 1, *tl.resets, *misses}
    for b, (_, chans) in zip(bounds, calls):
        for events, drop in chans:
            if drop >= 0:
                out.add(b + drop)
            out.update(b + m for k, _, _, m in events if k == nav.KIND_RAISED)
    r = tl.records
    key = np.concatenate([r["status"][:, None], r["n_ready"][:, None], r["channel"]], axis=1)
    out.update(int(m) + 1 for m in np.flatnonzero((key[1:] != key[:-1]).any(axis=1)))
    fixing = np.flatnonzero(np.isin(r["status"], FIXING))
    for m in tl.resets:
        after = fixing[fixing >= m]
        out.update(int(a) for a in after[:2])
    return sorted(m for m in out if 0 <= m < total)


# in-call indices an edge millisecond is placed at: lanes 0, 1, 30 and 31 of the plan's chunk 0, lanes 0 and 1 of chunk 1,
# the last lane of chunk 1 and the first of chunk 2
EDGE_INDICES = (0, 1, 30, 31, 32, 33, 63, 64)
PLACEMENTS = EDGE_INDICES + ("last", "alone")


def _placement(e, p, start, total):
    """(cuts, span) that put millisecond e at placement p of its call (the original call starting at `start`), span
    the milliseconds no other cut may fall in; None where the call starts after e - p."""
    if p == "last":
        return ({e + 1} if e + 1 < total else set()), range(0)
    if p == "alone":
        return {e, e + 1} - {total}, range(0)
    if e - p < start:
        return None
    return {e - p}, range(e - p + 1, e + 1)


def edge_splits(calls, edges, placements=PLACEMENTS):
    """The cut sets that place every edge millisecond at every placement, packed: the edges of one cut set each sit at
    their own placement.  Returns [(placement, cuts, edges placed)]."""
    bounds, total = call_starts(calls)
    out = []
    for p in placements:
        runs = []  # [cuts, spans, edges]
        for e in edges:
            pl = _placement(e, p, max(b for b in bounds if b <= e), total)
            if pl is None:
                continue
            cuts, span = pl
            for run in runs:
                if not any(c in sp for c in cuts for sp in run[1]) and not any(c in span for c in run[0]):
                    run[0].update(cuts)
                    run[1].append(span)
                    run[2].append(e)
                    break
            else:
                runs.append([set(cuts), [span], [e]])
        out.extend((p, sorted(cuts), placed) for cuts, _, placed in runs)
    return out


def sweep_cuts(calls, offset, width=33):
    """Cuts every `width` milliseconds from `offset` on."""
    return list(range(offset, call_starts(calls)[1], width))


class ChainCheck:
    """One timeline on the device, call after call, against the receiver oracle and the model of the device's passes:
    status, ready count and rows exact; slides and round-0 pseudoranges within SLIDE_ULPS, clock bias within BIAS_S and
    position within POS_M (the MANY_* bounds in the least-squares mode from the first millisecond with five or more
    ready on); every fixing record is device_passes' on the device's own observations bit for bit; and after every call
    receiver_state() holds the model's carried slide exactly, the oracle's order and stop, and the model's running
    repair count."""

    def __init__(self, compute, solver="reference"):
        import fix_lsq_oracle as lo

        self.compute = compute
        self.lsq = solver == "least_squares"
        self.oracle = lo if self.lsq else fx
        self.carried, self.repaired, self.many = None, 0, False
        self.worst = [0.0, 0.0, 0.0]  # slide ulp, clock bias s, position m

    def __call__(self, want, resets, order, stopped, got, obs, state, what=""):
        """One call: the oracle's records, call-relative resets, order and stop after it (ReceiverOracle.call, .resets,
        .order, .stopped), and the device's records, observations and receiver_state().  Returns the model's result."""
        assert np.array_equal(got["status"], want["status"]), what
        assert np.array_equal(got["n_ready"], want["n_ready"]) and np.array_equal(got["channel"], want["channel"]), what
        fixing = np.flatnonzero(np.isin(want["status"], FIXING))
        solved = np.flatnonzero(want["status"] == fx.FIX_SOLVED)
        many = np.full(len(want), self.many)
        if self.lsq:
            five = fixing[want["n_ready"][fixing] > 4]
            if len(five):
                many[five[0]:] = self.many = True
        ulps = np.where(many, MANY_SLIDE_ULPS, SLIDE_ULPS)
        for k in ("slide_in", "slide_out"):
            d = np.abs(got[k][fixing] - want[k][fixing]) / (2.0 ** -52 * np.abs(want[k][fixing]))
            assert (d <= ulps[fixing]).all(), (what, k, fixing[d > ulps[fixing]][:5])
            self.worst[0] = max([self.worst[0], *d])
        if len(solved):
            tol = ulps[solved] * 2.0 ** -52 * np.abs(want["slide_in"][solved])
            d = np.abs(got["pseudorange"][solved] - want["pseudorange"][solved]).max(axis=1)
            assert (d <= tol).all(), (what, solved[d > tol][:5])
            db = np.abs(got["clock_bias"][solved] - want["clock_bias"][solved])
            dp = np.max([np.abs(got[k][solved] - want[k][solved]) for k in "xyz"], axis=0)
            assert (db <= np.where(many[solved], MANY_BIAS_S, BIAS_S)).all(), (what, db.max())
            assert (dp <= np.where(many[solved], MANY_POS_M, POS_M)).all(), (what, dp.max())
            self.worst[1:] = [max(self.worst[1], float(db.max())), max(self.worst[2], float(dp.max()))]
        assert np.isnan(got["x"][got["status"] != fx.FIX_SOLVED]).all(), what
        # the model of the passes, on the rows the device observed
        if self.lsq:
            rows = {m: ready_rows(obs, state["order"], m) for m in fixing}
            assert all(len(rows[m]) == want[m]["n_ready"] for m in fixing), what
        else:
            rows = {m: rows_at(obs, want[m]["channel"], m) for m in fixing if want[m]["n_ready"] == 4}
        model = self.oracle.device_passes(self.compute, want, rows, resets, self.carried)
        assert sorted(model["out"]) == list(fixing), what
        for m in fixing:
            p, g = model["out"][m], got[m]
            assert p["status"] == g["status"] and p["slide_in"] == g["slide_in"] and p["slide_out"] == g["slide_out"], \
                (what, m)
            if m in solved or self.lsq:
                assert p.tobytes()[:88] == g.tobytes()[:88], (what, m)
        self.carried = model["slide"]
        self.repaired += len(model["repaired"])
        assert state["slide"] == self.carried, (what, state["slide"], self.carried)
        assert state["order"] == order and state["stopped"] == stopped, (what, state, order, stopped)
        assert state["repaired"] == self.repaired, (what, state["repaired"], self.repaired)
        return model
