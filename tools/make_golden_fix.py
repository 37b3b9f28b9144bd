"""Generate tests/golden/fix.npz and tests/golden/fix_repair.npz from the LIVE reference: subframes written by
oracle/orbit_oracle.py's LNAV encoder go through the real NavigationMessageDecoder, and its EmitSubframeEvents drive one
real GpsWorldModel through scripted
timelines in the receiver's per-millisecond order (receiver.py:106-137): lost locks, one handle_prn_observed per tracked
satellite, the subframes channel by channel, then attempt_position_fix with the chunk's start time.  Run with the
reference checkout on the path:
    PYTHONPATH=<reference checkout> python tools/make_golden_fix.py [fix | fix_repair] [--out-dir DIR]

The matplotlib stubs and the recording parser are make_golden_orbit.py's.  satellite_ids_to_orbital_parameters is a
defaultdict whose order decides the fix's rows, so nothing here indexes it.  A decoder raise (event kind 3) is scripted:
the reference's step never returns from it, so from that millisecond on the receiver is stopped.

A receiver-clock jump (call, ms, J) is what a gap in the sample stream does: from that millisecond on, J is added to
every chunk start time and to every later trailing edge.  fix_repair.npz holds timelines with such jumps, where the fix
from a segment's reset slide and the serial chain reach different roots, so the device's chain check fails and its
serial repair runs (DESIGN.md §8c):
  gap_mid    the realistic shape, J = -0.2 s at ms 600 of call 0: the miss and the repair lie inside one segment
  gap_two    J = -0.2 s at ms 600 and at ms 1200 of call 0, in two segments: the repair walks across the reset at 900
  gap_back   J = -0.2 s at ms 600, then +0.2 s at ms 750 of the same segment: the chain changes root twice
  gap_first  J = -0.2 s at ms 301, right after the segment's first fix at 300: the miss comes at its second fix
  gap_carry  J = -0.2 s at ms 1300 of call 0, in the segment that runs into call 1: the repair runs to the end of call 0
             and call 1 continues from the repaired slide
  gap_five   the five shape with J = -0.15 s at ms 350: the repair stops at the LinAlgError at 400
  gap_raise  the raise shape with J = -0.2 s at ms 400: the decoder raise at 500 ends the repaired stretch
  singular   two channels of different PRNs with the same ephemeris on the same schedule: identical rows, numpy's
             "Singular matrix" at the first fix, and the receiver stops

Per timeline T the file holds T_calls, T_sv, T_events, T_words and T_drop in make_golden_orbit.py's layout (events may
also be of kind 3), and
  T_fix  float64 [sum of n_ms, 15]: call, ms, receiver_timestamp, status (0 none, 1 solution, 2 LinAlgError, 3 stopped),
         ready count, slide before attempt_position_fix, slide after it, clock bias, x, y, z, and the channels of the
         first four ready satellites in the world model's order (-1 where unused)
"""
import argparse
import copy
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden_orbit as mgo  # noqa: E402  (stubs matplotlib, records the parser's input)

from gypsum.gps_ca_prn_codes import GpsSatelliteId  # noqa: E402
from gypsum.world_model import GpsWorldModel  # noqa: E402

from oracle import nav_oracle as nav  # noqa: E402
from oracle import orbit_oracle as orb  # noqa: E402

GOLDEN = os.path.join(mgo.ROOT, "tests", "golden")
TOW0 = 50000


def stream(rng, sv, n, first_id=1, tow0=TOW0, seed=0):
    """n reference EmitSubframeEvents (with the bits the parser got) of consecutive subframes carrying one ephemeris."""
    eph = orb.realistic_ephemeris(rng, sv)
    return mgo.reference_events(orb.ephemeris_subframes(eph, n + 1, first_id=first_id, tow0=tow0, seed=seed))[:n]


def timelines():
    """name -> (calls n_ms, satellite ids, per channel: per call [(stream event or "raise", ms)], per call drops,
    streams[, receiver-clock jumps [(call, ms, J)]]).  Every subframe of one TOW count lands at the same millisecond on every channel, so the satellites' times
    of week stay within a few tens of milliseconds of each other, as real ones do."""
    rng = np.random.default_rng(2027)
    T = {}
    # four satellites: complete at ms 300, then resets at 900 and in the next call; every reset lands on all four
    # channels in one millisecond, and their trailing edges differ, so channel order decides the slide
    svs = (3, 8, 17, 29)
    st = [stream(rng, sv, 5, seed=c) for c, sv in enumerate(svs)]
    T["realistic"] = ([1500, 1200], svs, [[[(0, 100), (1, 200), (2, 300), (3, 900)], [(4, 400)]] for _ in svs],
                      [[-1] * 4, [-1] * 4], st)
    # three complete satellites and a fourth with two subframes: no fix
    svs = (5, 9, 14, 22)
    st = [stream(rng, sv, 3, seed=10 + c) for c, sv in enumerate(svs)]
    sched = [[[(0, 100), (1, 150), (2, 200)]] for _ in range(3)] + [[[(0, 100), (1, 150)]]]
    T["three"] = ([600], svs, sched, [[-1] * 4], st)
    # channel 3 completes first; the others complete at 6260, when its count is 5960; it passes 6000 at 6301 and
    # leaves the ready set, and the next subframe of all four at 6350 brings it back
    svs = (2, 11, 19, 31)
    st = [stream(rng, sv, 4, tow0=TOW0 + 1, seed=20 + c) for c, sv in enumerate(svs[:3])]
    st.append(stream(rng, svs[3], 5, seed=23))
    sched = [[[], [(0, 220), (1, 240), (2, 260), (3, 350)]] for _ in range(3)]
    sched.append([[(0, 100), (1, 200), (2, 300)], [(4, 350)]])
    T["gate"] = ([6000, 700], svs, sched, [[-1] * 4, [-1] * 4], st)
    # first touches out of channel order (channel 2 loses lock before any subframe, then 3, 1, 0 complete in that
    # order), a lost lock during a run of fixes (channel 1 at 800 of the second call), and its return in the third
    svs = (6, 13, 21, 27)
    st = [stream(rng, sv, 5, seed=30 + c) for c, sv in enumerate(svs)]
    st[2] = stream(rng, svs[2], 4, tow0=TOW0 + 1, seed=32)
    sched = [
        [[(0, 120), (1, 220), (2, 320)], [(3, 300)], [(4, 200)]],
        [[(0, 110), (1, 210), (2, 310)], [(3, 300)], [(4, 200)]],
        [[], [(0, 100), (1, 200), (2, 300)], [(3, 200)]],
        [[(0, 100), (1, 200), (2, 300)], [(3, 300)], [(4, 200)]],
    ]
    T["lost"] = ([500, 1000, 600], svs, sched, [[-1, -1, 50, -1], [-1, 800, -1, -1], [-1] * 4], st)
    # a fifth satellite becomes ready at 400: the reference raises LinAlgError there and its receiver stops
    svs = (1, 7, 12, 20, 25)
    st = [stream(rng, sv, 3, seed=40 + c) for c, sv in enumerate(svs)]
    sched = [[[(0, 100), (1, 200), (2, 300)], []] for _ in range(4)] + [[[(0, 100), (1, 200), (2, 400)], []]]
    T["five"] = ([700, 300], svs, sched, [[-1] * 5, [-1] * 5], st)
    # channel 1's decoder raises at 500 (event kind 3): the receiver stops there
    svs = (4, 10, 16, 30)
    st = [stream(rng, sv, 3, seed=50 + c) for c, sv in enumerate(svs)]
    sched = [[[(0, 100), (1, 200), (2, 300)], []] for _ in range(4)]
    sched[1][0].append(("raise", 500))
    T["raise"] = ([800, 200], svs, sched, [[-1] * 4, [-1] * 4], st)
    return T


def repair_timelines():
    """The timelines of fix_repair.npz (see the module docstring), from their own random draws."""
    rng = np.random.default_rng(2029)
    T = {}
    realistic = [[[(0, 100), (1, 200), (2, 300), (3, 900)], [(4, 400)]] for _ in range(4)]
    svs = (3, 8, 17, 29)
    st = [stream(rng, sv, 5, seed=60 + c) for c, sv in enumerate(svs)]
    # not every geometry misses at a given jump: gap_two, gap_back and gap_first have gap_mid's satellites
    for name, jumps in (("gap_mid", [(0, 600, -0.2)]), ("gap_two", [(0, 600, -0.2), (0, 1200, -0.2)]),
                        ("gap_back", [(0, 600, -0.2), (0, 750, 0.2)]), ("gap_first", [(0, 301, -0.2)])):
        T[name] = ([1500, 1200], svs, realistic, [[-1] * 4, [-1] * 4], st, jumps)
    svs = (2, 11, 19, 31)
    st = [stream(rng, sv, 5, seed=65 + c) for c, sv in enumerate(svs)]
    T["gap_carry"] = ([1500, 1200], svs, realistic, [[-1] * 4, [-1] * 4], st, [(0, 1300, -0.2)])
    svs = (1, 7, 12, 20, 25)
    st = [stream(rng, sv, 3, seed=70 + c) for c, sv in enumerate(svs)]
    sched = [[[(0, 100), (1, 200), (2, 300)], []] for _ in range(4)] + [[[(0, 100), (1, 200), (2, 400)], []]]
    T["gap_five"] = ([700, 300], svs, sched, [[-1] * 5, [-1] * 5], st, [(0, 350, -0.15)])
    svs = (4, 10, 16, 30)
    st = [stream(rng, sv, 3, seed=80 + c) for c, sv in enumerate(svs)]
    sched = [[[(0, 100), (1, 200), (2, 300)], []] for _ in range(4)]
    sched[1][0].append(("raise", 500))
    T["gap_raise"] = ([800, 200], svs, sched, [[-1] * 4, [-1] * 4], st, [(0, 400, -0.2)])
    # channel 3 carries channel 2's subframes (same ephemeris, same TOW counts) under another PRN
    svs = (3, 8, 17, 29)
    st = [stream(rng, sv, 3, seed=90 + c) for c, sv in enumerate(svs[:3])]
    st.append(st[2])
    sched = [[[(0, 100), (1, 200), (2, 300)], []] for _ in range(4)]
    T["singular"] = ([500, 200], svs, sched, [[-1] * 4, [-1] * 4], st)
    return T


def run(calls, svs, sched, drops, streams, jumps=()):
    wm = GpsWorldModel(2046)
    ids = [GpsSatelliteId(sv) for sv in svs]
    ev_rows, words, fix = [], [], []
    stopped = False
    t = 0.0

    def offset(c, m):  # the receiver-clock jumps up to (call c, ms m)
        return sum(j for jc, jm, j in jumps if (jc, jm) <= (c, m))

    for c, n_ms in enumerate(calls):
        by_ms = {}
        for ch in range(len(svs)):
            for k, m in sched[ch][c]:
                if k == "raise":
                    by_ms.setdefault(m, []).append((ch, None))
                    ev_rows.append([c, ch, m, nav.KIND_RAISED, 0.0, 0.0])
                    words.append((0,) * 10)
                    continue
                ev, given = streams[ch][k]
                ev = copy.copy(ev)  # the trailing edge in receiver time, a little earlier on each later channel
                ev.trailing_edge_receiver_timestamp = round(t + 0.001 * m - 0.0003 * ch + offset(c, m), 7)
                by_ms.setdefault(m, []).append((ch, ev))
                ev_rows.append([c, ch, m, 0, ev.receiver_timestamp, ev.trailing_edge_receiver_timestamp])
                words.append(orb.words_of(given))
        tracked = [True] * len(svs)
        for m in range(n_ms):
            t0, t1 = t + offset(c, m), t + 0.001 + offset(c, m)
            t += 0.001
            row = [c, m, t0, 3, 0, np.nan, np.nan, np.nan, np.nan, np.nan, np.nan, -1, -1, -1, -1]
            if any(ev is None and tracked[ch] for ch, ev in by_ms.get(m, ())):
                stopped = True
            if stopped:
                fix.append(row)
                continue
            for ch in range(len(svs)):
                if drops[c][ch] == m and tracked[ch]:
                    wm.handle_lost_satellite_lock(ids[ch], t0)
                    tracked[ch] = False
            for ch in range(len(svs)):
                if tracked[ch]:
                    wm.handle_prn_observed(ids[ch], 0, t0, t1)
            wm.handle_processed_1ms(t0)
            for ch in range(len(svs)):
                for ch2, ev in by_ms.get(m, ()):
                    if ch2 == ch and tracked[ch]:
                        wm.handle_subframe_emitted(ids[ch], ev)
            counts = wm.satellite_ids_to_prn_observations_since_last_handover_timestamp
            ready = [ids.index(sv) for sv, op in wm.satellite_ids_to_orbital_parameters.items()
                     if op.is_complete() and counts.get(sv, 6001) <= 6000]
            before = wm.receiver_clock_slide
            row[3], row[4] = 0, len(ready)
            row[11:11 + min(4, len(ready))] = ready[:4]
            try:
                sol = wm.attempt_position_fix(t0, None)
                if sol is not None:
                    row[3] = 1
                    row[7:11] = [float(sol.clock_bias), float(sol.receiver_pos.x), float(sol.receiver_pos.y),
                                 float(sol.receiver_pos.z)]
            except np.linalg.LinAlgError:
                row[3] = 2
                stopped = True
            row[5] = np.nan if before is None else float(before)
            row[6] = np.nan if wm.receiver_clock_slide is None else float(wm.receiver_clock_slide)
            fix.append(row)
    return {"calls": np.array(calls, dtype=np.int64), "sv": np.array(svs, dtype=np.int64),
            "events": np.array(ev_rows, dtype=np.float64).reshape(-1, 6), "words": np.array(words, dtype=np.int64),
            "drop": np.array(drops, dtype=np.int64), "fix": np.array(fix, dtype=np.float64)}


def record(path, tls):
    out = {}
    names = []
    for name, args in tls.items():
        names.append(name)
        for k, v in run(*args).items():
            out[f"{name}_{k}"] = v
        f = out[f"{name}_fix"]
        print(f"{name:10s} ms {len(f)} status counts {np.bincount(f[:, 3].astype(int), minlength=4)}")
    out["timelines"] = np.array(names)
    np.savez_compressed(path, **out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("which", nargs="*", choices=["fix", "fix_repair"], help="the files to record (default: both)")
    ap.add_argument("--out-dir", default=GOLDEN)
    args = ap.parse_args()
    for which in args.which or ["fix", "fix_repair"]:
        record(os.path.join(args.out_dir, f"{which}.npz"), timelines() if which == "fix" else repair_timelines())


if __name__ == "__main__":
    main()
