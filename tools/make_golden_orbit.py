"""Generate tests/golden/orbit.npz from the LIVE reference: subframes written by oracle/orbit_oracle.py's LNAV encoder go
through the real NavigationMessageDecoder (which parses them with the real NavigationMessageSubframeParser), and the
EmitSubframeEvents it gives drive the real GpsWorldModel through scripted timelines, one handle_prn_observed per
millisecond per tracked satellite and handle_lost_satellite_lock where a timeline drops one, in the receiver's order
(receiver.py:106-137).  Run with the reference checkout on the path:
    PYTHONPATH=<reference checkout> python tools/make_golden_orbit.py

world_model imports tracker_visualizer, which imports matplotlib; stub modules stand in for it (nothing here plots).

Per timeline T the file holds
  T_calls      int64 [n_calls]: n_ms of each call; T_sv int64 [n_ch]: satellite ids
  T_events     float64 [n, 6]: call, channel, ms, kind (0), receiver_timestamp, trailing_edge_receiver_timestamp
  T_words      int64 [n, 10]: the 300 bits the reference's parser was given, 30 per word, first bit most significant
  T_fields     float64 [n, 18]: the reference parser's fields in gb200_subframe_fields order (subframe id, TOW seconds,
               ints[2], bits[4], values[10]; bit lists packed first bit first)
  T_drop       int64 [n_calls, n_ch]: drop millisecond (-1 = none)
  T_obs        float64 [m, 9]: call, channel, ms, tow, x, y, z, prn count (-1 = not counting), flags -- at sampled ms
  T_params     float64 [n_calls, n_ch, 26] and T_mask int64 [n_calls, n_ch]: the parameter set after each call
"""
import logging
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

for name in ("matplotlib", "matplotlib.pyplot", "matplotlib.axes"):
    sys.modules.setdefault(name, types.ModuleType(name))
sys.modules["matplotlib.axes"].Axes = object

import gypsum.navigation_message_decoder as nmd  # noqa: E402
import gypsum.navigation_message_parser as nmp  # noqa: E402
from gypsum.gps_ca_prn_codes import GpsSatelliteId  # noqa: E402
from gypsum.navigation_bit_intergrator import EmitNavigationBitEvent  # noqa: E402
from gypsum.tracker import BitValue  # noqa: E402
from gypsum.world_model import GpsWorldModel, OrbitalParameterType  # noqa: E402

from oracle import nav_oracle as nav  # noqa: E402
from oracle import orbit_oracle as orb  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "orbit.npz")
logging.disable(logging.CRITICAL)

_given: list = []


class _RecordingParser(nmp.NavigationMessageSubframeParser):
    def __init__(self, bits):
        _given.append(list(bits))
        super().__init__(bits)


nmd.NavigationMessageSubframeParser = _RecordingParser


def reference_events(subframes):
    """The EmitSubframeEvents of the real decoder on the concatenated subframes, with the bits its parser got."""
    bits = [b for sf in subframes for b in sf]
    t0, t1 = nav.bit_times(len(bits))
    dec = nmd.NavigationMessageDecoder()
    out = []
    for b, a, c in zip(bits, t0, t1):
        n = len(_given)
        evs = dec.process_bit_from_satellite(EmitNavigationBitEvent(float(a), float(c), BitValue.ONE if b else BitValue.ZERO))
        given = iter(_given[n:])  # one parser per subframe drained by this bit, in order (the streams parse cleanly)
        for ev in evs:
            if isinstance(ev, nmd.EmitSubframeEvent):
                out.append((ev, next(given)))
    return out


def _pack(bits):
    return int("".join(str(int(b)) for b in bits), 2) if bits else 0


def fields_row(sf) -> list:
    """The reference's subframe dataclass -> gb200_subframe_fields order (id, tow filled by the caller)."""
    i = sf.subframe_id.value
    if i == 1:
        ints, bl = [sf.week_num_mod_1024_bits, sf.l2_p_data_flag], [sf.ca_or_p_on_l2, sf.ura_index, sf.sv_health,
                                                                     sf.issue_of_data_clock]
        vals = [sf.estimated_group_delay_differential, sf.t_oc, sf.a_f2, sf.a_f1, sf.a_f0]
    elif i == 2:
        ints, bl = [int(sf.fit_interval_flag)], [sf.issue_of_data_ephemeris, sf.age_of_data_offset]
        vals = [sf.correction_to_orbital_radius_sin, sf.mean_motion_difference_from_computed_value,
                sf.mean_anomaly_at_reference_time, sf.correction_to_latitude_cos, sf.eccentricity,
                sf.correction_to_latitude_sin, sf.sqrt_semi_major_axis, sf.reference_time_ephemeris]
    elif i == 3:
        ints, bl = [], [sf.issue_of_data_ephemeris]
        vals = [sf.correction_to_inclination_angle_cos, sf.longitude_of_ascending_node,
                sf.correction_to_inclination_angle_sin, sf.inclination_angle, sf.correction_to_orbital_radius_cos,
                sf.argument_of_perigee, sf.rate_of_right_ascension, sf.rate_of_inclination_angle]
    elif i == 4:
        ints, bl, vals = [sf.data_id, sf.page_id], [], []
    else:
        ints, bl = [], [sf.data_id, sf.satellite_id, sf.sv_health]
        vals = [sf.eccentricity, sf.time_of_ephemeris, sf.delta_inclination_angle, sf.right_ascension_rate,
                sf.semi_major_axis_sqrt, sf.longitude_of_ascension_mode, sf.argument_of_perigree,
                sf.mean_anomaly_at_reference_time, sf.a_f0, sf.a_f1]
    ints = list(ints) + [0] * (2 - len(ints))
    packed = [_pack(b) for b in bl] + [0] * (4 - len(bl))
    return ints + packed + [float(v) for v in vals] + [0.0] * (10 - len(vals))


def extreme_ephemeris(sign: int) -> dict:
    """Every signed field at its most negative (sign < 0) or most positive value, unsigned ones at 0 / all ones."""
    widths = {"tgd": 8, "af2": 8, "af1": 16, "af0": 22, "crs": 16, "dn": 16, "m0": 32, "cuc": 16, "cus": 16, "cic": 16,
              "omega0": 32, "cis": 16, "i0": 32, "crc": 16, "omega": 32, "omegadot": 24, "idot": 14}
    eph = {k: (-(1 << (w - 1)) if sign < 0 else (1 << (w - 1)) - 1) for k, w in widths.items()}
    eph.update(wn=1023 if sign > 0 else 0, iodc=1023 if sign > 0 else 0, iode=255 if sign > 0 else 0, ura=15, health=63,
               l2_codes=3, l2p=1, fit=1, aodo=31, toc=65535 if sign > 0 else 0, toe=37799 if sign > 0 else 0,
               e=(1 << 32) - 1 if sign > 0 else 0, sqrta=round(5153.6 * 2 ** 19), data_id=1, page_id=63 if sign > 0 else 0,
               sv_id=63 if sign > 0 else 1)
    if sign > 0:
        eph["e"] = round(0.03 * 2 ** 33)  # a bound orbit; the extreme eccentricity is in the parse-only cases
    return eph


def timelines():
    """name -> (calls n_ms, per channel: (sv, subframes, per call [(stream event index, ms)], per call drop ms))."""
    rng = np.random.default_rng(2026)
    T = {}
    # several satellites with realistic ephemerides: subframes 1-5 then 1-3 again; the second call runs 7 s past the
    # last HOW, so the 6000-count gate is crossed
    chans = []
    for c, sv in enumerate((3, 17, 29)):
        eph = orb.realistic_ephemeris(rng, sv)
        sfs = orb.ephemeris_subframes(eph, 9, first_id=1, tow0=40000 + 7 * c, seed=c)
        sched = [[(k, 150 + 300 * k + 37 * c) for k in range(8)], []]
        chans.append((sv, sfs, sched, [-1, -1]))
    T["realistic"] = ([3000, 7200], chans)
    # extreme two's-complement values, both signs
    chans = []
    for c, sign in enumerate((-1, 1)):
        sfs = orb.ephemeris_subframes(extreme_ephemeris(sign), 7, first_id=1, tow0=1000 + c, seed=10 + c)
        chans.append((5 + c, sfs, [[(k, 100 + 200 * k) for k in range(6)]], [-1]))
    T["extreme"] = ([1600], chans)
    # toe at both week edges: tk wraps up and down
    chans = []
    for c, (toe, tow0) in enumerate(((37799, 2), (0, 100790))):
        eph = orb.realistic_ephemeris(rng, 9 + c)
        eph["toe"] = eph["toc"] = toe
        sfs = orb.ephemeris_subframes(eph, 5, first_id=1, tow0=tow0, seed=20 + c)
        chans.append((9 + c, sfs, [[(k, 60 + 90 * k) for k in range(4)], [(4, 500)]], [-1, -1]))
    T["week_edge"] = ([900, 1400], chans)
    # subframes in order 4, 5, 1, 2, 3: complete only after the third
    eph = orb.realistic_ephemeris(rng, 21)
    sfs = orb.ephemeris_subframes(eph, 6, first_id=4, tow0=7000, seed=30)
    T["order"] = ([2000], [(21, sfs, [[(k, 100 + 250 * k) for k in range(5)]], [-1])])
    # a second subframe 1 with another IODC and clock: the clock terms change, the ephemeris stays (no IODE / IODC check)
    eph = orb.realistic_ephemeris(rng, 30)
    eph2 = dict(eph, iodc=(eph["iodc"] + 5) % 1024, af0=eph["af0"] + 12345, af1=eph["af1"] - 7, toc=eph["toc"] + 225)
    sfs = orb.ephemeris_subframes(eph, 3, first_id=1, tow0=9000, seed=40)
    second = orb.encode_subframe(1, 9003, eph2, (sfs[-1][-2], sfs[-1][-1]), np.random.default_rng(41))
    tail = orb.ephemeris_subframes(eph2, 1, first_id=2, tow0=9004, seed=42)
    T["mixing"] = ([2400], [(30, sfs + [second] + tail, [[(0, 200), (1, 500), (2, 800), (3, 1500)]], [-1])])
    # lock lost after a complete set, then new subframes in the next call
    eph = orb.realistic_ephemeris(rng, 12)
    sfs = orb.ephemeris_subframes(eph, 7, first_id=1, tow0=3000, seed=50)
    T["lost"] = ([1500, 1800], [(12, sfs, [[(0, 100), (1, 300), (2, 500), (3, 1200)], [(5, 700), (6, 900)]], [1000, -1])])
    return T


def record_ms(n_ms, marks):
    keep = set(range(0, n_ms, 13)) | {n_ms - 1}
    for m in marks:
        keep |= {m - 1, m, m + 1}
    return sorted(k for k in keep if 0 <= k < n_ms)


def run(calls, chans):
    wm = GpsWorldModel(2046)
    svs = [GpsSatelliteId(sv) for sv, *_ in chans]
    streams = [reference_events(sfs) for _, sfs, _, _ in chans]
    ev_rows, words, fields, obs = [], [], [], []
    drops = np.array([[ch[3][c] for ch in chans] for c in range(len(calls))], dtype=np.int64)
    params = np.zeros((len(calls), len(chans), 26))
    masks = np.zeros((len(calls), len(chans)), dtype=np.int64)
    t = 0.0
    for c, n_ms in enumerate(calls):
        by_ms = {}
        for ch, (_, _, sched, _) in enumerate(chans):
            for k, m in sched[c]:
                ev, given = streams[ch][k]
                by_ms.setdefault(m, []).append((ch, ev))
                ev_rows.append([c, ch, m, 0, ev.receiver_timestamp, ev.trailing_edge_receiver_timestamp])
                words.append(orb.words_of(given))
                fields.append([ev.subframe.subframe_id.value, ev.handover_word.time_of_week_in_seconds]
                              + fields_row(ev.subframe))
        tracked = [True] * len(chans)
        marks = [m for ms in by_ms for m in [ms]] + [d for d in drops[c] if d >= 0]
        keep = set(record_ms(n_ms, marks))
        for m in range(n_ms):
            t0, t1 = t, t + 0.001
            t = t1
            for ch in range(len(chans)):
                if drops[c, ch] == m and tracked[ch]:
                    wm.handle_lost_satellite_lock(svs[ch], t0)
                    tracked[ch] = False
            for ch in range(len(chans)):
                if tracked[ch]:
                    wm.handle_prn_observed(svs[ch], 0, t0, t1)
            for ch, ev in by_ms.get(m, ()):
                if tracked[ch]:
                    wm.handle_subframe_emitted(svs[ch], ev)
            if m in keep:
                for ch, sv in enumerate(svs):
                    op = wm.satellite_ids_to_orbital_parameters[sv]
                    counting = sv in wm.satellite_ids_to_prn_observations_since_last_handover_timestamp
                    count = wm.satellite_ids_to_prn_observations_since_last_handover_timestamp[sv] if counting else -1
                    timing = wm._can_interrogate_precise_timings_for_satellite(sv)
                    complete = op.is_complete()
                    flags = (orb.OBS_COUNTING if counting else 0) | (orb.OBS_TIMING if timing else 0) | \
                        (orb.OBS_COMPLETE if complete else 0) | (orb.OBS_FIX_GATE if counting and count <= 6000 else 0)
                    tow = x = y = z = np.nan
                    if timing:
                        tow = wm._gps_observed_system_time_of_week_for_satellite(sv, t0, None)
                        if complete:
                            p = wm._get_satellite_position_at_time_of_week(sv, tow)
                            x, y, z = p.x, p.y, p.z
                    obs.append([c, ch, m, tow, x, y, z, count, flags])
        for ch, sv in enumerate(svs):
            op = wm.satellite_ids_to_orbital_parameters[sv]
            for k, ptype in enumerate(OrbitalParameterType):
                v = op.get_parameter(ptype)
                if v is not None:
                    params[c, ch, k] = float(v)
                    masks[c, ch] |= 1 << k
    return {"calls": np.array(calls, dtype=np.int64), "sv": np.array([ch[0] for ch in chans], dtype=np.int64),
            "events": np.array(ev_rows, dtype=np.float64).reshape(-1, 6), "words": np.array(words, dtype=np.int64),
            "fields": np.array(fields, dtype=np.float64), "drop": drops,
            "obs": np.array(obs, dtype=np.float64).reshape(-1, 9), "params": params, "mask": masks}


def main():
    out = {}
    names = []
    for name, (calls, chans) in timelines().items():
        names.append(name)
        for k, v in run(calls, chans).items():
            out[f"{name}_{k}"] = v
        o = out[f"{name}_obs"]
        print(f"{name:10s} calls {calls} events {len(out[f'{name}_events'])} rows {len(o)} "
              f"timing {int((o[:, 8].astype(int) & 1).sum())} complete {int((o[:, 8].astype(int) & 2).sum() // 2)}")
    out["timelines"] = np.array(names)
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
