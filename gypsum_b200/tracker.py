"""Drop-in for reference gypsum/tracker.py: GpsSatelliteTracker, GpsSatelliteTrackingParameters and the
pseudosymbol types, same names / fields / exception (tracker.py:33-110, :117-155, :206-389).

`GpsSatelliteTracker.process_samples(chunk)` keeps the reference's one-millisecond-per-call contract; the trackers of
one engine and code-phase mode share a channel pool, so a chunk handed to N trackers in turn costs one GPU round trip,
not N (`_ChannelPool`).  `TrackerBank` is the throughput interface: many channels x many milliseconds in one persistent-kernel
launch.  The correlators, loop filters, lock heuristics and the 6-second constellation check
all run on the device (gypsum_b200/csrc/tracker.cu, tracker_core.cuh); this module only mirrors the host-visible
state and histories the rest of gypsum reads.
"""
from __future__ import annotations

import collections
import math
from dataclasses import dataclass
from enum import Enum, auto

import numpy as np

from gypsum_b200 import _native
from gypsum_b200.constants import ONE_MILLISECOND
from gypsum_b200.utils import POOL, chips_of_satellite


class LostSatelliteLockError(Exception):  # tracker.py:33
    pass


class BitValue(Enum):  # tracker.py:48-84
    UNKNOWN = auto()
    ZERO = auto()
    ONE = auto()

    @classmethod
    def from_val(cls, val: int) -> "BitValue":
        return {0: BitValue.ZERO, 1: BitValue.ONE}[val]

    def as_val(self) -> int:
        if self == BitValue.UNKNOWN:
            raise ValueError("Cannot convert an unknown bit value into an integer")
        return {BitValue.ZERO: 0, BitValue.ONE: 1}[self]

    def inverted(self) -> "BitValue":
        if self == BitValue.UNKNOWN:
            raise ValueError("Cannot invert an unknown bit value")
        return {BitValue.ZERO: BitValue.ONE, BitValue.ONE: BitValue.ZERO}[self]

    def __eq__(self, other) -> bool:
        return isinstance(other, BitValue) and self.value == other.value

    def __hash__(self) -> int:
        return hash(self.value)


class NavigationBitPseudosymbol(Enum):  # tracker.py:87-102
    MINUS_ONE = auto()
    ONE = auto()

    @classmethod
    def from_val(cls, val: int) -> "NavigationBitPseudosymbol":
        return {-1: NavigationBitPseudosymbol.MINUS_ONE, 1: NavigationBitPseudosymbol.ONE}[val]

    def as_val(self) -> int:
        return {NavigationBitPseudosymbol.MINUS_ONE: -1, NavigationBitPseudosymbol.ONE: 1}[self]


@dataclass
class EmittedPseudosymbol:  # tracker.py:105-110
    start_of_pseudosymbol: float
    end_of_pseudosymbol: float
    pseudosymbol: NavigationBitPseudosymbol
    cursor_at_emit_time: int


_TRACKER_ITERATIONS_PER_SECOND = 1000  # tracker.py:114


@dataclass
class GpsSatelliteTrackingParameters:
    """tracker.py:117-155: current loop state + the rolling histories the visualiser reads.  `is_locked` reports the
    decision the device made for the most recent millisecond (tracker.py:157-203 runs on the GPU)."""

    satellite: object
    current_doppler_shift: float
    current_carrier_wave_phase_shift: float
    current_prn_code_phase_shift: int
    doppler_shifts: list
    carrier_wave_phases: collections.deque = None
    carrier_wave_phase_errors: collections.deque = None
    correlation_peaks_rolling_buffer: collections.deque = None
    correlation_peak_angles: collections.deque = None
    non_coherent_correlation_profiles: collections.deque = None
    discriminators: collections.deque = None

    def __post_init__(self) -> None:
        for field in (self.correlation_peaks_rolling_buffer, self.correlation_peak_angles, self.carrier_wave_phases,
                      self.carrier_wave_phase_errors):
            if field is not None:
                raise RuntimeError("This field is not intended to be initialized at a call site.")  # tracker.py:145
        n = _TRACKER_ITERATIONS_PER_SECOND
        self.correlation_peaks_rolling_buffer = collections.deque(maxlen=n)
        self.correlation_peak_strengths_rolling_buffer = collections.deque(maxlen=n)
        self.correlation_peak_angles = collections.deque(maxlen=n)
        self.carrier_wave_phases = collections.deque(maxlen=n * 5)
        self.carrier_wave_phase_errors = collections.deque(maxlen=n * 5)
        self.non_coherent_correlation_profiles = collections.deque(maxlen=n // 4)
        self.discriminators = collections.deque(maxlen=n)
        self._last_is_locked = False

    def is_locked(self) -> bool:
        return self._last_is_locked


# A record travels through this module as the plain tuple `np.void.item()` gives (one conversion per record instead of one
# numpy scalar per field: with 32 trackers asked once per millisecond the host glue is what limits the drop-in path).
_F = {name: i for i, name in enumerate(_native.TRACK_DTYPE.names)}
(_DOPPLER, _CPHASE, _ERROR, _DISC, _PHASE_ACC, _DOPPLER_HIST, _CPHASE_HIST, _PEAK_RE, _PEAK_IM, _STRENGTH, _CODE_PHASE, _SYMBOL,
 _LOCKED, _LOST) = (_F[k] for k in ("doppler", "carrier_phase", "error", "disc", "phase_acc", "doppler_hist", "carrier_phase_hist",
                                    "peak_re", "peak_im", "strength", "code_phase", "symbol", "locked", "lost"))


def _apply_record(params: GpsSatelliteTrackingParameters, rec: tuple, profile=None) -> None:
    """What tracker.py:299-387 appends / assigns during one process_samples call."""
    peak = complex(rec[_PEAK_RE], rec[_PEAK_IM])
    params.current_prn_code_phase_shift = rec[_CODE_PHASE]
    params.discriminators.append(rec[_DISC])
    params.discriminators.append(0)  # tracker.py:305 self.accumulator
    if profile is not None:
        params.non_coherent_correlation_profiles.append(profile)
    params.correlation_peaks_rolling_buffer.append(peak)
    params.correlation_peak_strengths_rolling_buffer.append(rec[_STRENGTH])
    params.carrier_wave_phase_errors.append(rec[_ERROR])
    params.correlation_peak_angles.append(math.atan2(peak.imag, peak.real))  # np.angle
    # tracker.py:352-353 append the loop state to the histories BEFORE the 6-second constellation adjustment of :370-387;
    # current_* end up with the adjusted values
    params.doppler_shifts.append(rec[_DOPPLER_HIST])
    params.carrier_wave_phases.append(rec[_CPHASE_HIST])
    params.current_carrier_wave_phase_shift = rec[_CPHASE]
    params.current_doppler_shift = rec[_DOPPLER]
    params._last_is_locked = bool(rec[_LOCKED])


def _pseudosymbol(rec, start_time: float, end_time: float, wrap: int = _native.REFERENCE_CODE_WRAP) -> EmittedPseudosymbol:
    """tracker.py:319-325: the chunk's times delayed by code_phase / wrap ms (track_symbol_delay in tracker_core.cuh)."""
    if not isinstance(rec, tuple):
        rec = rec.item()
    delay = (rec[_CODE_PHASE] / wrap) * ONE_MILLISECOND
    return EmittedPseudosymbol(
        start_of_pseudosymbol=start_time + delay, end_of_pseudosymbol=end_time + delay,
        pseudosymbol=NavigationBitPseudosymbol.from_val(rec[_SYMBOL]), cursor_at_emit_time=0)


def _chunk_key(chunk) -> tuple:
    ring = getattr(chunk, "device_ring", None)
    if ring is not None:
        return ("ring", id(ring), int(chunk.ring_index))
    return (id(chunk.samples), float(chunk.start_time))


class _ChannelPool:
    """Every GpsSatelliteTracker of one engine and code-phase mode is a channel slot of ONE native pool
    (gb200_tracker_create_pool).

    The receiver hands the same chunk to every tracked satellite in turn (receiver.py:103-106, :237-257).  When the first
    tracker is asked about a chunk, all channels of the pool advance through it in one launch (one upload, one kernel, one
    read-back instead of one of each per satellite); the others find their millisecond already computed.  The kernel keeps
    each channel's previous state, so a channel that is then asked about a DIFFERENT chunk, or whose loop state the host
    edited in between, takes the step back (gb200_tracker_undo_channel) and is recomputed -- results never depend on the
    batching."""

    CAPACITY = 64  # 32 GPS PRNs; room for re-acquisitions that overlap a dropped tracker's lifetime

    def __init__(self, ent, code_phase: str, samples_per_ms: int):
        self.engine = ent["engine"]
        self.native = _native.Tracker.pool(self.engine, self.CAPACITY)
        self.code_wrap = _native.REFERENCE_CODE_WRAP  # what the pseudosymbol delay divides by
        if code_phase != "reference":
            self.native.set_code_phase_mode(code_phase)
            self.code_wrap = samples_per_ms
        self.free = list(range(self.CAPACITY - 1, -1, -1))
        self.members: dict = {}   # channel -> weakref to its GpsSatelliteTracker
        self.ahead: dict = {}     # channel -> (chunk key, record, profile or None): computed, not yet asked for
        self.stopped: set = set()  # channels whose device state carries `lost` (cleared by the next set_state)
        self.last: dict = {}      # channel -> key of the chunk it was last asked about

    def join(self, tracker, prn_idx: int, doppler: float, carrier_phase: float, code_phase: int) -> int:
        import weakref

        if not self.free:
            raise RuntimeError(f"more than {self.CAPACITY} live trackers on one engine")
        ch = self.free.pop()
        self.native.reset_channel(ch, prn_idx, doppler, carrier_phase, code_phase)
        self.members[ch] = weakref.ref(tracker)
        self.last.pop(ch, None)
        return ch

    def leave(self, ch: int) -> None:
        if self.members.pop(ch, None) is not None:
            self.ahead.pop(ch, None)
            self.stopped.discard(ch)
            self.free.append(ch)

    def drop_ahead(self, ch: int) -> None:
        """The channel was advanced through a chunk nobody asked it about: put its previous state back."""
        if self.ahead.pop(ch, None) is not None:
            self.native.undo_channel(ch)

    def _load(self, chunk, key) -> None:
        ring = getattr(chunk, "device_ring", None)
        if ring is not None and ring.holds_newest(chunk):
            ring.native.bind_newest(1)  # the millisecond is already on the device (one upload for detector and trackers)
        elif self.engine.iq_tag != key:
            self.engine.upload_iq(chunk.samples, tag=key)

    def step(self, ch: int, chunk, want_profile: bool):
        key = _chunk_key(chunk)
        got = self.ahead.pop(ch, None)
        self.last[ch] = key
        if got is not None:
            if got[0] == key and (got[2] is not None or not want_profile):
                return got[1], got[2]
            self.native.undo_channel(ch)
        # every other channel that has not seen this chunk and has nothing computed ahead will be asked about it next
        sel, profs = [ch], want_profile
        for c, ref in list(self.members.items()):
            trk = ref()
            if trk is None:
                self.leave(c)
            elif (c != ch and c not in self.ahead and c not in self.stopped and self.last.get(c) != key
                  and not trk._host_edited()):
                sel.append(c)
                profs = profs or trk.keep_correlation_profiles
        self._load(chunk, key)
        got = self.native.process_channels(sel, 1, [float(chunk.start_time)], want_profiles=profs, keep_undo=True)
        recs, prof = got if profs else (got, None)
        rows = recs[:, 0].tolist()  # one tuple of Python scalars per channel
        for i, c in enumerate(sel[1:], start=1):
            self.ahead[c] = (key, rows[i], None if prof is None else prof[i, 0])
        return rows[0], (None if prof is None else prof[0, 0])


def _pool_of(ent, code_phase: str, samples_per_ms: int) -> _ChannelPool:
    if code_phase not in _native.CODE_PHASE_MODES:
        raise ValueError(f"code-phase mode must be one of {sorted(_native.CODE_PHASE_MODES)}, not {code_phase!r}")
    pools = ent.setdefault("tracker_pools", {})
    if code_phase not in pools:
        pools[code_phase] = _ChannelPool(ent, code_phase, samples_per_ms)
    return pools[code_phase]


class GpsSatelliteTracker:
    """tracker.py:206-389.  code_phase: "reference" (the default) counts code phase as the reference does, wrapping at
    2046 at every rate; "samples" wraps at the stream's samples per millisecond, so that a satellite acquired at any code
    phase stays tracked above 2.046 Msps (_native.Tracker.set_code_phase_mode).  The trackers of each mode batch within
    their own pool: a chunk handed to trackers of both modes costs two launches."""

    def __init__(self, tracking_params: GpsSatelliteTrackingParameters, stream_attributes,
                 keep_correlation_profiles: bool = True, code_phase: str = "reference") -> None:
        self.tracking_params = tracking_params
        self.stream_attributes = stream_attributes
        self.keep_correlation_profiles = keep_correlation_profiles
        self.accumulator = 0
        self.phase = tracking_params.current_prn_code_phase_shift  # tracker.py:224
        fs, n = int(stream_attributes.samples_per_second), int(stream_attributes.samples_per_prn_transmission)
        self._ent = POOL.get(fs, n)
        self._eng = self._ent["engine"]
        idx = POOL.replica_index(self._ent, chips_of_satellite(tracking_params.satellite, n))
        self._pool = _pool_of(self._ent, code_phase, n)
        self._channel = self._pool.join(self, idx, tracking_params.current_doppler_shift,
                                        tracking_params.current_carrier_wave_phase_shift,
                                        tracking_params.current_prn_code_phase_shift)
        self._device_view = self._host_view()

    def close(self) -> None:
        if getattr(self, "_channel", None) is not None:
            self._pool.leave(self._channel)
            self._channel = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _host_view(self) -> tuple:
        p = self.tracking_params
        return (float(p.current_doppler_shift), float(p.current_carrier_wave_phase_shift),
                int(p.current_prn_code_phase_shift), float(self.phase))

    def _host_edited(self) -> bool:
        return self._host_view() != self._device_view

    def _push_host_edits(self) -> None:
        """If a caller changed tracking_params.current_* (or self.phase) since the last call, the device follows.  A
        channel that raised LostSatelliteLockError keeps working when asked again, like the reference object: its device
        flag is cleared by the same call."""
        now = self._host_view()
        stopped = self._channel in self._pool.stopped
        if now != self._device_view or stopped:
            self._pool.drop_ahead(self._channel)  # anything computed ahead used the old state
            self._pool.native.set_state(self._channel, now[0], now[1], now[3], now[2])
            self._pool.stopped.discard(self._channel)
            self._device_view = now

    def process_samples(self, receiver_samples_chunk) -> EmittedPseudosymbol:
        """tracker.py:331-389."""
        self._push_host_edits()
        rec, prof = self._pool.step(self._channel, receiver_samples_chunk, self.keep_correlation_profiles)
        if rec[_LOST] >= 2:  # cannot happen through this class (the flag is cleared above); never hand out a placeholder
            raise LostSatelliteLockError()
        if rec[_SYMBOL] == 0:
            raise KeyError(0)  # tracker.py:317: NavigationBitPseudosymbol.from_val has no entry for 0
        keep = self.keep_correlation_profiles and prof is not None
        _apply_record(self.tracking_params, rec, prof.astype(np.float64) if keep else None)
        self.phase = rec[_PHASE_ACC]
        self._device_view = self._host_view()
        if rec[_LOST]:
            self._pool.stopped.add(self._channel)
            raise LostSatelliteLockError()  # tracker.py:378
        return _pseudosymbol(rec, receiver_samples_chunk.start_time, receiver_samples_chunk.end_time, self._pool.code_wrap)


class TrackerBank:
    """Throughput interface: `n` channels advance through a block of milliseconds in one persistent-kernel launch
    (BASELINE config 4).  channels: iterable of (satellite, doppler_hz, carrier_phase_rad, code_phase_samples).
    fix_solver: what position_fixes does with five or more ready satellites, "reference" (raise and stop, as the
    reference receiver does) or "least_squares" (solve over all of them).  code_phase: "reference" wraps the DLL at 2046
    at every rate, as the reference does; "samples" wraps it at samples_per_ms, keeping every acquired code phase and
    stamping each pseudosymbol with its true delay (_native.Tracker.set_code_phase_mode)."""

    def __init__(self, channels, stream_attributes, device: int = 0, fix_solver: str = "reference",
                 code_phase: str = "reference"):
        fs, n = int(stream_attributes.samples_per_second), int(stream_attributes.samples_per_prn_transmission)
        self.samples_per_ms = n
        self._ent = POOL.get(fs, n, device)
        self.engine = self._ent["engine"]
        channels = list(channels)
        idx = [POOL.replica_index(self._ent, chips_of_satellite(c[0], n)) for c in channels]
        self.native = _native.Tracker(self.engine, idx, [c[1] for c in channels], [c[2] for c in channels],
                                      [c[3] for c in channels])
        self.native.set_fix_solver(fix_solver)
        self.native.set_code_phase_mode(code_phase)
        self.n_channels = len(channels)

    def process(self, samples: np.ndarray, start_times, want_profiles: bool = False):
        """samples: complex64[n_ms * N]; returns TRACK_DTYPE records [n_channels, n_ms] (and profiles)."""
        x = np.ascontiguousarray(samples, dtype=np.complex64)
        n_ms = x.size // self.samples_per_ms
        self.engine.upload_iq(x[: n_ms * self.samples_per_ms])
        return self.native.process(n_ms, start_times, want_profiles)

    def process_ring(self, ring, n_ms: int, start_times, want_profiles: bool = False):
        """The newest n_ms milliseconds of a DeviceSampleRing, in place (no upload)."""
        ring.native.bind_newest(n_ms)
        return self.native.process(n_ms, start_times, want_profiles)

    def integrate_bits(self, start_times, end_times) -> list:
        """Navigation bits of every channel from the records the last `process` call left on the device
        (navigation_bit_intergrator.py:278-288; one integrator per channel, persistent across calls).  Returns one
        _native.BIT_DTYPE array per channel: timestamps of the bit's edges, value 1 / 0 / -1 (unknown)."""
        return self.native.integrate_bits(len(start_times), start_times, end_times)

    def decode_subframes(self) -> list:
        """Navigation-message subframes of every channel from the bit events the last `integrate_bits` call left on the
        device (navigation_message_decoder.py:173-196; one decoder per channel, persistent across calls).  Returns one
        _native.SUBFRAME_DTYPE array per channel; _native.subframe_bits gives an event's 300 upright bits."""
        self._last_subframes = self.native.decode_subframes()
        return self._last_subframes

    def parse_subframes(self) -> list:
        """The subframes the last `decode_subframes` call produced, parsed on the device (navigation_message_parser.py),
        and the world model's per-satellite state advanced over the same milliseconds (world_model.py:707-861, one
        satellite per channel).  Returns per channel a list of (subframe, receiver_timestamp,
        trailing_edge_receiver_timestamp, ms) with `subframe` a NavigationMessageSubframe1..5."""
        from gypsum_b200.navigation_message_parser import subframe_from_fields

        fields = self.native.parse_subframes()
        out = []
        for c, rows in enumerate(fields):
            evs = [self._last_subframes[c][int(r["event_index"])] for r in rows]
            out.append([(subframe_from_fields(r), float(e["receiver_timestamp"]), float(e["trailing_edge_receiver_timestamp"]),
                         int(r["ms"])) for r, e in zip(rows, evs)])
        return out

    def orbital_parameters(self, channel: int) -> dict:
        """One channel's OrbitalParameters (world_model.py:151-199) as {OrbitalParameterType name: value or None}."""
        st = self.native.orbit_state(channel)
        return {name: (float(st["params"][k]) if st["set_mask"] >> k & 1 else None)
                for k, name in enumerate(ORBITAL_PARAMETER_NAMES)}

    def observations(self) -> np.ndarray:
        """_native.OBSERVATION_DTYPE [channel][ms] over the milliseconds of the last parse_subframes call: satellite
        time of week, clock correction and ECEF position as the world model computes them (world_model.py:379-487,
        :635-705), the PRN count and flags."""
        return self.native.observations()

    def position_fixes(self, start_times) -> np.ndarray:
        """_native.FIX_DTYPE [ms] over the milliseconds of the last parse_subframes call: the position fix the world
        model attempts every millisecond (world_model.py:567-633), start_times being the chunk start times.  The bank is
        one receiver: its clock slide, world-model order and stop carry from call to call.  With five or more ready
        satellites the reference raises: with fix_solver="reference" that millisecond has status 2 and the receiver
        stops for good; with "least_squares" it is fixed over all of them (n_ready of them; channel and pseudorange
        hold the first four), and only a rank-deficient system raises.
        gypsum_b200.world_model.solution_from_fix turns a status-1 record into a ReceiverSolution."""
        return self.native.position_fixes(start_times)

    def velocity_fixes(self) -> np.ndarray:
        """_native.VELOCITY_DTYPE [ms] over the milliseconds of the last parse_subframes call, after position_fixes: the
        receiver's ECEF velocity (m/s) and clock drift (s/s) from the channels' tracker Dopplers of the last `process`
        call, solved by least squares over the rows of each solved fix, with the fix's WGS-84 latitude, longitude and
        height and the GDOP / PDOP / HDOP / VDOP / TDOP of its geometry (DESIGN.md §8d).  status 1: solved (residual_rms
        with more than four rows); 0: no solved fix at that millisecond; 2: rank-deficient rows or a non-finite input,
        where only the geodetic position is set."""
        return self.native.velocity_fixes()

    def signal_quality(self, start_times, window_ms: int = 1000) -> list:
        """Each channel's carrier-to-noise density (dB-Hz) and phase-lock indicator over windows of window_ms consecutive
        milliseconds of the tracking records the last `process` / `process_ring` call left on the device (DESIGN.md
        §8e).  One estimator per channel, kept across calls: a window a call leaves open carries into the next, and
        window_ms is fixed by the first call.  A channel stops at its first lost record.  Returns one
        _native.SIGNAL_DTYPE array per channel; status 1: a signal (cn0_dbhz at least 1 dB above
        cn0_noise_floor_dbhz), 2: nothing distinguishable from noise, 0: a stop cut the window below 20 ms.  Reads the
        chain without changing it: integrate_bits and the calls after it give the same results with or without it."""
        return self.native.signal_windows(len(start_times), start_times, window_ms)


def cn0_noise_floor_dbhz(samples_per_ms: int) -> float:
    """What the C/N0 estimate of TrackerBank.signal_quality reads for noise alone at this many samples per
    millisecond: 10 log10((H_N - 1) / 1 ms), H_N the N-th harmonic number (38.57 dB-Hz at 2046, 39.68 at 16368)."""
    h = 0.0
    for k in range(1, int(samples_per_ms) + 1):
        h += 1.0 / k
    return 10.0 * math.log10((h - 1.0) / 1e-3)


# OrbitalParameterType (world_model.py:151-199), in order
ORBITAL_PARAMETER_NAMES = (
    "SQRT_SEMI_MAJOR_AXIS", "SEMI_MAJOR_AXIS", "ECCENTRICITY", "INCLINATION", "LONGITUDE_OF_ASCENDING_NODE",
    "ARGUMENT_OF_PERIGEE", "MEAN_ANOMALY_AT_REFERENCE_TIME", "MEAN_MOTION_DIFFERENCE",
    "CORRECTION_TO_ARGUMENT_OF_LATITUDE_COS", "CORRECTION_TO_ARGUMENT_OF_LATITUDE_SIN", "CORRECTION_TO_ORBITAL_RADIUS_COS",
    "CORRECTION_TO_ORBITAL_RADIUS_SIN", "CORRECTION_TO_INCLINATION_ANGLE_COS", "CORRECTION_TO_INCLINATION_ANGLE_SIN",
    "RATE_OF_RIGHT_ASCENSION", "RATE_OF_INCLINATION_ANGLE", "WEEK_NUMBER", "EPHEMERIS_REFERENCE_TIME",
    "GPS_TIME_OF_WEEK_AT_LAST_TIMESTAMP", "RECEIVER_TIMESTAMP_AT_LAST_HOW_TIMESTAMP", "PRN_TIMESTAMP_OF_LEADING_EDGE_OF_TOW",
    "A_F0", "A_F1", "A_F2", "T_OC", "ESTIMATED_GROUP_DELAY_DIFFERENTIAL")
