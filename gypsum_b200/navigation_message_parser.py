"""The subframe types of gypsum/navigation_message_parser.py, built from the fields the device parses
(gb200_tracker_parse_subframes, _native.FIELDS_DTYPE).  Names, field order and types are the reference's: bit-list
fields are list[int], first bit first."""
from __future__ import annotations

import math
from dataclasses import dataclass
from enum import Enum, auto

GPS_EPOCH_BASE_WEEK_NUMBER = 2048  # config.py


class GpsSubframeId(Enum):
    ONE = auto()
    TWO = auto()
    THREE = auto()
    FOUR = auto()
    FIVE = auto()


@dataclass
class HandoverWord:
    time_of_week: list[int]
    alert_flag: int
    anti_spoof_flag: int
    subframe_id: GpsSubframeId
    to_be_solved: list[int]

    @property
    def time_of_week_in_seconds(self) -> float:
        acc = 0
        for i, bit in enumerate(reversed(self.time_of_week)):
            if bit == 1:
                acc += 1.5 * (math.pow(2, i + 2))
        return acc


@dataclass
class NavigationMessageSubframe:
    @property
    def subframe_id(self) -> GpsSubframeId:
        raise NotImplementedError("Must be provided by subclasses")


@dataclass
class NavigationMessageSubframe1(NavigationMessageSubframe):
    week_num_mod_1024_bits: int
    ca_or_p_on_l2: list[int]
    ura_index: list[int]
    sv_health: list[int]
    issue_of_data_clock: list[int]
    l2_p_data_flag: int
    estimated_group_delay_differential: float
    t_oc: float
    a_f2: float
    a_f1: float
    a_f0: float

    @property
    def subframe_id(self) -> GpsSubframeId:
        return GpsSubframeId.ONE

    @property
    def week_num(self) -> int:
        return self.week_num_mod_1024_bits + GPS_EPOCH_BASE_WEEK_NUMBER


@dataclass
class NavigationMessageSubframe2(NavigationMessageSubframe):
    issue_of_data_ephemeris: list[int]
    correction_to_orbital_radius_sin: float
    mean_motion_difference_from_computed_value: float
    mean_anomaly_at_reference_time: float
    correction_to_latitude_cos: float
    eccentricity: float
    correction_to_latitude_sin: float
    sqrt_semi_major_axis: float
    reference_time_ephemeris: float
    fit_interval_flag: bool
    age_of_data_offset: list[int]

    @property
    def subframe_id(self) -> GpsSubframeId:
        return GpsSubframeId.TWO


@dataclass
class NavigationMessageSubframe3(NavigationMessageSubframe):
    correction_to_inclination_angle_cos: float
    longitude_of_ascending_node: float
    correction_to_inclination_angle_sin: float
    inclination_angle: float
    correction_to_orbital_radius_cos: float
    argument_of_perigee: float
    rate_of_right_ascension: float
    rate_of_inclination_angle: float
    issue_of_data_ephemeris: list[int]

    @property
    def subframe_id(self) -> GpsSubframeId:
        return GpsSubframeId.THREE


@dataclass
class NavigationMessageSubframe4(NavigationMessageSubframe):
    data_id: int
    page_id: int

    @property
    def subframe_id(self) -> GpsSubframeId:
        return GpsSubframeId.FOUR


@dataclass
class NavigationMessageSubframe5(NavigationMessageSubframe):
    data_id: list[int]
    satellite_id: list[int]
    eccentricity: float
    time_of_ephemeris: float
    delta_inclination_angle: float
    right_ascension_rate: float
    sv_health: list[int]
    semi_major_axis_sqrt: float
    longitude_of_ascension_mode: float
    argument_of_perigree: float
    mean_anomaly_at_reference_time: float
    a_f0: float
    a_f1: float

    @property
    def subframe_id(self) -> GpsSubframeId:
        return GpsSubframeId.FIVE


def _bits(v: int, n: int) -> list[int]:
    return [(int(v) >> (n - 1 - i)) & 1 for i in range(n)]


def _num(v: float, integral: bool = False):
    """The reference's get_num: int * 2**exp is an int for exp >= 0, a float otherwise."""
    return int(v) if integral else float(v)


def subframe_from_fields(rec) -> NavigationMessageSubframe:
    """One FIELDS_DTYPE record -> the NavigationMessageSubframe1..5 the reference's parser returns for it."""
    sf = int(rec["subframe_id"])
    ints = [int(v) for v in rec["ints"]]
    bits = [_bits(b, int(w)) for b, w in zip(rec["bits"], rec["bit_widths"])]
    v = [float(x) for x in rec["values"]]
    if sf == 1:
        return NavigationMessageSubframe1(ints[0], bits[0], bits[1], bits[2], bits[3], ints[1], v[0], _num(v[1], True),
                                          v[2], v[3], v[4])
    if sf == 2:
        return NavigationMessageSubframe2(bits[0], v[0], v[1], v[2], v[3], v[4], v[5], v[6], _num(v[7], True),
                                          bool(ints[0]), bits[1])
    if sf == 3:
        return NavigationMessageSubframe3(v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7], bits[0])
    if sf == 4:
        return NavigationMessageSubframe4(ints[0], ints[1])
    if sf == 5:
        return NavigationMessageSubframe5(bits[0], bits[1], v[0], _num(v[1], True), v[2], v[3], bits[2], v[4], v[5],
                                          v[6], v[7], v[8], v[9])
    raise ValueError(f"subframe id {sf}")
