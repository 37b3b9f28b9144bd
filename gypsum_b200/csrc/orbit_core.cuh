// Subframe field parsing (reference gypsum/navigation_message_parser.py:426-673), the per-satellite orbit and clock
// parameter set the receiver's world model keeps (gypsum/world_model.py:151-199, :707-861), its PRN counting
// (receiver.py:106-137, world_model.py:297-328) and the per-millisecond satellite time of transmission and ECEF position
// (world_model.py:379-487, :635-705).  Host/device code: orbit.cu runs it on the device, tests/emu/orbit_emu.cu on the
// host.
//
// Every scaling of a parsed field is an exact power of two on an integer of at most 32 bits, so parsed values are
// bit-exact.  The time and position arithmetic is written with o_add / o_sub / o_mul, which the device does not contract
// into fused multiply-adds, in the reference's order of operations; only sin, cos, atan2 and the correctly rounded
// math.pow(A, 3) (see orbit_cube) can round differently from the reference's libm.
//
// Like the reference, parameters of different issues (IODE / IODC) mix: a new subframe 1 replaces the clock terms and
// leaves the ephemeris of subframes 2 and 3 as they were, and nothing checks that they belong together.
#pragma once
#include <math.h>

#include "nav_core.cuh"

namespace gb {

// OrbitalParameterType (world_model.py:151-199), in its order; auto() starts at 1, these start at 0.
enum OrbitParam {
    kSqrtA = 0, kSemiMajorAxis, kEccentricity, kInclination, kLongitudeOfAscendingNode, kArgumentOfPerigee,
    kMeanAnomaly, kMeanMotionDifference, kCuc, kCus, kCrc, kCrs, kCic, kCis, kRateOfRightAscension,
    kRateOfInclination, kWeekNumber, kToe, kTowAtLastTimestamp, kRxTimestampAtLastHow, kPrnTimestampOfLeadingEdge,
    kAf0, kAf1, kAf2, kToc, kTgd, kOrbitParams
};
static_assert(kOrbitParams == 26, "OrbitalParameterType has 26 members");
constexpr uint32_t kAllOrbitParams = (1u << kOrbitParams) - 1u;

constexpr double kPiReference = 3.1415926535898;           // world_model.py:39 _PI
constexpr int kWeekBase = 2048;                             // config.py GPS_EPOCH_BASE_WEEK_NUMBER
constexpr double kMu = 3.986004418e14;                      // world_model.py:384
constexpr double kEarthRotationRate = 7.2921151467e-5;      // :431
constexpr double kRelativisticF = -4.442807633e-10;         // :686
constexpr long long kFixGateCount = 6000;                   // :584

// gb200_sv_observation.flags
enum ObservationFlag {
    kObsTiming = 1,     // _can_interrogate_precise_timings_for_satellite (:330-360): time of week computed
    kObsComplete = 2,   // OrbitalParameters.is_complete(): position computed (with kObsTiming)
    kObsFixGate = 4,    // counting and the count <= 6000 (attempt_position_fix, :582-585)
    kObsCounting = 8,   // the receiver counts this satellite's PRNs (it is tracked)
    kObsFrozen = 16,    // the decoder raised (event kind 3): the reference receiver's step never returns
};

struct SubframeFields {  // mirrors include/gypsum_b200.h gb200_subframe_fields, 144 bytes
    int event_index;     // index of the event among the channel's events of the decode call
    int ms;              // millisecond (within the call) that produced the event
    int subframe_id;     // 1..5
    int reserved;
    double tow_seconds;  // HandoverWord.time_of_week_in_seconds
    int ints[2];         // plain integer fields, dataclass order
    uint32_t bits[4];    // bit-list fields, packed with the first bit most significant, dataclass order
    int widths[4];       // their lengths in bits (0 = unused)
    double values[10];   // float fields, dataclass order
};
static_assert(sizeof(SubframeFields) == 144, "subframe fields must stay 144 bytes");

// One satellite's world-model entry as it stands at the end of millisecond `ms` of a call.
struct OrbitSnap {
    double p[kOrbitParams];
    uint32_t set;     // bit k: parameter k is not None
    int ms;           // -1: before the call's first millisecond
    long long count;  // satellite_ids_to_prn_observations_since_last_handover_timestamp
    int counting;     // the satellite is in that map
    int frozen;       // the decoder raised at millisecond ms + 1: nothing changes any more
};

struct SvObservation {  // mirrors gb200_sv_observation, 56 bytes
    double tow;         // _gps_observed_system_time_of_week_for_satellite
    double dsv;         // its last delta_sv_time
    double x, y, z;     // _get_satellite_position_at_time_of_week at that time
    long long prn_count;
    int flags;          // ObservationFlag
    int reserved;
};
static_assert(sizeof(SvObservation) == 56, "observation must stay 56 bytes");

GB_HD GB_INLINE double o_add(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
GB_HD GB_INLINE double o_sub(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
GB_HD GB_INLINE double o_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}

GB_HD inline void orbit_state_init(OrbitSnap& s) {
    for (int k = 0; k < kOrbitParams; ++k) s.p[k] = 0.0;
    s.set = 0;
    s.ms = -1;
    s.count = 0;
    s.counting = 0;
    s.frozen = 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// parsing
// ---------------------------------------------------------------------------------------------------------------------

// Data bits [first, first + n) of data word `word` (both 1-based, IS-GPS-200 numbering).
GB_HD GB_INLINE uint32_t orbit_bits(const uint32_t* d, int word, int first, int n) {
    return (d[word - 1] >> (25 - first - n)) & static_cast<uint32_t>((1ull << n) - 1ull);
}
GB_HD GB_INLINE long long orbit_signed(uint32_t v, int n) {  // _get_twos_complement
    return (v >> (n - 1)) & 1u ? static_cast<long long>(v) - (1ll << n) : static_cast<long long>(v);
}
// get_num_from_bits: value * 2**exp, exact
GB_HD GB_INLINE double orbit_num(uint32_t v, int n, int exp, bool twos) {
    const double x = twos ? static_cast<double>(orbit_signed(v, n)) : static_cast<double>(v);
    return ldexp(x, exp);
}

// NavigationMessageSubframeParser on a subframe event's words: subframes 1-5 (5 only with data id 01, the decoder has
// already turned the others into event kind 3).
GB_HD inline void orbit_parse(const SubframeEvent& ev, SubframeFields& f) {
    uint32_t d[10];
    uint32_t d30 = 0;  // preprocess_next_word: word 1 starts from D30* = 0
    for (int k = 0; k < 10; ++k) {
        const uint32_t w = ev.words[k];
        d[k] = ((w >> 6) ^ (d30 ? 0xFFFFFFu : 0u)) & 0xFFFFFFu;
        d30 = w & 1u;
    }
    f.subframe_id = static_cast<int>(orbit_bits(d, 2, 20, 3));
    f.tow_seconds = static_cast<double>(orbit_bits(d, 2, 1, 17)) * 6.0;  // sum of 1.5 * 2**(i + 2), exact
    f.reserved = 0;
    for (int k = 0; k < 2; ++k) f.ints[k] = 0;
    for (int k = 0; k < 4; ++k) f.bits[k] = 0, f.widths[k] = 0;
    for (int k = 0; k < 10; ++k) f.values[k] = 0.0;
    double* v = f.values;
    switch (f.subframe_id) {
        case 1:  // :426-474
            f.ints[0] = static_cast<int>(orbit_bits(d, 3, 1, 10));  // week_num_mod_1024_bits
            f.bits[0] = orbit_bits(d, 3, 11, 2), f.widths[0] = 2;   // ca_or_p_on_l2
            f.bits[1] = orbit_bits(d, 3, 13, 4), f.widths[1] = 4;   // ura_index
            f.bits[2] = orbit_bits(d, 3, 17, 6), f.widths[2] = 6;   // sv_health
            f.bits[3] = (orbit_bits(d, 3, 23, 2) << 8) | orbit_bits(d, 8, 1, 8), f.widths[3] = 10;  // issue_of_data_clock
            f.ints[1] = static_cast<int>(orbit_bits(d, 4, 1, 1));   // l2_p_data_flag
            v[0] = orbit_num(orbit_bits(d, 7, 17, 8), 8, -31, true);    // estimated_group_delay_differential
            v[1] = orbit_num(orbit_bits(d, 8, 9, 16), 16, 4, false);    // t_oc
            v[2] = orbit_num(orbit_bits(d, 9, 1, 8), 8, -55, true);     // a_f2
            v[3] = orbit_num(orbit_bits(d, 9, 9, 16), 16, -43, true);   // a_f1
            v[4] = orbit_num(orbit_bits(d, 10, 1, 22), 22, -31, true);  // a_f0
            break;
        case 2:  // :476-537
            f.bits[0] = orbit_bits(d, 3, 1, 8), f.widths[0] = 8;  // issue_of_data_ephemeris
            v[0] = orbit_num(orbit_bits(d, 3, 9, 16), 16, -5, true);    // correction_to_orbital_radius_sin
            v[1] = orbit_num(orbit_bits(d, 4, 1, 16), 16, -43, true);   // mean_motion_difference_from_computed_value
            v[2] = orbit_num((orbit_bits(d, 4, 17, 8) << 24) | orbit_bits(d, 5, 1, 24), 32, -31, true);  // M0
            v[3] = orbit_num(orbit_bits(d, 6, 1, 16), 16, -29, true);   // correction_to_latitude_cos
            v[4] = orbit_num((orbit_bits(d, 6, 17, 8) << 24) | orbit_bits(d, 7, 1, 24), 32, -33, false);  // e
            v[5] = orbit_num(orbit_bits(d, 8, 1, 16), 16, -29, true);   // correction_to_latitude_sin
            v[6] = orbit_num((orbit_bits(d, 8, 17, 8) << 24) | orbit_bits(d, 9, 1, 24), 32, -19, false);  // sqrt A
            v[7] = orbit_num(orbit_bits(d, 10, 1, 16), 16, 4, false);   // reference_time_ephemeris
            f.ints[0] = static_cast<int>(orbit_bits(d, 10, 17, 1));     // fit_interval_flag
            f.bits[1] = orbit_bits(d, 10, 18, 5), f.widths[1] = 5;      // age_of_data_offset
            break;
        case 3:  // :539-597
            v[0] = orbit_num(orbit_bits(d, 3, 1, 16), 16, -29, true);   // correction_to_inclination_angle_cos
            v[1] = orbit_num((orbit_bits(d, 3, 17, 8) << 24) | orbit_bits(d, 4, 1, 24), 32, -31, true);  // Omega0
            v[2] = orbit_num(orbit_bits(d, 5, 1, 16), 16, -29, true);   // correction_to_inclination_angle_sin
            v[3] = orbit_num((orbit_bits(d, 5, 17, 8) << 24) | orbit_bits(d, 6, 1, 24), 32, -31, true);  // i0
            v[4] = orbit_num(orbit_bits(d, 7, 1, 16), 16, -5, true);    // correction_to_orbital_radius_cos
            v[5] = orbit_num((orbit_bits(d, 7, 17, 8) << 24) | orbit_bits(d, 8, 1, 24), 32, -31, true);  // omega
            v[6] = orbit_num(orbit_bits(d, 9, 1, 24), 24, -43, true);   // rate_of_right_ascension
            v[7] = orbit_num(orbit_bits(d, 10, 9, 14), 14, -43, true);  // rate_of_inclination_angle
            f.bits[0] = orbit_bits(d, 10, 1, 8), f.widths[0] = 8;       // issue_of_data_ephemeris
            break;
        case 4:  // :599-618
            f.ints[0] = static_cast<int>(orbit_bits(d, 3, 1, 2));  // data_id
            f.ints[1] = static_cast<int>(orbit_bits(d, 3, 3, 6));  // page_id
            break;
        case 5:  // :620-673
            f.bits[0] = orbit_bits(d, 3, 1, 2), f.widths[0] = 2;   // data_id
            f.bits[1] = orbit_bits(d, 3, 3, 6), f.widths[1] = 6;   // satellite_id
            v[0] = orbit_num(orbit_bits(d, 3, 9, 16), 16, -21, false);  // eccentricity
            v[1] = orbit_num(orbit_bits(d, 4, 1, 8), 8, 12, false);     // time_of_ephemeris
            v[2] = orbit_num(orbit_bits(d, 4, 9, 16), 16, -19, true);   // delta_inclination_angle
            v[3] = orbit_num(orbit_bits(d, 5, 1, 16), 16, -38, true);   // right_ascension_rate
            f.bits[2] = orbit_bits(d, 5, 17, 8), f.widths[2] = 8;       // sv_health
            v[4] = orbit_num(orbit_bits(d, 6, 1, 24), 24, -11, false);  // semi_major_axis_sqrt
            v[5] = orbit_num(orbit_bits(d, 7, 1, 24), 24, -23, true);   // longitude_of_ascension_mode
            v[6] = orbit_num(orbit_bits(d, 8, 1, 24), 24, -23, true);   // argument_of_perigree
            v[7] = orbit_num(orbit_bits(d, 9, 1, 24), 24, -23, true);   // mean_anomaly_at_reference_time
            v[8] = orbit_num((orbit_bits(d, 10, 1, 8) << 3) | orbit_bits(d, 10, 20, 3), 11, -20, true);  // a_f0
            v[9] = orbit_num(orbit_bits(d, 10, 9, 11), 11, -38, true);  // a_f1
            break;
        default:
            break;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// the world model's per-satellite state
// ---------------------------------------------------------------------------------------------------------------------

GB_HD GB_INLINE void orbit_set(OrbitSnap& s, int k, double v) {
    s.p[k] = v;
    s.set |= 1u << k;
}

// The count at the end of millisecond m >= s.ms: handle_prn_observed adds one per millisecond while the satellite is
// tracked.
GB_HD GB_INLINE long long orbit_count_at(const OrbitSnap& s, int m) {
    return s.counting && !s.frozen ? s.count + (m - s.ms) : s.count;
}

GB_HD GB_INLINE void orbit_advance(OrbitSnap& s, int m) {
    s.count = orbit_count_at(s, m);
    s.ms = m;
}

// handle_subframe_emitted (:707-807) with _process_subframe1..3 (:809-861), at the end of millisecond s.ms.
GB_HD inline void orbit_apply(OrbitSnap& s, const SubframeEvent& ev, const SubframeFields& f) {
    s.count = 0;
    s.counting = 1;
    orbit_set(s, kTowAtLastTimestamp, f.tow_seconds);
    orbit_set(s, kRxTimestampAtLastHow, ev.trailing_edge_receiver_timestamp);
    orbit_set(s, kPrnTimestampOfLeadingEdge, ev.trailing_edge_receiver_timestamp);
    const double* v = f.values;
    if (f.subframe_id == 1) {
        orbit_set(s, kWeekNumber, static_cast<double>(f.ints[0] + kWeekBase));
        orbit_set(s, kAf0, v[4]);
        orbit_set(s, kAf1, v[3]);
        orbit_set(s, kAf2, v[2]);
        orbit_set(s, kToc, v[1]);
        orbit_set(s, kTgd, v[0]);
    } else if (f.subframe_id == 2) {
        orbit_set(s, kMeanAnomaly, o_mul(v[2], kPiReference));
        orbit_set(s, kEccentricity, v[4]);
        orbit_set(s, kSqrtA, v[6]);
        orbit_set(s, kSemiMajorAxis, o_mul(v[6], v[6]));  // math.pow(sqrt A, 2)
        orbit_set(s, kMeanMotionDifference, o_mul(v[1], kPiReference));
        orbit_set(s, kToe, v[7]);
        orbit_set(s, kCuc, v[3]);
        orbit_set(s, kCus, v[5]);
        orbit_set(s, kCrs, v[0]);
    } else if (f.subframe_id == 3) {
        orbit_set(s, kInclination, o_mul(v[3], kPiReference));
        orbit_set(s, kArgumentOfPerigee, o_mul(v[5], kPiReference));
        orbit_set(s, kLongitudeOfAscendingNode, o_mul(v[1], kPiReference));
        orbit_set(s, kCic, v[0]);
        orbit_set(s, kCis, v[2]);
        orbit_set(s, kRateOfRightAscension, o_mul(v[6], kPiReference));
        orbit_set(s, kRateOfInclination, o_mul(v[7], kPiReference));
        orbit_set(s, kCrc, v[4]);
    }
}

// handle_lost_satellite_lock (:314-328): counting stops and the time of week is forgotten; the rest of the set stays.
GB_HD GB_INLINE void orbit_drop(OrbitSnap& s) {
    s.count = 0;
    s.counting = 0;
    s.set &= ~(1u << kTowAtLastTimestamp);
    s.p[kTowAtLastTimestamp] = 0.0;
}

// ---------------------------------------------------------------------------------------------------------------------
// time and position
// ---------------------------------------------------------------------------------------------------------------------

// math.pow(a, 3), correctly rounded as the reference's libm rounds it (a * a * a rounds twice): a double-double product.
GB_HD GB_INLINE double orbit_cube(double a) {
    const double p = o_mul(a, a);
    const double pe = fma(a, a, -p);
    const double q = o_mul(p, a);
    const double qe = fma(p, a, -q);
    return o_add(q, o_add(qe, o_mul(pe, a)));
}

// get_eccentric_anomaly (:379-408): seven fixed-point iterations of Kepler's equation.  n: corrected mean motion.
GB_HD GB_INLINE double orbit_mean_motion(const double* p) {
    const double a = o_mul(p[kSqrtA], p[kSqrtA]);
    return o_add(sqrt(kMu) / sqrt(orbit_cube(a)), p[kMeanMotionDifference]);
}
GB_HD GB_INLINE double orbit_eccentric_anomaly(const double* p, double n, double tk) {
    const double m = o_add(p[kMeanAnomaly], o_mul(n, tk));
    double e = m;
    for (int i = 0; i < 7; ++i) e = o_add(m, o_mul(p[kEccentricity], sin(e)));
    return e;
}

// _gps_observed_system_time_of_week_for_satellite (:635-705): the time of week at the last HOW plus 1 ms per PRN, less
// the clock correction of ten iterations.  `t` stays the uncorrected time, and Ek is taken at tk - delta_sv.
GB_HD inline double orbit_time_of_week(const double* p, long long count, double& dsv_out) {
    const double t = o_add(p[kTowAtLastTimestamp], o_mul(0.001, static_cast<double>(count)));
    const double tk = o_sub(t, p[kToe]);
    const double n = orbit_mean_motion(p);
    const double tc = o_sub(t, p[kToc]);
    double dsv = 0.0;
    for (int i = 0; i < 10; ++i) {
        const double ek = orbit_eccentric_anomaly(p, n, o_sub(tk, dsv));
        const double dtr = o_mul(o_mul(o_mul(kRelativisticF, p[kEccentricity]), p[kSqrtA]), sin(ek));
        const double a2 = o_mul(p[kAf2], tc);
        dsv = o_sub(o_add(o_add(o_add(p[kAf0], o_mul(p[kAf1], tc)), o_mul(a2, a2)), dtr), p[kTgd]);
    }
    dsv_out = dsv;
    return o_sub(t, dsv);
}

// _get_satellite_position_at_time_of_week (:410-487), with the +-302 400 s wrap of tk.
GB_HD inline void orbit_position(const double* p, double tow, double& x, double& y, double& z) {
    double tk = o_sub(tow, p[kToe]);
    if (tk > 302400.0) tk = o_sub(tk, 604800.0);
    else if (tk < -302400.0) tk = o_add(tk, 604800.0);
    const double e = p[kEccentricity];
    const double ek = orbit_eccentric_anomaly(p, orbit_mean_motion(p), tk);
    const double vk = atan2(o_mul(sqrt(o_sub(1.0, o_mul(e, e))), sin(ek)), o_sub(cos(ek), e));
    const double phi = o_add(vk, p[kArgumentOfPerigee]);
    const double s2 = sin(o_mul(2.0, phi)), c2 = cos(o_mul(2.0, phi));
    const double duk = o_add(o_mul(p[kCus], s2), o_mul(p[kCuc], c2));
    const double drk = o_add(o_mul(p[kCrs], s2), o_mul(p[kCrc], c2));
    const double dik = o_add(o_mul(p[kCis], s2), o_mul(p[kCic], c2));
    const double uk = o_add(phi, duk);
    const double rk = o_add(o_mul(p[kSemiMajorAxis], o_sub(1.0, o_mul(e, cos(ek)))), drk);
    const double ik = o_add(o_add(p[kInclination], o_mul(p[kRateOfInclination], tk)), dik);
    const double xp = o_mul(rk, cos(uk)), yp = o_mul(rk, sin(uk));
    const double om = o_sub(o_add(p[kLongitudeOfAscendingNode], o_mul(o_sub(p[kRateOfRightAscension], kEarthRotationRate), tk)),
                            o_mul(kEarthRotationRate, p[kToe]));
    const double so = sin(om), co = cos(om), ci = cos(ik);
    x = o_sub(o_mul(xp, co), o_mul(o_mul(yp, ci), so));
    y = o_add(o_mul(xp, so), o_mul(o_mul(yp, ci), co));
    z = o_mul(yp, sin(ik));
}

// The time derivative of orbit_position at the same tow, in the same frame (Omega's rate includes -omega_e; no Sagnac
// term, as the position fix has none), and of orbit_time_of_week's clock correction dsv: the satellite's ECEF velocity
// (m/s) and clock drift (s/s).  Ek is the same seven-iteration value, and Ek' = n / (1 - e cos Ek) that of Kepler's
// equation.  The drift differentiates the reference's own dsv expression: af1 + 2 af2^2 (t - toc) + F e sqrtA cos(Ek) Ek'.
// The af2^2 is the reference's pow(af2 * (t - toc), 2) (world_model.py:686), where IS-GPS-200 has af2 (t - toc)^2; t is
// taken as tow, which differs from the reference's uncorrected t by dsv (< 1 ms).  Like dsv, the relativistic term takes
// Ek at tow - toe without the week wrap.
GB_HD inline void orbit_velocity(const double* p, double tow, double& vx, double& vy, double& vz, double& drift) {
    const double tk0 = o_sub(tow, p[kToe]);
    double tk = tk0;
    if (tk > 302400.0) tk = o_sub(tk, 604800.0);
    else if (tk < -302400.0) tk = o_add(tk, 604800.0);
    const double e = p[kEccentricity];
    const double n = orbit_mean_motion(p);
    const double ek = orbit_eccentric_anomaly(p, n, tk);
    const double se = sin(ek), ce = cos(ek);
    const double den = o_sub(1.0, o_mul(e, ce));
    const double ekd = n / den;
    const double sq = sqrt(o_sub(1.0, o_mul(e, e)));
    const double vk = atan2(o_mul(sq, se), o_sub(ce, e));
    const double vkd = o_mul(sq, ekd) / den;  // d(vk)/dt
    const double phi = o_add(vk, p[kArgumentOfPerigee]);
    const double s2 = sin(o_mul(2.0, phi)), c2 = cos(o_mul(2.0, phi));
    const double duk = o_add(o_mul(p[kCus], s2), o_mul(p[kCuc], c2));
    const double drk = o_add(o_mul(p[kCrs], s2), o_mul(p[kCrc], c2));
    const double dik = o_add(o_mul(p[kCis], s2), o_mul(p[kCic], c2));
    const double w2 = o_mul(2.0, vkd);
    const double uk = o_add(phi, duk);
    const double ukd = o_add(vkd, o_mul(w2, o_sub(o_mul(p[kCus], c2), o_mul(p[kCuc], s2))));
    const double rk = o_add(o_mul(p[kSemiMajorAxis], o_sub(1.0, o_mul(e, ce))), drk);
    const double rkd = o_add(o_mul(o_mul(o_mul(p[kSemiMajorAxis], e), se), ekd), o_mul(w2, o_sub(o_mul(p[kCrs], c2), o_mul(p[kCrc], s2))));
    const double ik = o_add(o_add(p[kInclination], o_mul(p[kRateOfInclination], tk)), dik);
    const double ikd = o_add(p[kRateOfInclination], o_mul(w2, o_sub(o_mul(p[kCis], c2), o_mul(p[kCic], s2))));
    const double cu = cos(uk), su = sin(uk);
    const double xp = o_mul(rk, cu), yp = o_mul(rk, su);
    const double xpd = o_sub(o_mul(rkd, cu), o_mul(o_mul(rk, ukd), su));
    const double ypd = o_add(o_mul(rkd, su), o_mul(o_mul(rk, ukd), cu));
    const double omd = o_sub(p[kRateOfRightAscension], kEarthRotationRate);
    const double om = o_sub(o_add(p[kLongitudeOfAscendingNode], o_mul(omd, tk)), o_mul(kEarthRotationRate, p[kToe]));
    const double so = sin(om), co = cos(om), ci = cos(ik), si = sin(ik);
    const double x = o_sub(o_mul(xp, co), o_mul(o_mul(yp, ci), so));
    const double y = o_add(o_mul(xp, so), o_mul(o_mul(yp, ci), co));
    const double yi = o_mul(o_mul(yp, si), ikd);  // d(cos ik)/dt = -sin(ik) ik'
    vx = o_sub(o_add(o_sub(o_mul(xpd, co), o_mul(o_mul(ypd, ci), so)), o_mul(yi, so)), o_mul(y, omd));
    vy = o_add(o_sub(o_add(o_mul(xpd, so), o_mul(o_mul(ypd, ci), co)), o_mul(yi, co)), o_mul(x, omd));
    vz = o_add(o_mul(ypd, si), o_mul(o_mul(yp, ci), ikd));
    const double tc = o_sub(tow, p[kToc]);
    const double ec = tk == tk0 ? ek : orbit_eccentric_anomaly(p, n, tk0);
    const double cc = tk == tk0 ? ce : cos(ec);
    const double rel = o_mul(o_mul(o_mul(o_mul(kRelativisticF, e), p[kSqrtA]), cc), n / o_sub(1.0, o_mul(e, cc)));
    drift = o_add(o_add(p[kAf1], o_mul(o_mul(2.0, o_mul(p[kAf2], p[kAf2])), tc)), rel);
}

// What the world model knows about one satellite at the end of millisecond m (>= s.ms, with no change in between).
GB_HD inline void orbit_observe(const OrbitSnap& s, int m, SvObservation& o) {
    const long long count = orbit_count_at(s, m);
    constexpr uint32_t kTimingParams = (1u << kTowAtLastTimestamp) | (1u << kEccentricity) | (1u << kSqrtA) | (1u << kAf0) |
                                       (1u << kAf1) | (1u << kAf2) | (1u << kToc) | (1u << kTgd);
    int flags = 0;
    if (s.counting) flags |= kObsCounting;
    if (s.counting && (s.set & kTimingParams) == kTimingParams) flags |= kObsTiming;
    if (s.set == kAllOrbitParams) flags |= kObsComplete;
    if (s.counting && count <= kFixGateCount) flags |= kObsFixGate;
    if (s.frozen) flags |= kObsFrozen;
    o.prn_count = s.counting ? count : -1;
    o.flags = flags;
    o.reserved = 0;
    o.tow = o.dsv = o.x = o.y = o.z = NAN;
    if (flags & kObsTiming) {
        o.tow = orbit_time_of_week(s.p, count, o.dsv);
        if (flags & kObsComplete) orbit_position(s.p, o.tow, o.x, o.y, o.z);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// one channel's call
// ---------------------------------------------------------------------------------------------------------------------

// The state the call starts from: the carried state, tracked from millisecond 0 unless it is dropped there.  Returns
// true when the satellite starts counting here, so that millisecond 0 is the first one it is seen in.
GB_HD GB_INLINE bool orbit_begin(OrbitSnap& s, int drop_ms) {
    s.ms = -1;
    if (!s.frozen && drop_ms != 0 && !s.counting) {  // handle_prn_observed: a satellite seen for the first time starts at 0
        s.counting = 1;
        s.count = 0;
        return true;
    }
    return false;
}

// One decoder event at millisecond m (non-decreasing within the call) of a channel dropped at drop_ms (-1 = never); f:
// the event's fields when it is a subframe (kind 0); fresh: orbit_begin started the channel counting.  The events of
// one millisecond apply in order, so a subframe before a raise in the same millisecond holds and one after it does not
// (DESIGN.md §8b).  Returns true when the state changed and `s` (the state at the end of m) belongs in the change table.
GB_HD inline bool orbit_event(OrbitSnap& s, const SubframeEvent& ev, int m, int drop_ms, const SubframeFields& f, bool fresh) {
    if (s.frozen || (drop_ms >= 0 && m >= drop_ms)) return false;  // the receiver has dropped this pipeline
    if (ev.kind == kNavSubframe) {
        orbit_advance(s, m);
        orbit_apply(s, ev, f);
        return true;
    }
    if (ev.kind == kNavRaised) {  // uncaught ValueError: the receiver stops before it counts millisecond m
        if (fresh && m == 0 && s.ms < 0) s.counting = 0;  // ... so a satellite first seen at m was never counted
        s.count = orbit_count_at(s, m - 1 > s.ms ? m - 1 : s.ms);
        s.ms = m;
        s.frozen = 1;
        return true;
    }
    return false;  // kinds 1 and 2 (2 is the drop, placed by the caller)
}

// One channel's call: the n decoder events ev (event j at millisecond ms_of(j)) and the drop.  Writes the fields of every
// subframe event and the change table (entry 0: the state before millisecond 0), and leaves in `s` the state carried to
// the next call.
template <class MsOf>
GB_HD inline void orbit_walk(OrbitSnap& s, const SubframeEvent* ev, int n, MsOf ms_of, int drop_ms, int n_ms,
                             SubframeFields* fields, int& n_fields, OrbitSnap* chg, int& n_chg) {
    const bool fresh = orbit_begin(s, drop_ms);
    n_fields = n_chg = 0;
    chg[n_chg++] = s;
    for (int j = 0; j < n; ++j) {
        const SubframeEvent e = ev[j];
        const int m = ms_of(j, e);
        SubframeFields f;
        if (e.kind == kNavSubframe) {
            orbit_parse(e, f);
            f.event_index = j;
            f.ms = m;
            fields[n_fields++] = f;
        }
        if (orbit_event(s, e, m, drop_ms, f, fresh)) chg[n_chg++] = s;
    }
    if (drop_ms >= 0 && !s.frozen) {
        orbit_advance(s, drop_ms);
        orbit_drop(s);
        chg[n_chg++] = s;
    }
    orbit_advance(s, n_ms - 1);
    s.ms = -1;
}

// The change that holds at millisecond m: the last entry at or before it.
GB_HD GB_INLINE const OrbitSnap& orbit_change_at(const OrbitSnap* chg, int n_chg, int m) {
    int k = n_chg - 1;
    while (k > 0 && chg[k].ms > m) --k;
    return chg[k];
}

}  // namespace gb
