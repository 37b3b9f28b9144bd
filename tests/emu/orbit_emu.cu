// Host build of the subframe field parser, the per-satellite world-model state and the per-millisecond time and position
// (gypsum_b200/csrc/orbit_core.cuh), for tests/test_orbit_cpu.py.  Built with nvcc for the host only; no device code runs.
#include <cstddef>
#include <cstring>
#include <vector>

#include "../../gypsum_b200/csrc/orbit_core.cuh"
#include "../../include/gypsum_b200.h"

using namespace gb;

static_assert(sizeof(gb200_subframe_fields) == sizeof(SubframeFields), "ABI and device subframe fields must match");
static_assert(sizeof(gb200_sv_observation) == sizeof(SvObservation), "ABI and device observations must match");

extern "C" {
int orbit_emu_state_size() { return (int)sizeof(OrbitSnap); }
void orbit_emu_init(OrbitSnap* st) { orbit_state_init(*st); }
// One channel's call, as k_parse_subframes and k_sv_observations run it: n events with their milliseconds, the drop
// millisecond (-1 = none); fields_out [n], obs_out [n_ms].  Returns the number of fields.
int orbit_emu_call(OrbitSnap* st, int n, const SubframeEvent* ev, const int* ms, int drop_ms, int n_ms, SubframeFields* fields_out,
                   SvObservation* obs_out) {
    std::vector<OrbitSnap> chg(n + 2);
    int n_fields = 0, n_chg = 0;
    orbit_walk(*st, ev, n, [&](int j, const SubframeEvent&) { return ms[j]; }, drop_ms, n_ms, fields_out, n_fields, chg.data(), n_chg);
    for (int m = 0; m < n_ms; ++m) orbit_observe(orbit_change_at(chg.data(), n_chg, m), m, obs_out[m]);
    return n_fields;
}
void orbit_emu_params(const OrbitSnap* st, double* params /*[26]*/, long long* out /*[3]: mask, count, counting*/) {
    memcpy(params, st->p, sizeof(st->p));
    out[0] = st->set;
    out[1] = st->count;
    out[2] = st->counting;
}
// offsets of gb200_subframe_fields' and gb200_sv_observation's fields as the C++ compiler lays them out
void orbit_emu_layout(long long* out /*[17]*/) {
    out[0] = offsetof(gb200_subframe_fields, event_index);
    out[1] = offsetof(gb200_subframe_fields, ms);
    out[2] = offsetof(gb200_subframe_fields, subframe_id);
    out[3] = offsetof(gb200_subframe_fields, tow_seconds);
    out[4] = offsetof(gb200_subframe_fields, ints);
    out[5] = offsetof(gb200_subframe_fields, bits);
    out[6] = offsetof(gb200_subframe_fields, bit_widths);
    out[7] = offsetof(gb200_subframe_fields, values);
    out[8] = sizeof(gb200_subframe_fields);
    out[9] = offsetof(gb200_sv_observation, tow);
    out[10] = offsetof(gb200_sv_observation, dsv);
    out[11] = offsetof(gb200_sv_observation, x);
    out[12] = offsetof(gb200_sv_observation, y);
    out[13] = offsetof(gb200_sv_observation, z);
    out[14] = offsetof(gb200_sv_observation, prn_count);
    out[15] = offsetof(gb200_sv_observation, flags);
    out[16] = sizeof(gb200_sv_observation);
}
}
