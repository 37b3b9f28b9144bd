// Host build of the scalar tracking loop (gypsum_b200/csrc/tracker_core.cuh) with the code-phase modulus as an
// argument, and of the pseudosymbol delay rule the bit integrator stamps with.  Test infrastructure; never loaded by
// the product.
#include "../../gypsum_b200/csrc/tracker_core.cuh"

using namespace gb;

extern "C" {
int track_emu_state_size() { return (int)sizeof(TrackState); }
void track_emu_init(TrackState* st, int prn, double doppler, double carrier_phase, int code_phase) {
    track_state_init(*st, prn, doppler, carrier_phase, code_phase);
}
// elp: E.re E.im L.re L.im P.re P.im
void track_emu_update(TrackState* st, const float* elp, float strength, int off, double t0, double fs, double wrap,
                      TrackMsRecord* out) {
    const TrackConsts tc = track_consts(fs, wrap);
    track_update(*st, make_float2(elp[0], elp[1]), make_float2(elp[2], elp[3]), make_float2(elp[4], elp[5]), strength, off,
                 t0, tc, nullptr, *out);
}
// n symbols: start / end stamps of each from its code phase and chunk times, as k_integrate_bits forms them
void track_emu_stamps(int n, const int* code_phase, const double* t0, const double* t1, double wrap, double* ts, double* te) {
    for (int k = 0; k < n; ++k) {
        const double delay = track_symbol_delay(code_phase[k], wrap);
        ts[k] = t0[k] + delay;
        te[k] = t1[k] + delay;
    }
}
}
