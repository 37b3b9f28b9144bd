// Navigation-message subframe decoding (reference gypsum/navigation_message_decoder.py:88-269 and the parts of
// gypsum/navigation_message_parser.py:307-424 it relies on) as a per-channel state machine over the 50 bps bit events of
// bits_core.cuh: subframe phase and polarity search, TLM prelude and HOW subframe-id checks, and the reference's
// decisions on every odd path (a reset inside the drain loop keeps draining, the phase is consumed modulo 300, subframe
// 5 with a data id other than 01 raises).
//
// The queue of bits is a ring of kNavQueueCap bits held as two bit planes (value, known) plus the per-bit timestamps.
// It is the one known difference from the reference, whose queue grows without bound while no phase is found: a bit
// that arrives while kNavQueueCap bits are queued latches `stopped = kNavStopOverflow` and is not taken.
// Host/device code: the device runs it on one lane per channel with a warp-parallel full preamble scan (nav.cu), the
// host emulator (tests/emu/nav_emu.cu) runs it with the scalar scan below.
#pragma once
#include "bits_core.cuh"

namespace gb {

constexpr int kSubframeBits = 300;        // navigation_message_decoder.py:23 BITS_PER_SUBFRAME
constexpr int kNavSearchMinBits = 600;    // :125 two subframes queued before the phase search runs
constexpr int kNavGiveUpBits = 3600;      // :155 twelve subframes queued without a phase: CannotDetermine on every bit
constexpr int kNavQueueCap = 4096;        // bits; see `stopped`
constexpr int kNavQueueWords = kNavQueueCap / 32;
constexpr uint32_t kPreambleUp = 0xD1u;   // 10001011 (:24-33), first bit in bit 0
constexpr uint32_t kPreambleInv = 0x2Eu;  // the same, inverted
constexpr uint32_t kWordMask = 0x3FFFFFFFu;

enum SubframeEventKind { kNavSubframe = 0, kNavDeterminedPhase = 1, kNavCannotDetermine = 2, kNavRaised = 3 };
enum NavStop { kNavRunning = 0, kNavStopRaised = 1, kNavStopOverflow = 2, kNavStopLostLock = 3 };

struct SubframeEvent {  // mirrors include/gypsum_b200.h gb200_subframe_event, 96 bytes
    double receiver_timestamp;                // first bit's receiver_timestamp (:203)
    double trailing_edge_receiver_timestamp;  // last bit's trailing edge (:204)
    uint32_t words[10];  // the 300 bits after the polarity flip, IS-GPS-200 bit 1 of each word in bit 29
    int kind;            // SubframeEventKind
    int bit_index;       // bit (within the call) whose arrival produced the event
    int subframe_id;     // HOW subframe id, 1..5
    int tow;             // HOW time-of-week count (17 bits)
    int phase;           // determined_subframe_phase, -1 = None
    int polarity;        // +1 POSITIVE, -1 NEGATIVE, 0 None
    int parity_ok;       // bit k: word k+1 satisfies the IS-GPS-200 parity equations
    int pad_[3];
};
static_assert(sizeof(SubframeEvent) == 96, "subframe event must stay 96 bytes");

// Scalar part of the decoder: lives in registers while the kernel walks a channel.
struct NavHead {
    long long bits;   // bit events taken
    int phase;        // history.determined_subframe_phase, -1 = None
    int polarity;     // determined_polarity: +1 / -1 / 0 = None
    int emitted;      // history.emitted_subframe_count
    int qlen, qhead;  // queued_bit_events as a ring of kNavQueueCap bits
    int scanned;      // queue length at which the last search found no pair (queue unchanged since but for appends), -1
    int stopped;      // NavStop
};

struct NavState {
    NavHead h;
    uint32_t val[kNavQueueWords];    // bit value (1 = BitValue.ONE), ring position p in word p >> 5, bit p & 31
    uint32_t known[kNavQueueWords];  // 0 = BitValue.UNKNOWN
    double qstart[kNavQueueCap], qend[kNavQueueCap];
};

// The pieces of one channel's state the state machine touches; the device points the planes at shared memory.
struct NavQueue {
    uint32_t* val;
    uint32_t* known;
    double* qstart;
    double* qend;
};

GB_HD inline void nav_state_init(NavHead& h) {
    h.bits = 0;
    h.phase = -1;
    h.polarity = 0;
    h.emitted = 0;
    h.qlen = h.qhead = 0;
    h.scanned = -1;
    h.stopped = kNavRunning;
}

GB_HD inline uint32_t nav_brev(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __brev(x);
#else
    uint32_t r = 0;
    for (int i = 0; i < 32; ++i) r |= ((x >> i) & 1u) << (31 - i);
    return r;
#endif
}

GB_HD inline int nav_popc(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __popc(x);
#else
    return __builtin_popcount(x);
#endif
}

// 32 bits of a plane starting at ring position `pos`: bit j is the bit at ring position pos + j.
GB_HD inline uint32_t nav_ring_bits(const uint32_t* plane, int pos) {
    const int w = pos >> 5, o = pos & 31;
    const uint64_t lo = plane[w], hi = plane[(w + 1) & (kNavQueueWords - 1)];
    return static_cast<uint32_t>(((hi << 32) | lo) >> o);
}

// utils.get_indexes_of_sublist for one position: queued bits [i, i+8) equal the pattern, none of them UNKNOWN.
GB_HD inline bool nav_preamble_at(const NavQueue& q, int qhead, int i, uint32_t pattern) {
    const int pos = (qhead + i) & (kNavQueueCap - 1);
    return (nav_ring_bits(q.val, pos) & 0xFFu) == pattern && (nav_ring_bits(q.known, pos) & 0xFFu) == 0xFFu;
}

// _identify_preamble_in_queued_bits (:88-114): the first candidate, in ascending order, with another candidate 300 bits
// later; -1 if there is none.  Scalar; nav.cu has the warp-parallel equivalent.
GB_HD inline int nav_first_pair(const NavQueue& q, int qhead, int qlen, uint32_t pattern) {
    for (int c = 0; c + kSubframeBits + 8 <= qlen; ++c)
        if (nav_preamble_at(q, qhead, c, pattern) && nav_preamble_at(q, qhead, c + kSubframeBits, pattern)) return c;
    return -1;
}

GB_HD inline void nav_pop(NavHead& h, int n) {
    h.qhead = (h.qhead + n) & (kNavQueueCap - 1);
    h.qlen -= n;
    h.scanned = -1;  // the front moved: the next search scans the whole queue
}

GB_HD inline void nav_reset(NavHead& h) {  // _reset_selected_subframe_phase (:116-121); the queue is kept
    h.phase = -1;
    h.polarity = 0;
}

GB_HD inline void nav_emit(const SubframeEvent& ev, SubframeEvent* out, int max_out, int& n_out) {
    if (n_out < max_out) out[n_out] = ev;
    n_out++;  // counts past max_out so the caller can see the truncation
}

GB_HD inline void nav_event_clear(SubframeEvent& ev, int kind, int bit_index, const NavHead& h) {
    ev.receiver_timestamp = ev.trailing_edge_receiver_timestamp = 0.0;
    for (int k = 0; k < 10; ++k) ev.words[k] = 0;
    ev.kind = kind;
    ev.bit_index = bit_index;
    ev.subframe_id = ev.tow = ev.parity_ok = 0;
    ev.phase = h.phase;
    ev.polarity = h.polarity;
    ev.pad_[0] = ev.pad_[1] = ev.pad_[2] = 0;
}

enum ParseResult { kParseNothing = 0, kParseEmit = 1, kParseRaise = 2 };

// parse_subframe (:198-269) on the first 300 queued bits, which it consumes.  Fills ev (kind left to the caller) when
// the result is kParseEmit or kParseRaise.
GB_HD inline int nav_parse_subframe(NavHead& h, const NavQueue& q, SubframeEvent& ev) {
    const int head = h.qhead;
    ev.receiver_timestamp = q.qstart[head];
    ev.trailing_edge_receiver_timestamp = q.qend[(head + kSubframeBits - 1) & (kNavQueueCap - 1)];
    bool all_known = true;
    for (int k = 0; k < 10; ++k) {
        const int pos = (head + 30 * k) & (kNavQueueCap - 1);
        ev.words[k] = nav_brev(nav_ring_bits(q.val, pos) & kWordMask) >> 2;
        all_known &= (nav_ring_bits(q.known, pos) & kWordMask) == kWordMask;
    }
    nav_pop(h, kSubframeBits);
    if (!all_known) {  // :209-224
        nav_reset(h);
        return kParseNothing;
    }
    if (h.polarity < 0)  // :226-229; None leaves the bits as they are
        for (int k = 0; k < 10; ++k) ev.words[k] ^= kWordMask;
    // preprocess_next_word (:307-369): data bits complemented by the previous word's D30; word 1 starts from 00.
    // Parity is only reported, as the reference only logs it (:383-391).
    // IS-GPS-200 Table 20-XIV: the source data bits d1..d24 (d1 in bit 23) that enter parity bits D25..D30, and
    // whether D29* (0) or D30* (1) of the previous word does.
    const uint32_t parity_mask[6] = {0xEC7CD2u, 0x763E69u, 0xBB1F34u, 0x5D8F9Au, 0xAEC7CDu, 0x2DEA27u};
    const int parity_prev[6] = {0, 1, 0, 1, 1, 0};
    uint32_t data[3] = {0, 0, 0};
    int parity_ok = 0;
    uint32_t d29 = 0, d30 = 0;
    for (int k = 0; k < 10; ++k) {
        const uint32_t w = ev.words[k];
        const uint32_t d = (w >> 6) ^ (d30 ? 0xFFFFFFu : 0u);
        bool ok = true;
        for (int j = 0; j < 6; ++j) {
            const uint32_t want = (static_cast<uint32_t>(nav_popc(d & parity_mask[j])) ^ (parity_prev[j] ? d30 : d29)) & 1u;
            ok &= want == ((w >> (5 - j)) & 1u);
        }
        parity_ok |= (ok ? 1 : 0) << k;
        if (k < 3) data[k] = d;
        d29 = (w >> 1) & 1u;
        d30 = w & 1u;
    }
    ev.parity_ok = parity_ok;
    if ((data[0] >> 16) != 0x8Bu) {  // parse_telemetry_word (:393-409)
        nav_reset(h);
        return kParseNothing;
    }
    const int id = static_cast<int>((data[1] >> 2) & 7u);  // parse_handover_word (:411-424): HOW bits 20-22
    if (id < 1 || id > 5) {
        nav_reset(h);
        return kParseNothing;
    }
    ev.subframe_id = id;
    ev.tow = static_cast<int>(data[1] >> 7);
    ev.phase = h.phase;
    ev.polarity = h.polarity;
    if (id == 5 && (data[2] >> 22) != 1u) return kParseRaise;  // parse_subframe_5: match_bits([0, 1]) on word 3
    return kParseEmit;
}

enum NavPush { kNavNoScan = 0, kNavFullScan = 1, kNavSkip = 2 };

// First half of process_bit_from_satellite (:173-196): queue the bit.  Returns kNavFullScan when the phase search that
// follows has to look at the whole queue (the caller runs it, see nav_first_pair), kNavSkip when the decoder is or just
// became stopped.
GB_HD inline int nav_push(NavHead& h, const NavQueue& q, int bit_value, double start, double end) {
    if (h.stopped) return kNavSkip;
    if (h.qlen == kNavQueueCap) {
        h.stopped = kNavStopOverflow;
        return kNavSkip;
    }
    const int pos = (h.qhead + h.qlen) & (kNavQueueCap - 1);
    const uint32_t bit = 1u << (pos & 31);
    uint32_t& v = q.val[pos >> 5];
    uint32_t& k = q.known[pos >> 5];
    v = bit_value == 1 ? (v | bit) : (v & ~bit);
    k = bit_value >= 0 ? (k | bit) : (k & ~bit);
    q.qstart[pos] = start;
    q.qend[pos] = end;
    h.qlen++;
    h.bits++;
    if (h.phase < 0 && h.qlen >= kNavSearchMinBits && h.scanned != h.qlen - 1) return kNavFullScan;
    return kNavNoScan;
}

// Second half: the phase search (:123-171) and the drain loop (:182-194).  pair_up / pair_inv: nav_first_pair of the
// upright / inverted preamble when nav_push asked for a full scan (ignored otherwise).  n_at_bit: events produced
// before this bit, so that a raise can drop the ones this bit produced -- the reference's exception takes them along.
GB_HD inline void nav_finish(NavHead& h, const NavQueue& q, int scan, int pair_up, int pair_inv, int bit_index,
                             SubframeEvent* out, int max_out, int& n_out, int n_at_bit) {
    if (scan == kNavSkip) return;
    SubframeEvent ev;
    if (h.phase < 0 && h.qlen >= kNavSearchMinBits) {
        if (scan != kNavFullScan) {
            // Nothing but this append since a search without a pair: the only new candidate is at qlen - 8, so the only
            // new pair is (qlen - 308, qlen - 8), and it is the first one if it exists.
            const int c = h.qlen - kSubframeBits - 8;
            pair_up = nav_preamble_at(q, h.qhead, c, kPreambleUp) && nav_preamble_at(q, h.qhead, c + kSubframeBits, kPreambleUp) ? c : -1;
            pair_inv = nav_preamble_at(q, h.qhead, c, kPreambleInv) && nav_preamble_at(q, h.qhead, c + kSubframeBits, kPreambleInv) ? c : -1;
        }
        if (pair_up >= 0 || pair_inv >= 0) {
            h.phase = pair_up >= 0 ? pair_up : pair_inv;  // the upright preamble is searched first
            h.polarity = pair_up >= 0 ? 1 : -1;
            nav_event_clear(ev, kNavDeterminedPhase, bit_index, h);
            nav_emit(ev, out, max_out, n_out);
            nav_pop(h, h.phase % kSubframeBits);  // :145-146: phase % 300 bits, not phase
        } else {
            h.scanned = h.qlen;
            if (h.qlen >= kNavGiveUpBits) {
                nav_event_clear(ev, kNavCannotDetermine, bit_index, h);
                nav_emit(ev, out, max_out, n_out);
            }
        }
    }
    if (h.phase < 0) return;
    // The drain loop does not look at the phase again: after a reset inside it the remaining whole subframes are still
    // parsed, with polarity None.
    while (h.qlen >= kSubframeBits) {
        nav_event_clear(ev, kNavSubframe, bit_index, h);
        const int r = nav_parse_subframe(h, q, ev);
        if (r == kParseEmit) {
            h.emitted++;
            nav_emit(ev, out, max_out, n_out);
        } else if (r == kParseRaise) {
            n_out = n_at_bit;
            ev.kind = kNavRaised;
            nav_emit(ev, out, max_out, n_out);
            h.stopped = kNavStopRaised;
            return;
        }
    }
}

// process_bit_from_satellite for one bit with the scalar scan (the host emulator's path).
GB_HD inline void nav_step(NavHead& h, const NavQueue& q, int bit_value, double start, double end, int bit_index,
                           SubframeEvent* out, int max_out, int& n_out) {
    const int n_at_bit = n_out;
    const int scan = nav_push(h, q, bit_value, start, end);
    int up = -1, inv = -1;
    if (scan == kNavFullScan) {
        up = nav_first_pair(q, h.qhead, h.qlen, kPreambleUp);
        if (up < 0) inv = nav_first_pair(q, h.qhead, h.qlen, kPreambleInv);
    }
    nav_finish(h, q, scan, up, inv, bit_index, out, max_out, n_out, n_at_bit);
}

}  // namespace gb
