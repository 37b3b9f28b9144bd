"""Generate tests/golden/nav_decoder.npz by running the LIVE reference NavigationMessageDecoder
(gypsum/navigation_message_decoder.py) on synthetic LNAV bit streams, fed as reference EmitNavigationBitEvents.
Run with the reference checkout on the path: PYTHONPATH=<reference checkout> python tools/make_golden_subframes.py

Per stream s the file holds s_bits (1 / 0 / -1 = unknown), s_t0 / s_t1 (bit timestamps), s_events (float64 rows:
bit index, kind, subframe id, TOW count, phase, polarity, parity_ok, t0, t1), s_words (int64 [n, 10]: the 300 bits the
reference's NavigationMessageSubframeParser was given, 30 per word, first bit most significant) and s_final
(phase or -1, emitted_subframe_count, polarity, queued bits, stopped, bits taken).  Kinds: 0 EmitSubframeEvent,
1 DeterminedSubframePhaseEvent, 2 CannotDetermineSubframePhaseEvent, 3 the decoder raised (ValueError; the stream
stops there).  parity_ok comes from the reference parser's own parity check (one bit per word without a logged
failure)."""
import logging
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import gypsum.navigation_message_decoder as nmd  # noqa: E402
import gypsum.navigation_message_parser as nmp  # noqa: E402
from gypsum.navigation_bit_intergrator import EmitNavigationBitEvent  # noqa: E402
from gypsum.tracker import BitValue  # noqa: E402

from oracle import nav_oracle as nav  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "nav_decoder.npz")
BITVAL = {1: BitValue.ONE, 0: BitValue.ZERO, -1: BitValue.UNKNOWN}


class _Failures(logging.Handler):
    def __init__(self):
        super().__init__(logging.INFO)
        self.n = 0

    def emit(self, record):
        if "Failed parity check" in record.getMessage():
            self.n += 1


_FAIL = _Failures()
_plog = logging.getLogger(nmp.__name__)
_plog.addHandler(_FAIL)
_plog.setLevel(logging.INFO)
_plog.propagate = False
logging.getLogger(nmd.__name__).setLevel(logging.WARNING)

_given: list = []  # bits handed to each NavigationMessageSubframeParser the decoder builds


class _RecordingParser(nmp.NavigationMessageSubframeParser):
    def __init__(self, bits):
        _given.append(list(bits))
        super().__init__(bits)


nmd.NavigationMessageSubframeParser = _RecordingParser


def _word_values(bits):
    return tuple(nav.word_value(bits[30 * k: 30 * k + 30]) for k in range(10))


def _parity_ok(bits) -> int:
    p = nmp.NavigationMessageSubframeParser(bits)
    ok = 0
    for k in range(10):
        before = _FAIL.n
        p.preprocess_next_word()
        ok |= (1 if _FAIL.n == before else 0) << k
    return ok


def _polarity(p) -> int:
    return {None: 0, nmd.BitPolarity.POSITIVE: 1, nmd.BitPolarity.NEGATIVE: -1}[p]


def run(bits, t0, t1):
    dec = nmd.NavigationMessageDecoder()
    parsed = []  # per successful / raising parse: (t0, t1, bits given, phase, polarity)
    orig = dec.parse_subframe

    def parse_subframe():
        block = dec.queued_bit_events[:nav.SUBFRAME]
        n_given = len(_given)
        try:
            res = orig()
        except ValueError:
            parsed.append((block[0].receiver_timestamp, block[-1].trailing_edge_receiver_timestamp, _given[n_given],
                           dec.history.determined_subframe_phase, _polarity(dec.determined_polarity)))
            raise
        if res is not None:
            parsed.append((res.receiver_timestamp, res.trailing_edge_receiver_timestamp, _given[n_given],
                           dec.history.determined_subframe_phase, _polarity(dec.determined_polarity)))
        return res

    dec.parse_subframe = parse_subframe
    rows, words = [], []
    stopped, processed = 0, 0
    for k, (b, a, c) in enumerate(zip(bits, t0, t1)):
        processed += 1
        n_parsed = len(parsed)
        try:
            evs = dec.process_bit_from_satellite(EmitNavigationBitEvent(float(a), float(c), BITVAL[int(b)]))
        except ValueError:
            ta, tb, given, ph, pol = parsed[-1]
            p = nmp.NavigationMessageSubframeParser(given)
            p.parse_telemetry_word()
            how = p.parse_handover_word()
            rows.append([k, nav.KIND_RAISED, how.subframe_id.value, nav.word_value(how.time_of_week),
                         -1 if ph is None else ph, pol, _parity_ok(given), ta, tb])
            words.append(_word_values(given))
            stopped = 1
            break
        emitted = iter(parsed[n_parsed:])
        for ev in evs:
            if isinstance(ev, nmd.EmitSubframeEvent):
                ta, tb, given, ph, pol = next(emitted)
                assert (ta, tb) == (ev.receiver_timestamp, ev.trailing_edge_receiver_timestamp)
                rows.append([k, nav.KIND_SUBFRAME, ev.handover_word.subframe_id.value,
                             nav.word_value(ev.handover_word.time_of_week), -1 if ph is None else ph, pol,
                             _parity_ok(given), ta, tb])
                words.append(_word_values(given))
            elif isinstance(ev, nmd.DeterminedSubframePhaseEvent):
                rows.append([k, nav.KIND_PHASE, 0, 0, ev.subframe_phase, _polarity(ev.polarity), 0, 0.0, 0.0])
                words.append((0,) * 10)
            else:
                assert isinstance(ev, nmd.CannotDetermineSubframePhaseEvent)
                rows.append([k, nav.KIND_CANNOT, 0, 0, -1, 0, 0, 0.0, 0.0])
                words.append((0,) * 10)
    h = dec.history
    final = [-1 if h.determined_subframe_phase is None else h.determined_subframe_phase, h.emitted_subframe_count,
             _polarity(dec.determined_polarity), len(dec.queued_bit_events), stopped, processed]
    return (np.array(rows, dtype=np.float64).reshape(-1, 9), np.array(words, dtype=np.int64).reshape(-1, 10),
            np.array(final, dtype=np.int64))


def _concat(subframes):
    return np.array([b for sf in subframes for b in sf], dtype=np.int8)


def streams():
    s = {}
    # (a) clean LNAV, 6 frames, the recording starting 137 bits into a subframe
    s["clean"] = _concat(nav.lnav_frames(1, 30))[137:]
    # (b) the same, negated: found with the inverted preamble
    s["negated"] = 1 - s["clean"]
    # (c) starting on a subframe boundary with an unknown bit in the first subframe: the first drain (two subframes)
    # resets on it and still parses the second subframe with no polarity; two more unknown bits later on reset the
    # steady state and force a re-sync
    c = _concat(nav.lnav_frames(3, 25))
    c[100] = -1
    c[300 * 14 + 57: 300 * 14 + 59] = -1
    s["unknown"] = c
    # (d) a corrupted TLM prelude in subframe 8, invalid HOW subframe ids (6 in subframe 16, 0 in subframe 20)
    sf = nav.lnav_frames(4, 25)
    sf[8][3] ^= 1
    for k, bad in ((16, (1, 1, 0)), (20, (0, 0, 0))):
        d30 = sf[k][29]  # the id bits go out complemented by word 1's D30
        sf[k][49:52] = [v ^ d30 for v in bad]
    s["bad_tlm_how"] = _concat(sf)[50:]
    # (e) the preamble planted in the data of the first two subframes, 300 bits apart and ahead of the real one (the
    # first candidate with a partner wins), a lone upright copy in subframe 10 and an inverted one in subframe 12
    sf = nav.lnav_frames(5, 25)
    for k, at, pat in ((0, 150, nav.PREAMBLE), (1, 150, nav.PREAMBLE), (10, 215, nav.PREAMBLE),
                       (12, 65, tuple(1 - v for v in nav.PREAMBLE))):
        sf[k][at: at + 8] = pat
    s["false_pair"] = _concat(sf)[100:]
    # (f) 3700 bits without any preamble, then LNAV: CannotDetermine on every bit from 3600 queued, then a phase of 3700
    # of which only 3700 % 300 bits are dropped; 4090 bits stay within the device queue
    s["no_preamble"] = np.concatenate([nav.no_preamble_noise(6, 3700), _concat(nav.lnav_frames(6, 2))[:390]])
    # (g) subframe 4, then a subframe 5 with data id 00 in the first drain: the reference raises
    s["raise"] = _concat(nav.lnav_frames(7, 6, first_id=4, sf5_data_id=lambda k: 0 if k == 1 else 1))
    # (h) a flipped data bit (subframe 5, word 4) and a flipped D30 (subframe 9, word 5: words 5 and 6 fail parity)
    sf = nav.lnav_frames(8, 25)
    sf[5][30 * 3 + 9] ^= 1
    sf[9][30 * 4 + 29] ^= 1
    s["parity"] = _concat(sf)[10:]
    return s


def main():
    out = {}
    for name, bits in streams().items():
        t0, t1 = nav.bit_times(bits.size)
        rows, words, final = run(bits, t0, t1)
        out[f"{name}_bits"], out[f"{name}_t0"], out[f"{name}_t1"] = bits.astype(np.int8), t0, t1
        out[f"{name}_events"], out[f"{name}_words"], out[f"{name}_final"] = rows, words, final
        kinds = np.bincount(rows[:, 1].astype(int), minlength=4) if rows.size else np.zeros(4, int)
        print(f"{name:12s} bits {bits.size:5d} kinds {list(kinds)} final {list(final)}")
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
