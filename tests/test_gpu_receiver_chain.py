"""The tracker's call chain process -> integrate_bits -> decode_subframes -> parse_subframes -> observations /
position_fixes: what each call needs from the calls before it, and what it leaves on the device for the calls after it
(include/gypsum_b200.h).  Small inputs: two channels, tens of milliseconds of synthetic IQ, hand-made device arrays."""
import ctypes as C

import numpy as np
import pytest

from gpu_support import make_engine

pytestmark = pytest.mark.gpu
N, FS = 2046, 2046000
CHUNK = 20  # milliseconds per process call
IQ_MS = 30  # milliseconds of IQ loaded: a process call of more fails at its launch


def _iq(n_ms):
    from gypsum_b200 import synth

    return synth.synth_tracking_iq(5, N, n_ms, FS, [(25, 1500.3, 0.0, 777, 0.3, 0.004), (7, -100.0, 0.0, 5, 1.0, 0.004)])


def _ts(n_ms=CHUNK):
    return np.round(np.arange(n_ms) * 0.001, 6)


@pytest.fixture(scope="module")
def engine(native_lib):
    e = make_engine(FS, N)
    yield e
    e.close()


@pytest.fixture
def trk(engine):
    from gypsum_b200 import _native

    engine.upload_iq(_iq(IQ_MS))
    t = _native.Tracker(engine, [24, 6], [1500.0, -100.0], [0.0, 0.0], [777, 5])
    yield t
    t.close()


def process(t, n_ms=CHUNK):
    return t.process(n_ms, _ts(n_ms))


def integrate(t, n_ms=CHUNK, records=None):
    return t.integrate_bits(n_ms, _ts(n_ms), _ts(n_ms) + 0.001, records)


def chain(t):
    """process -> integrate_bits -> decode_subframes over the tracker's own records."""
    process(t)
    integrate(t)
    t.decode_subframes()


def device(host):
    import torch

    return torch.from_numpy(np.ascontiguousarray(host).view(np.uint8).reshape(host.shape[0], -1)).cuda()


def zero_bits(n_bits):
    from gypsum_b200._native import BIT_DTYPE

    b = np.zeros((2, n_bits), dtype=BIT_DTYPE)
    b["receiver_timestamp"] = np.arange(n_bits) * 0.02
    b["trailing_edge_receiver_timestamp"] = np.arange(n_bits) * 0.02 + 0.02
    return device(b)


def parse_empty(t, n_ms, drop=-1):
    """parse_subframes over a caller's device array holding no events."""
    from gypsum_b200._native import SUBFRAME_DTYPE

    ev = device(np.zeros((2, 1), dtype=SUBFRAME_DTYPE))
    return t.parse_subframes(ev.data_ptr(), [0, 0], 1, np.zeros((2, 1), dtype=np.int32), [drop, -1], n_ms)


def no_records(n_ms=CHUNK):
    return pytest.raises(RuntimeError, match=f"no records of {n_ms} ms")


def no_bits():
    return pytest.raises(RuntimeError, match="no undecoded bit events")


def no_subframes():
    return pytest.raises(RuntimeError, match="no unparsed subframe events")


def no_parse():
    return pytest.raises(RuntimeError, match="no gb200_tracker_parse_subframes call yet")


def test_process_puts_its_records_on_the_chain(trk):
    with no_records():
        integrate(trk)
    process(trk)
    with no_records(10):
        integrate(trk, 10)
    integrate(trk)
    integrate(trk)  # the records stay for the next integrate call
    trk.decode_subframes()
    trk.parse_subframes()
    assert trk.observations().shape == (2, CHUNK)


def test_process_takes_everything_off_the_chain_before_its_launch(trk):
    chain(trk)
    with pytest.raises(ValueError, match="samples"):
        process(trk, IQ_MS + 10)
    with no_records():
        integrate(trk)
    with no_subframes():
        trk.parse_subframes()


def test_process_between_decode_and_parse_breaks_the_chain(trk):
    chain(trk)
    process(trk)
    with no_subframes():
        trk.parse_subframes()


def test_process_keeps_pending_bits(trk):
    process(trk)
    integrate(trk)
    process(trk)
    trk.decode_subframes()  # the bits are still pending, but no longer on the chain
    with no_subframes():
        trk.parse_subframes()


def test_process_channels_takes_everything_off_the_chain(trk):
    process(trk)
    trk.process_channels([0, 1], CHUNK, _ts())
    with no_records():
        integrate(trk)
    process(trk)
    integrate(trk)
    trk.process_channels([0, 1], CHUNK, _ts())
    trk.decode_subframes()  # pending bits stay pending
    with no_subframes():
        trk.parse_subframes()
    chain(trk)
    trk.process_channels([1], CHUNK, _ts())
    with no_subframes():
        trk.parse_subframes()


def test_process_device_changes_nothing(trk):
    import torch

    from gypsum_b200._native import TRACK_DTYPE

    out = torch.empty(2 * CHUNK * TRACK_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    ts = _ts()
    trk.process_device(CHUNK, ts, out.data_ptr())
    with no_records():
        integrate(trk)
    process(trk)
    trk.process_device(CHUNK, ts, out.data_ptr())
    integrate(trk)
    trk.process_device(CHUNK, ts, out.data_ptr())
    trk.decode_subframes()
    trk.process_device(CHUNK, ts, out.data_ptr())
    trk.parse_subframes()
    assert trk.observations().shape == (2, CHUNK)
    torch.cuda.synchronize()


def test_integrate_over_the_tracker_records(trk):
    chain(trk)
    integrate(trk)  # new bits on the chain: the subframes decoded before are off it
    with no_subframes():
        trk.parse_subframes()
    trk.decode_subframes()
    trk.parse_subframes()
    assert trk.observations().shape == (2, CHUNK)
    with no_subframes():  # a parse call consumes the subframes
        trk.parse_subframes()
    chain(trk)
    with no_records(10):  # a failed call changes nothing
        integrate(trk, 10)
    trk.parse_subframes()


def test_integrate_over_caller_records(trk):
    recs = device(process(trk))
    integrate(trk, records=recs.data_ptr())
    trk.decode_subframes()  # the bits were pending, but off the chain
    with no_subframes():
        trk.parse_subframes()
    chain(trk)
    integrate(trk, records=recs.data_ptr())
    with no_subframes():
        trk.parse_subframes()
    integrate(trk)  # the tracker's records are still on the chain
    trk.decode_subframes()
    trk.parse_subframes()


def test_decode_needs_pending_bits_that_fit(engine, trk):
    from gypsum_b200 import _native

    with no_bits():
        trk.decode_subframes()
    # hand-made records whose bit events do not all fit the integrate call's stride of 1
    rec = np.zeros((2, 400), dtype=_native.TRACK_DTYPE)
    rec["symbol"] = 1
    dev = device(rec)
    ts = np.arange(400) * 0.001
    ev = np.empty((2, 1), dtype=_native.BIT_DTYPE)
    cnt = np.empty(2, dtype=np.int32)
    rc = engine._lib.gb200_tracker_integrate_bits(trk._h, 400, ts.ctypes.data, (ts + 0.001).ctypes.data,
                                                  C.c_void_p(dev.data_ptr()), ev.ctypes.data, 1, cnt.ctypes.data)
    assert rc == _native.OK and (cnt > 1).all()
    with pytest.raises(ValueError, match="kept 1"):
        trk.decode_subframes()
    with pytest.raises(ValueError, match="kept 1"):  # the failed call left the bits pending
        trk.decode_subframes()
    trk.integrate_bits(400, ts, ts + 0.001, dev.data_ptr())
    trk.decode_subframes()
    with no_bits():
        trk.decode_subframes()


def test_explicit_decode_keeps_the_bits_and_takes_the_subframes_off_the_chain(trk):
    bits = zero_bits(50)
    process(trk)
    integrate(trk)
    trk.decode_subframes(bits.data_ptr(), [50, 50], 50)
    trk.decode_subframes()  # the chain's bits were still pending, and still on the chain
    trk.parse_subframes()
    chain(trk)
    trk.decode_subframes(bits.data_ptr(), [50, 50], 50)
    with no_subframes():
        trk.parse_subframes()
    with no_bits():
        trk.decode_subframes()
    chain(trk)
    with pytest.raises(ValueError, match="51 bit events do not fit a stride of 50"):
        trk.decode_subframes(bits.data_ptr(), [51, 0], 50)
    trk.parse_subframes()  # the failed call changed nothing


def test_parse_checks_the_replica_rows_first(engine):
    from gypsum_b200 import _native
    from gypsum_b200._native import SUBFRAME_DTYPE

    t = _native.Tracker(engine, [4, 4], [0.0, 0.0], [0.0, 0.0], [0, 0])
    with pytest.raises(ValueError, match="same replica row"):
        t.parse_subframes()  # before the missing chain
    ev = device(np.zeros((2, 1), dtype=SUBFRAME_DTYPE))
    with pytest.raises(ValueError, match="same replica row"):  # before the explicit arguments
        t.parse_subframes(ev.data_ptr(), [5, 0], 1, np.zeros((2, 1), dtype=np.int32), [-1, -1], 10)
    t.close()


def test_parse_needs_chain_counts_that_fit(engine):
    from gypsum_b200 import _native

    engine.upload_iq(_iq(200))
    t = _native.Tracker(engine, [24, 6], [1500.0, -100.0], [0.0, 0.0], [777, 5])
    # 3599 queued bits without a preamble pair: every further bit is a CannotDetermine event
    t.decode_subframes(zero_bits(3599).data_ptr(), [3599, 3599], 3599)
    assert t.subframe_state(0)["queued_bit_count"] == 3599
    process(t, 200)
    assert max(len(b) for b in integrate(t, 200)) > 1
    ev = np.empty((2, 1), dtype=_native.SUBFRAME_DTYPE)
    cnt = np.empty(2, dtype=np.int32)
    rc = engine._lib.gb200_tracker_decode_subframes(t._h, None, None, 0, ev.ctypes.data, 1, cnt.ctypes.data)
    assert rc == _native.OK and (cnt > 1).any()
    with pytest.raises(ValueError, match="kept 1"):
        t.parse_subframes()
    t.close()


def test_explicit_parse_leaves_the_chain(trk):
    chain(trk)
    parse_empty(trk, 7)
    assert trk.observations().shape == (2, 7)
    trk.parse_subframes()
    assert trk.observations().shape == (2, CHUNK)
    chain(trk)
    with pytest.raises(ValueError, match="drop millisecond"):
        parse_empty(trk, 7, drop=7)
    trk.parse_subframes()  # the failed call changed nothing


def test_observations_need_a_parse_call(trk):
    import torch

    out = torch.empty(64, dtype=torch.uint8, device="cuda")
    with no_parse():
        trk.observations()
    with no_parse():
        trk.observations_device(out.data_ptr())


def test_fix_rules(engine, trk):
    import torch

    from gypsum_b200 import _native

    out = torch.empty(10 * _native.FIX_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    host = np.empty(10, dtype=_native.FIX_DTYPE)
    lib = engine._lib
    assert lib.gb200_tracker_position_fixes(trk._h, None, host.ctypes.data) == _native.EINVAL  # before the parse check
    assert b"null receiver timestamps" in lib.gb200_last_error(engine._h)
    with no_parse():
        trk.position_fixes([])
    with no_parse():
        trk.position_fixes_device([], out.data_ptr())
    ts = _ts(10)
    parse_empty(trk, 10)
    assert lib.gb200_tracker_position_fixes(trk._h, None, host.ctypes.data) == _native.EINVAL
    parse_empty(trk, 10)  # no fix call has run yet: no gap
    assert (trk.position_fixes(ts)["status"] == _native.FIX_NONE).all()
    assert trk.receiver_state() == {"slide": None, "stopped": False, "order": [], "repaired": 0}
    with pytest.raises(RuntimeError, match="already computed"):
        trk.position_fixes(ts)
    with pytest.raises(RuntimeError, match="already computed"):
        trk.position_fixes_device(ts, out.data_ptr())
    parse_empty(trk, 10)
    trk.position_fixes_device(ts, out.data_ptr())
    torch.cuda.synchronize()
    parse_empty(trk, 10)
    parse_empty(trk, 10)  # the fixes of the call before were skipped
    with pytest.raises(RuntimeError, match="gap"):
        trk.position_fixes(ts)
    with pytest.raises(RuntimeError, match="gap"):
        trk.position_fixes_device(ts, out.data_ptr())
    parse_empty(trk, 10)
    with pytest.raises(RuntimeError, match="gap"):  # for the tracker's lifetime
        trk.position_fixes(ts)


def test_fixes_follow_the_chain_parse(trk):
    chain(trk)
    trk.parse_subframes()
    fixes = trk.position_fixes(_ts())
    assert fixes.shape == (CHUNK,)
    with pytest.raises(ValueError, match="one start time per millisecond"):
        trk.position_fixes(_ts(10))
