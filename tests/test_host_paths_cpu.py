"""The host-to-host paths' rules, without a GPU (restated in host_paths_support): every shape tests/test_gpu_host_paths.py
runs lands on the edge it is named for -- staged vs copied from the caller's pinned buffer, records stored directly vs
copied, graph path vs plain path under a 1 MB budget -- and the grid stream's slots and staging, and the ring's copy runs,
are the ones its cases mean to exercise."""
import pytest

from host_paths_support import (BUDGET_D, BUDGET_MB, CO, HOST_CASES, NC, RING_APPENDS, RING_CAPACITY, STREAM_CASES,
                                host_branch, iq_bytes, records_direct, records_to_caller, ring_runs, spec_bytes,
                                stream_pinning, stream_slots)


def test_input_staging_edges():
    """8 ms at S = 1 and 4 ms at S = 2 are 65 472 B and stage; 9 ms and 5 ms go eager_src when pinned.  Pageable inputs
    always stage, and the call index then walks eager, capture, replay, replay."""
    assert iq_bytes(1, 8, 1) == iq_bytes(2, 4, 1) == iq_bytes(2, 2, 2) == 65472
    for s, ms_in, ms_out in ((1, 8, 9), (2, 4, 5)):
        assert iq_bytes(s, ms_in, 1) <= 65536 < iq_bytes(s, ms_out, 1)
        assert [host_branch(s, ms_in, 1, 5, True, k) for k in range(4)] == ["eager", "capture", "replay", "replay"]
        assert [host_branch(s, ms_out, 1, 5, True, k) for k in range(4)] == ["eager_src"] * 4
        assert host_branch(s, ms_out, 1, 5, False, 3) == "replay"


def test_record_edges():
    """32 x 256 records are 262 144 B and go straight into pinned memory; 32 x 257 are copied out of the device."""
    assert 32 * 256 * 32 == 262144
    assert records_direct(1, 32, 256) and not records_direct(1, 32, 257)
    assert records_to_caller(1, 32, 256, True) and not records_to_caller(1, 32, 256, False)
    assert not records_to_caller(1, 32, 257, True)


def test_budget_edge():
    """Under a 1 MB budget at S = 2, M = 1, D = 32 fills it exactly and takes the graph path; D = 33 takes the plain path
    on every call, and so does any call with kernel timing on."""
    lo, hi = BUDGET_D
    assert spec_bytes(2, 1, 1, lo) == BUDGET_MB << 20 < spec_bytes(2, 1, 1, hi)
    assert [host_branch(2, 1, 1, lo, False, k, BUDGET_MB) for k in range(3)] == ["eager", "capture", "replay"]
    assert [host_branch(2, 1, 1, hi, False, k, BUDGET_MB) for k in range(3)] == ["plain"] * 3
    assert host_branch(2, 1, 1, lo, False, 2, timing=True) == "plain"
    # the default budget holds every shape of the GPU tests
    for _, s, nb, m, _, _, d, pin_in, _ in HOST_CASES:
        assert host_branch(s, nb, m, d, pin_in, 0) != "plain"


@pytest.mark.parametrize("case", HOST_CASES, ids=[c[0] for c in HOST_CASES])
def test_host_case_lands_on_its_edge(case):
    """Each host-call shape of the GPU tests takes the branch and the record path its name says."""
    name, s, nb, m, kind, p, d, pin_in, pin_out = case
    assert kind in (NC, CO)
    branches = [host_branch(s, nb, m, d, pin_in, k) for k in range(4)]
    want = ["eager_src"] * 4 if "eager_src" in name else ["eager", "capture", "replay", "replay"]
    assert branches == want, name
    if "eager_src" in name:  # on the far side of the 64 KB edge, by at most one millisecond when the case is named for it
        assert iq_bytes(s, nb, m) > 65536
    elif pin_in:
        assert iq_bytes(s, nb, m) <= 65536
    if "d256" in name:
        assert records_direct(nb, p, d) and nb * p * d * 32 == 262144
        assert records_to_caller(nb, p, d, pin_out) == ("to_caller" in name)
    if "d257" in name:
        assert not records_direct(nb, p, d) and not records_to_caller(nb, p, d, pin_out)
    if name.startswith("s1_8ms") or name.startswith("s2_4ms"):
        assert iq_bytes(s, nb, m) == 65472
    if name.startswith("s1_9ms") or name.startswith("s2_5ms"):
        assert iq_bytes(s, nb, m) - iq_bytes(s, 1, 1) == 65472


def test_host_cases_cover_the_matrix():
    """Both sides of both edges, every input / output pinning, the three kinds and S = 1, 2, 5 and 16."""
    assert {(c[4], c[3]) for c in HOST_CASES} == {(NC, 1), (NC, 3), (CO, 2)}
    assert all(c[2] == 2 for c in HOST_CASES if c[3] == 3)  # non-coherent M = 3 over two blocks
    assert {c[1] for c in HOST_CASES} == {1, 2, 5, 16}
    assert {(c[7], c[8]) for c in HOST_CASES} == {(False, False), (False, True), (True, False), (True, True)}
    paths = {(host_branch(c[1], c[2], c[3], c[6], c[7], 0), records_direct(c[2], c[5], c[6]),
              records_to_caller(c[2], c[5], c[6], c[8])) for c in HOST_CASES}
    assert {("eager", True, True), ("eager", True, False), ("eager", False, False), ("eager_src", True, True),
            ("eager_src", True, False)} <= paths


@pytest.mark.parametrize("case", STREAM_CASES, ids=[f"d{c[0]}_s{c[1]}_{c[4]}_m{c[3]}" for c in STREAM_CASES])
def test_stream_slots_flip_staging(case):
    """Every slot is used at least twice, and its staged_out flips between consecutive uses; inputs mix pinned and
    pageable within every run."""
    depth = case[0]
    slots = stream_slots(depth, stream_pinning(depth))
    uses = {}
    for slot, staged_in, staged_out in slots:
        uses.setdefault(slot, []).append((staged_in, staged_out))
    assert sorted(uses) == list(range(depth))
    for slot, u in uses.items():
        assert len(u) >= 2
        assert all(a[1] != b[1] for a, b in zip(u, u[1:])), slot
    assert {si for _, si, _ in slots} == {True, False}


def test_stream_cases_cover_the_matrix():
    assert {c[0] for c in STREAM_CASES} == {1, 2, 3, 8}
    assert {c[1] for c in STREAM_CASES} == {1, 2, 5, 16}
    assert {(c[4], c[3]) for c in STREAM_CASES} >= {(NC, 1), (NC, 3), (CO, 2)}


def test_ring_appends_hit_every_edge():
    """Appends of 1, 3, 6 and 7 ms; the 6-ms append and one 7-ms append wrap (two copy runs); full-capacity appends start
    at slots 1 and 6."""
    appended, runs = 0, []
    for n_ms in RING_APPENDS:
        runs.append((appended % RING_CAPACITY, n_ms, ring_runs(RING_CAPACITY, appended, n_ms)))
        appended += n_ms
    assert {n for _, n, _ in runs} == {1, 3, 6, 7}
    assert {slot for slot, n, _ in runs if n == RING_CAPACITY} == {1, 6}
    assert any(n == 6 and len(r) == 2 for _, n, r in runs)
    assert any(n == RING_CAPACITY and len(r) == 2 for _, n, r in runs)
    for slot, n, r in runs:
        assert sum(k for _, k in r) == n and r[0][0] == slot and len(r) <= 2
