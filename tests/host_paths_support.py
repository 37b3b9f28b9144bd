"""The host-to-host paths' rules, restated only to choose test shapes (as acq_support.fused_choice does for the cell kernels),
and the shapes the GPU tests run at each of their edges: which branch a gb200_acquire_grid_host call takes, where its
records go, and which slot of a grid stream a submit uses."""
from acq_support import DEFAULT_SPEC_BUDGET_MB

EAGER_SRC_BYTES = 64 << 10  # pinned inputs above this are copied from the caller's buffer, eagerly, on every call
DIRECT_RECORD_BYTES = 256 << 10  # record sets up to this are stored by the kernel into mapped pinned memory
RECORD_BYTES = 32
NC, CO = "non_coherent", "coherent"


def spec_bytes(s, nb, m, d):
    """The spectra scratch a grid needs in one batch: unit_floats2 (M * S * 2 * 1024 float2) per (block, Doppler)."""
    return m * s * 2 * 1024 * 8 * d * nb


def iq_bytes(s, nb, m):
    return nb * m * 1023 * s * 8


def host_branch(s, nb, m, d, pinned_in, call, budget_mb=DEFAULT_SPEC_BUDGET_MB, timing=False):
    """gb200_acquire_grid_host's branch on the call-th call (0-based) of a shape: "plain" (upload + gb200_acquire_grid) with
    kernel timing on or a grid over the scratch budget; else "eager_src" for a pinned input over 64 KB, copied from the
    caller's buffer and run eagerly every time; else "eager" on the first call, "capture" on the second and "replay" after."""
    if timing or spec_bytes(s, nb, m, d) > budget_mb << 20:
        return "plain"
    if pinned_in and iq_bytes(s, nb, m) > EAGER_SRC_BYTES:
        return "eager_src"
    return ("eager", "capture", "replay")[min(call, 2)]


def records_direct(nb, p, d):
    """Whether the correlate kernel stores the records straight into pinned memory (no device-to-host copy node)."""
    return nb * p * d * RECORD_BYTES <= DIRECT_RECORD_BYTES


def records_to_caller(nb, p, d, pinned_out):
    """Whether it stores them into the caller's own (pinned) buffer, with no host copy after the call."""
    return records_direct(nb, p, d) and pinned_out


def stream_slots(depth, pinned):
    """[(slot, staged in, staged out)] of successive gb200_grid_stream_submit calls: batch k uses slot k % depth, and stages
    its input and its records through the slot's pinned buffers when the caller's are pageable.  pinned: [(in, out)]."""
    return [(k % depth, not pi, not po) for k, (pi, po) in enumerate(pinned)]


# gb200_acquire_grid_host shapes: (name, S, n_blocks, M, kind, P, D, pinned in, pinned out).  Each sits on one side of an
# edge: 8 ms at S = 1 and 4 ms at S = 2 are the largest inputs that stage (65 472 B), 9 and 5 ms the smallest that do not;
# 32 x 256 records are the largest set stored directly (262 144 B), 32 x 257 the smallest that is copied.
HOST_CASES = [
    ("s1_8ms_staged", 1, 8, 1, NC, 3, 5, True, True),
    ("s1_9ms_eager_src", 1, 9, 1, NC, 3, 5, True, False),
    ("s2_4ms_staged", 2, 2, 2, CO, 3, 4, True, False),
    ("s2_5ms_eager_src", 2, 5, 1, NC, 3, 4, True, True),
    ("s2_d256_to_caller", 2, 1, 1, NC, 32, 256, False, True),
    ("s2_d256_direct_pageable", 2, 1, 1, NC, 32, 256, True, False),
    ("s2_d257_pinned_out", 2, 1, 1, NC, 32, 257, False, True),
    ("s2_d257_pageable", 2, 1, 1, NC, 32, 257, False, False),
    ("s5_nc3_pageable", 5, 2, 3, NC, 3, 5, False, False),
    ("s5_nc3_eager_src", 5, 2, 3, NC, 3, 5, True, True),
    ("s16_co2_staged", 16, 1, 2, CO, 2, 3, False, True),
    ("s16_co2_eager_src", 16, 1, 2, CO, 2, 3, True, False),
]

# The 1 MB budget at S = 2, M = 1: D = 32 fills it exactly (graph path), D = 33 is one bin past it (plain path).
BUDGET_MB = 1
BUDGET_D = (32, 33)

# gb200_grid_stream shapes: (depth, S, n_blocks, M, kind, P, D).  Batch k's input is pinned when k % 3 == 0 and its
# records when (k // depth) is even, so a slot's staged_out flips on every reuse; 2 * depth + 1 batches reuse every slot.
STREAM_CASES = [
    (1, 1, 2, 1, NC, 3, 4),
    (2, 2, 1, 2, CO, 3, 3),
    (3, 5, 2, 3, NC, 2, 3),
    (8, 16, 1, 1, NC, 2, 3),
    (8, 2, 2, 3, NC, 3, 3),
    (3, 1, 1, 2, CO, 2, 3),
]


def stream_pinning(depth):
    """[(pinned in, pinned out)] of the 2 * depth + 1 batches of a STREAM_CASES run."""
    return [(k % 3 == 0, (k // depth) % 2 == 0) for k in range(2 * depth + 1)]


# The device ring: capacity 7 and appends of 1, 7, 3, 6, 3, 7, 1 ms.  The 7-ms appends start at slots 1 and 6 (the second
# wraps), the 6-ms one at slot 4 wraps; sources alternate pageable / pinned.
RING_CAPACITY = 7
RING_APPENDS = [1, 7, 3, 6, 3, 7, 1]


def ring_runs(capacity, appended, n_ms):
    """gb200_ring_append's copy runs: [(first slot, milliseconds)], at most two, wrapping at capacity."""
    runs, done = [], 0
    while done < n_ms:
        slot = (appended + done) % capacity
        run = min(n_ms - done, capacity - slot)
        runs.append((slot, run))
        done += run
    return runs
