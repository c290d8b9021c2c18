"""TEST INFRASTRUCTURE: the host-side cluster geometry of the vocabulary-row kernels (csrc/vocab_select.cuh: slice_of,
slice_fits, cluster_geometry), restated so that tests can pick the batch sizes that run each cluster size C and name their cases
by it.  tests/test_vocab_geometry_cpu.py reads the constants below back from the sources and fails when they drift.

    slice_of(V, c, align)   entries per CTA: ceil(V / c) rounded up to a multiple of `align`;
    slice_fits              slice_of(V, c, align) * bytes_per_entry <= MAX_SLICE_BYTES;
    cluster_geometry        the smallest c (1, 2, 4, 8) whose slice fits, then doubled while rows * c * 2 <= SM_TARGET.

With c = 1 fitting, batches of 1-16 rows run C = 8, 17-33 rows C = 4, 34-66 rows C = 2 and 67 or more C = 1."""
from __future__ import annotations

MAX_CLUSTER = 8
MAX_SLICE_BYTES = 200 * 1024
SM_TARGET = 132                                  # the `132` of cluster_geometry: rows * C * 2 <= 132 doubles C

# (bytes per entry, slice alignment in entries) of each kernel's shared-memory slice
KEYS = (2, 8)                                    # sampling.cu, logprobs.cu: uint16 keys, slices of whole uint4 vectors
SLOTS = (4, 4)                                   # penalties.cu: uint32 slots, zeroed as whole uint4 vectors
ENTRY = {"sampling": KEYS, "logprobs": KEYS, "penalties": SLOTS}

# prompt_logprobs.cu: keys staged in shared memory before the rest of the row is streamed, and the top-N candidate buffer
STAGE_KEYS = 48 * 1024
MAX_CAND = 1024

# one batch size per cluster size when c = 1 fits (see the module docstring); cluster_geometry decides, this only proposes
BATCHES = (12, 24, 40, 67)


def slice_of(V: int, c: int, align: int) -> int:
    return ((V + c - 1) // c + align - 1) // align * align


def slice_fits(V: int, c: int, bytes_per_entry: int, align: int) -> bool:
    return slice_of(V, c, align) * bytes_per_entry <= MAX_SLICE_BYTES


def cluster_geometry(rows: int, V: int, bytes_per_entry: int, align: int) -> tuple:
    """(C, slice) of a launch of `rows` rows of V entries; the C ABI refuses V where slice_fits(V, MAX_CLUSTER, ...) fails."""
    c = 1
    while c < MAX_CLUSTER and not slice_fits(V, c, bytes_per_entry, align):
        c *= 2
    while c < MAX_CLUSTER and rows * c * 2 <= SM_TARGET:
        c *= 2
    return c, slice_of(V, c, align)


def accepted(V: int, bytes_per_entry: int, align: int) -> bool:
    return V > 0 and slice_fits(V, MAX_CLUSTER, bytes_per_entry, align)


def smallest_cluster(V: int, bytes_per_entry: int, align: int) -> int:
    """The C of a large batch: the smallest cluster whose slice fits."""
    return cluster_geometry(1 << 20, V, bytes_per_entry, align)[0]


def batch_for(C: int, V: int, bytes_per_entry: int, align: int):
    """A batch size (from BATCHES) whose launch runs clusters of C CTAs at V, or None when V does not allow C."""
    for b in BATCHES:
        if cluster_geometry(b, V, bytes_per_entry, align)[0] == C:
            return b
    return None


def cta_ranges(V: int, C: int, align: int) -> list:
    """[begin, end) of each CTA's slice of the row (empty ranges for CTAs past the end)."""
    s = slice_of(V, C, align)
    return [(min(V, k * s), min(V, (k + 1) * s)) for k in range(C)]
