"""TEST INFRASTRUCTURE: the launch geometry of the KV-cache and block-table kernels (csrc/kvcache.cu, csrc/swap_gather.cu,
csrc/rotary_store.cu) and of the launchers that size dynamic shared memory near 48 KB (csrc/exchange.cuh), restated so that
tests can pick shapes that run each regime and name their cases by it.  tests/test_kv_geometry_cpu.py holds this file to the
sources.

Every launcher with dynamic shared memory raises its kernel's limit through fit_dynamic_smem (csrc/common.cuh) once dynamic
plus static shared memory pass the 48 KB default; the static size is the compiled kernel's, which STATIC_SMEM states.
allocate_blocks_kernel (one CTA of ALLOC_THREADS threads) keeps start[batch + 1] and have[batch] in (2 * batch + 1) int32 of
dynamic shared memory.  Its launcher refuses more than ALLOC_SMEM_MAX bytes.  Step 1 scans the batch ALLOC_THREADS entries at a time; steps 2 and 3 walk the
free map ALLOC_WINDOW blocks at a time (16 per thread).
copy_block_tails_kernel moves one TAIL_CHUNK of a page per CTA.  swap_blocks_gather_kernel cuts each page into SW_SPLIT slices
of ceil(vecs / SW_SPLIT) 16-byte vectors; a thread moves vectors i and i + SW_THREADS of its slice per iteration."""
from __future__ import annotations

SMEM_DEFAULT = 48 * 1024              # shared memory (static + dynamic) a kernel may use without cudaFuncSetAttribute
# static shared memory of each kernel launched with dynamic shared memory that can cross 48 KB, as ptxas lays it out
# (rmsnorm_kernel<QUANT>: its quantizing instances)
STATIC_SMEM = {"allocate_blocks_kernel": 144,               # warp_sums[32], s_err
               "allreduce_add_rmsnorm_kernel": 64,          # red[16]
               "allreduce_add_rmsnorm_2shot_kernel": 80,    # red[16], s_last
               "allreduce_add_rmsnorm_ll_kernel": 64,       # red[16]
               "rmsnorm_kernel": 64,                        # red[16]
               "rmsnorm_kernel<QUANT>": 128,                # red[16], redmax[16]
               "silu_and_mul_quant_kernel": 64}             # redmax[16]

ALLOC_THREADS = 1024
ALLOC_WINDOW = ALLOC_THREADS * 16
ALLOC_SMEM_MAX = 200 * 1024
ALLOC_FLAGS = {"short": 1, "have>target": 2, "target>mbps": 4, "new_out small": 8}

TAIL_THREADS, TAIL_UNROLL = 256, 8
TAIL_CHUNK = TAIL_THREADS * TAIL_UNROLL * 16

SW_SPLIT, SW_THREADS = 8, 256

PREFILL_THREADS, DECODE_THREADS, ROTARY_STORE_THREADS = 256, 128, 256


def cdiv(a: int, b: int) -> int:
    return -(-a // b)


# ----------------------------------------------------------------------------- allocator
def alloc_smem(batch: int) -> int:
    return (2 * batch + 1) * 4


def alloc_needs_raise(batch: int) -> bool:
    """Whether the launch fails unless the limit is raised."""
    return alloc_smem(batch) + STATIC_SMEM["allocate_blocks_kernel"] > SMEM_DEFAULT


def alloc_band(batch: int) -> str:
    """'default' (fits the 48 KB default), 'raised' (the launcher raises the limit) or 'refused' (the launcher refuses)."""
    if alloc_smem(batch) > ALLOC_SMEM_MAX:
        return "refused"
    return "raised" if alloc_needs_raise(batch) else "default"


MAX_ALLOC_BATCH = max(b for b in range(1, 1 << 16) if alloc_band(b) != "refused")


def scan_passes(batch: int) -> int:
    """Passes of step 1's loop (its carry is added across passes)."""
    return max(1, cdiv(batch, ALLOC_THREADS))


def windows(ids) -> set:
    """ALLOC_WINDOW windows of step 3 that hold the given block ids."""
    return {int(i) // ALLOC_WINDOW for i in ids}


# ----------------------------------------------------------------------------- copies
def tail_chunks(block_bytes: int) -> int:
    return cdiv(block_bytes, TAIL_CHUNK)


def swap_slices(block_bytes: int) -> list:
    """Vectors of each of the SW_SPLIT slices of a page."""
    vecs = block_bytes // 16
    per = cdiv(vecs, SW_SPLIT)
    return [max(0, min(vecs, lo + per) - lo) for lo in range(0, per * SW_SPLIT, per)]


def swap_second_access(block_bytes: int) -> bool:
    """Whether some thread moves a second vector (i + SW_THREADS) in one iteration."""
    return max(swap_slices(block_bytes)) > SW_THREADS


# ----------------------------------------------------------------------------- stores
def prefill_grid(max_len: int, num_seqs: int, bs: int, chunked: bool) -> tuple:
    return (cdiv(max_len, bs) + (1 if chunked else 0), num_seqs)


def prefill_items(ntok: int, nkv: int, D: int) -> int:
    """16-byte items a prefill CTA moves for a page holding ntok tokens (each of its PREFILL_THREADS threads loops over them)."""
    return ntok * nkv * (D // 8)


def rotary_store_grid(num_seqs: int, nq: int, nkv: int, D: int) -> int:
    return cdiv(num_seqs * (nq + 2 * nkv) * (D // 16), ROTARY_STORE_THREADS)


# ----------------------------------------------------------------------------- exchange
def exchange_needs_raise(H: int, kernel: str) -> bool:
    return (H // 8) * 16 + STATIC_SMEM[kernel] > SMEM_DEFAULT


LL_MAX_HIDDEN = SMEM_DEFAULT // 16 * 8          # the LL launcher refuses a row of more than 48 KB


# ----------------------------------------------------------------------------- case tables
# Allocator batches: one and several warps, one to three scan passes, both sides of the 48 KB edge (6125 fits; 6126 ... 6143
# need the raised limit only because of the static 144 B; 6144 passes 48 KB on dynamic memory alone), and the largest batch.
ALLOC_BATCHES = (1, 31, 32, 33, 1023, 1024, 1025, 2049, 6125, 6126, 6143, 6144, 12287, 12288, MAX_ALLOC_BATCH)


def batch_id(batch: int) -> str:
    if alloc_band(batch) == "raised" and not alloc_smem(batch) > SMEM_DEFAULT:
        tag = "edge"
    elif alloc_band(batch) == "raised":
        tag = "raised"
    else:
        tag = f"{scan_passes(batch)}pass"
    return f"B{batch}-{tag}"


# Free maps: (num_blocks, pattern).  Patterns: 'all', 'odd' (every other block free), 'every16', 'past-window' (free only
# from ALLOC_WINDOW on), 'straddle' (runs of 100 free blocks across each window boundary, one free block in 7 elsewhere).
H100_BLOCKS = 500_000                 # about what an 80 GB H100 holds for an 8B model's cache at 16 tokens per block
FREE_MAPS = ((1, "all"), (15, "all"), (16, "all"), (17, "all"), (16383, "odd"), (16384, "every16"), (16385, "all"),
             (3 * ALLOC_WINDOW + 5, "odd"), (3 * ALLOC_WINDOW + 5, "every16"), (3 * ALLOC_WINDOW + 5, "past-window"),
             (3 * ALLOC_WINDOW + 5, "straddle"), (H100_BLOCKS, "straddle"), (H100_BLOCKS, "every16"))


def free_map_id(case) -> str:
    n, pattern = case
    return f"N{n}-{pattern}-W{cdiv(n, ALLOC_WINDOW)}-window"


# Pages of the copy kernels: (shape of one block [layers, nkv, bs, D] in 16-bit elements, id).
PAGES = (((32, 8, 16, 128), "P1MiB-32chunks"),        # Llama-3-8B: 32 layers x 8 kv heads x 16 x 128 x 2 B
         ((1, 1, 4099, 8), "P65584B-short-slice"),     # 4099 vectors: slices of 513, the last one 508
         ((1, 1, 13, 8), "P208B-short-slice"))         # 13 vectors: slices of 2, the last one 1, then an empty one

# Stores: block sizes and (nq, nkv, D) of real GQA groups
BLOCK_SIZES = (1, 8, 16, 32, 64, 128)
HEADS = ((4, 1, 64), (32, 8, 128), (64, 8, 128), (16, 2, 64))


def heads_id(h) -> str:
    return "q%d-kv%d-D%d" % h
