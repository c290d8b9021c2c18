"""Reference: swiftllm/worker/kernels/block_mgmt.py (:26-46, :66-80, :106-127) + the sync-free allocator that
replaces swiftllm/worker/block_manager.py:43-79."""
import torch

from swiftllm_b200 import _lib

# Largest batch sllm_allocate_blocks_for_seqs takes: its kernel keeps 2 * batch + 1 int32 in at most 200 KB of shared memory.
MAX_ALLOCATE_BATCH = (200 * 1024 // 4 - 1) // 2


def set_block_table_and_num_seq_alloc_blocks(
    num_seq_allocated_blocks: torch.Tensor,  # [max_seqs_in_block_table]
    block_table: torch.Tensor,               # [max_seqs_in_block_table, max_blocks_per_seq]
    candidate_blocks: torch.Tensor,          # [sum(block_needed)] int64
    seq_ids: torch.Tensor,                   # [batch_size]
    block_needed: torch.Tensor,              # [batch_size]
):
    _lib.require_device(block_table)
    assert candidate_blocks.dtype == torch.int64 and seq_ids.dtype == torch.int32
    block_needed = block_needed.to(torch.int32).contiguous()
    cumsum = torch.cumsum(block_needed, 0, dtype=torch.int32)
    _lib.check(_lib.lib().sllm_set_block_table_and_num_seq_alloc_blocks(
        num_seq_allocated_blocks.data_ptr(), block_table.data_ptr(), candidate_blocks.data_ptr(), seq_ids.data_ptr(),
        block_needed.data_ptr(), cumsum.data_ptr(), seq_ids.shape[0], block_table.shape[1], _lib.stream()),
        "set_block_table_and_num_seq_alloc_blocks")


def unset_block_table_and_num_seq_alloc_blocks(
    num_seq_allocated_blocks: torch.Tensor,
    block_table: torch.Tensor,
    seq_ids: torch.Tensor,
    is_block_free: torch.Tensor,             # [num_blocks], bool
):
    _lib.require_device(block_table)
    assert seq_ids.dtype == torch.int32 and is_block_free.dtype == torch.bool
    _lib.check(_lib.lib().sllm_unset_block_table_and_num_seq_alloc_blocks(
        num_seq_allocated_blocks.data_ptr(), block_table.data_ptr(), seq_ids.data_ptr(), is_block_free.data_ptr(),
        seq_ids.shape[0], block_table.shape[1], _lib.stream()), "unset_block_table_and_num_seq_alloc_blocks")


def gather_allocated_blocks_and_unset(
    num_seq_allocated_blocks: torch.Tensor,
    block_table: torch.Tensor,
    seq_ids: torch.Tensor,
    is_block_free: torch.Tensor,
    total_blocks: int = None,                # host-known total (avoids the reference's .item() sync, block_mgmt.py:118)
) -> torch.Tensor:
    if seq_ids.numel() == 0:
        return torch.empty((0,), dtype=torch.int32, device=block_table.device)
    _lib.require_device(block_table)
    cumsum = torch.cumsum(num_seq_allocated_blocks[seq_ids.long()], 0, dtype=torch.int32)
    if total_blocks is None:
        total_blocks = int(cumsum[-1].item())
    gathered = torch.empty((total_blocks,), dtype=torch.int32, device=block_table.device)
    _lib.check(_lib.lib().sllm_gather_allocated_blocks_and_unset(
        num_seq_allocated_blocks.data_ptr(), block_table.data_ptr(), seq_ids.data_ptr(), is_block_free.data_ptr(),
        cumsum.data_ptr(), gathered.data_ptr(), seq_ids.shape[0], block_table.shape[1], _lib.stream()),
        "gather_allocated_blocks_and_unset")
    return gathered


def truncate_blocks_for_seqs(
    num_seq_allocated_blocks: torch.Tensor,
    block_table: torch.Tensor,
    is_block_free: torch.Tensor,
    seq_ids: torch.Tensor,                   # [batch] int32, distinct
    target_lens: torch.Tensor,               # [batch] int32
    block_size: int,
):
    """Free the blocks past ceil(target_lens[i] / block_size) of every sequence (one launch, no host sync)."""
    _lib.require_device(block_table)
    assert seq_ids.dtype == torch.int32 and target_lens.dtype == torch.int32 and is_block_free.dtype == torch.bool
    _lib.check(_lib.lib().sllm_truncate_blocks_for_seqs(
        num_seq_allocated_blocks.data_ptr(), block_table.data_ptr(), is_block_free.data_ptr(), seq_ids.data_ptr(),
        target_lens.data_ptr(), seq_ids.shape[0], block_size, block_table.shape[1], _lib.stream()), "truncate_blocks_for_seqs")


def allocate_blocks_for_seqs(
    num_seq_allocated_blocks: torch.Tensor,
    block_table: torch.Tensor,
    is_block_free: torch.Tensor,
    seq_ids: torch.Tensor,                   # [batch] int32
    target_lens: torch.Tensor,               # [batch] int32
    block_size: int,
    new_blocks_out: torch.Tensor,            # int64 [>= number of new blocks] or None
    status_out: torch.Tensor,                # int32 [2]
):
    """One launch, no host sync: lowest-free-id-first allocation in batch order (bit-exact with the reference)."""
    _lib.require_device(block_table)
    assert seq_ids.dtype == torch.int32 and target_lens.dtype == torch.int32 and is_block_free.dtype == torch.bool
    _lib.check(_lib.lib().sllm_allocate_blocks_for_seqs(
        num_seq_allocated_blocks.data_ptr(), block_table.data_ptr(), is_block_free.data_ptr(), seq_ids.data_ptr(),
        target_lens.data_ptr(), seq_ids.shape[0], block_size, is_block_free.shape[0], block_table.shape[1],
        _lib.ptr(new_blocks_out), 0 if new_blocks_out is None else new_blocks_out.shape[0], status_out.data_ptr(),
        _lib.stream()), "allocate_blocks_for_seqs")


def fork_blocks_for_seqs(
    num_seq_allocated_blocks: torch.Tensor,
    block_table: torch.Tensor,
    block_extra_refs: torch.Tensor,          # [num_blocks] int32
    src_seq_ids: torch.Tensor,               # [batch] int32
    dst_seq_ids: torch.Tensor,               # [batch] int32, distinct, empty rows
    lens: torch.Tensor,                      # [batch] int32
    block_size: int,
):
    """dst row i <- the first lens[i] // block_size blocks of src row i, each gaining one extra owner (one launch, no host sync)."""
    _lib.require_device(block_table)
    assert src_seq_ids.dtype == dst_seq_ids.dtype == lens.dtype == block_extra_refs.dtype == torch.int32
    _lib.check(_lib.lib().sllm_fork_blocks_for_seqs(
        num_seq_allocated_blocks.data_ptr(), block_table.data_ptr(), block_extra_refs.data_ptr(), src_seq_ids.data_ptr(),
        dst_seq_ids.data_ptr(), lens.data_ptr(), src_seq_ids.shape[0], block_size, block_table.shape[1], _lib.stream()),
        "fork_blocks_for_seqs")


def copy_block_tails(
    k_cache: torch.Tensor,                   # [num_blocks, ...] (one block of every layer is contiguous)
    v_cache: torch.Tensor,
    token_cache: torch.Tensor,               # [num_blocks, block_size] int32 or None
    block_table: torch.Tensor,
    src_seq_ids: torch.Tensor,               # [batch] int32
    dst_seq_ids: torch.Tensor,               # [batch] int32
    lens: torch.Tensor,                      # [batch] int32
    block_size: int,
):
    """For every entry with lens[i] % block_size != 0: block lens[i] // block_size of src -> the same block index of dst (K, V
    and token pages; ids read from the block table on the device)."""
    _lib.require_device(k_cache)
    assert k_cache.is_contiguous() and v_cache.is_contiguous() and k_cache.shape == v_cache.shape
    assert src_seq_ids.dtype == dst_seq_ids.dtype == lens.dtype == torch.int32
    block_bytes = k_cache[0].numel() * k_cache.element_size()
    _lib.check(_lib.lib().sllm_copy_block_tails(
        k_cache.data_ptr(), v_cache.data_ptr(), _lib.ptr(token_cache), block_table.data_ptr(), src_seq_ids.data_ptr(),
        dst_seq_ids.data_ptr(), lens.data_ptr(), src_seq_ids.shape[0], block_bytes, block_size, block_table.shape[1],
        _lib.stream()), "copy_block_tails")


def release_blocks_for_seqs(
    num_seq_allocated_blocks: torch.Tensor,
    block_table: torch.Tensor,
    is_block_free: torch.Tensor,
    block_extra_refs: torch.Tensor,
    seq_ids: torch.Tensor,                   # [batch] int32
    total_blocks: int = None,                # host-known total of the gathered ids; None: no gather (a plain free)
):
    """Drop one owner of every block of the sequences; a block becomes free when its last owner lets go.  With total_blocks, also
    returns every block id of the sequences in batch order (int32), like gather_allocated_blocks_and_unset."""
    _lib.require_device(block_table)
    assert seq_ids.dtype == torch.int32 and is_block_free.dtype == torch.bool and block_extra_refs.dtype == torch.int32
    cumsum = gathered = None
    if total_blocks is not None:
        cumsum = torch.cumsum(num_seq_allocated_blocks[seq_ids.long()], 0, dtype=torch.int32)
        gathered = torch.empty((total_blocks,), dtype=torch.int32, device=block_table.device)
    _lib.check(_lib.lib().sllm_release_blocks_for_seqs(
        num_seq_allocated_blocks.data_ptr(), block_table.data_ptr(), is_block_free.data_ptr(), block_extra_refs.data_ptr(),
        seq_ids.data_ptr(), _lib.ptr(cumsum), _lib.ptr(gathered), seq_ids.shape[0], block_table.shape[1], _lib.stream()),
        "release_blocks_for_seqs")
    return gathered
