"""Repetition / frequency / presence penalties over the device-resident token history (new: the reference has no sampling
controls).  csrc/penalties.cu."""
import torch

from swiftllm_b200 import _lib


def apply_penalties(
    logits: torch.Tensor,               # [batch_size, vocab_size] (or this rank's vocabulary shard), fp16 / bf16, unit column stride
    repetition_penalty: torch.Tensor,   # [batch_size] float32; 1: off
    frequency_penalty: torch.Tensor,    # [batch_size] float32; 0: off
    presence_penalty: torch.Tensor,     # [batch_size] float32; 0: off (a row with all three off is left alone, nothing recorded)
    pos: torch.Tensor,                  # [batch_size] int32, sequence length after this step's input
    seq_ids: torch.Tensor,              # [batch_size] int32 block-table rows
    input_ids: torch.Tensor,            # [num_tokens] int32, the step's input tokens (prefill entries first)
    last_token_indices: torch.Tensor,   # [batch_size] int32, each entry's last input token
    prefill_seq_lens: torch.Tensor,     # [num_prefill_rows] int32, new tokens of each prefill entry
    num_prefill_rows: int,
    block_table: torch.Tensor,          # int32 [max_seqs, max_blocks_per_seq]
    token_cache: torch.Tensor,          # int32 [num_blocks, block_size], id | is_output << 31; the step's tokens are written here
    vocab_offset: int = 0,
):
    """Penalises `logits` in place and records the step's tokens of the penalised rows in `token_cache`."""
    assert logits.dim() == 2 and logits.stride(1) == 1
    B, V = logits.shape
    for t in (repetition_penalty, frequency_penalty, presence_penalty):
        assert t.dtype == torch.float32 and t.shape == (B,) and t.is_contiguous()
    for t in (pos, seq_ids, last_token_indices):
        assert t.dtype == torch.int32 and t.shape == (B,) and t.is_contiguous()
    assert input_ids.dtype == torch.int32 and input_ids.is_contiguous()
    assert prefill_seq_lens.dtype == torch.int32 and prefill_seq_lens.numel() >= num_prefill_rows
    assert block_table.dtype == torch.int32 and block_table.dim() == 2 and block_table.is_contiguous()
    assert token_cache.dtype == torch.int32 and token_cache.dim() == 2 and token_cache.is_contiguous()
    _lib.require_device(logits)
    _lib.check(_lib.lib().sllm_apply_penalties(
        logits.data_ptr(), B, V, logits.stride(0) if B > 1 else V, vocab_offset, repetition_penalty.data_ptr(),
        frequency_penalty.data_ptr(), presence_penalty.data_ptr(), seq_ids.data_ptr(), pos.data_ptr(), input_ids.data_ptr(),
        last_token_indices.data_ptr(), prefill_seq_lens.data_ptr() if num_prefill_rows else None, num_prefill_rows,
        block_table.data_ptr(), block_table.shape[1], token_cache.shape[1], token_cache.data_ptr(), token_cache.shape[0],
        _lib.dtype_tag(logits.dtype), _lib.stream()), "apply_penalties")
