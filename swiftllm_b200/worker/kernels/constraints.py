"""Constrained decoding: allowed-token bitmasks and logit bias applied to the logits before penalties and the token choice (new:
the reference has no sampling controls).  csrc/constraints.cu."""
import torch

from swiftllm_b200 import _lib


def constrain_logits(
    logits: torch.Tensor,               # [rows, vocab_size] (or this rank's vocabulary shard), fp16 / bf16, unit column stride
    mask_index: torch.Tensor,           # [rows] int32: row of `masks`, -1 = no mask
    masks: torch.Tensor,                # [num_masks, W] int32 bit words of global ids (bit v % 32 of word v // 32 = v allowed)
    bias_index: torch.Tensor,           # [rows] int32: bias entry, -1 = no bias
    bias_starts: torch.Tensor,          # [num_entries + 1] int32 CSR row starts into bias_ids / bias_values
    bias_ids: torch.Tensor,             # [num_bias] int32 global ids, ascending within an entry
    bias_values: torch.Tensor,          # [num_bias] float32
    vocab_offset: int = 0,
):
    """Masks and biases `logits` in place: disallowed ids become -inf, then allowed biased ids round(l + b)."""
    assert logits.dim() == 2 and logits.stride(1) == 1
    B, V = logits.shape
    for t in (mask_index, bias_index):
        assert t.dtype == torch.int32 and t.shape == (B,) and t.is_contiguous()
    assert masks.dtype == torch.int32 and masks.dim() == 2 and masks.is_contiguous()
    for t in (bias_starts, bias_ids):
        assert t.dtype == torch.int32 and t.dim() == 1 and t.is_contiguous()
    assert bias_values.dtype == torch.float32 and bias_values.shape == bias_ids.shape and bias_values.is_contiguous()
    _lib.require_device(logits)
    _lib.check(_lib.lib().sllm_constrain_logits(
        logits.data_ptr(), B, V, logits.stride(0) if B > 1 else V, vocab_offset, mask_index.data_ptr(), _lib.ptr(masks),
        masks.shape[0], masks.shape[1], bias_index.data_ptr(), _lib.ptr(bias_starts), max(bias_starts.shape[0] - 1, 0),
        _lib.ptr(bias_ids), _lib.ptr(bias_values), bias_ids.shape[0], _lib.dtype_tag(logits.dtype), _lib.stream()),
        "constrain_logits")
