"""Token sampling (new: the reference decodes greedily, swiftllm/worker/layers/post_layer.py:39).  csrc/sampling.cu."""
from typing import Optional

import torch

from swiftllm_b200 import _lib


def sample_tokens(
    logits: torch.Tensor,           # [batch_size, vocab_size] (or this rank's vocabulary shard), fp16 / bf16, unit column stride
    temperature: torch.Tensor,      # [batch_size] float32; <= 0: greedy
    top_k: torch.Tensor,            # [batch_size] int32; 0: off
    top_p: torch.Tensor,            # [batch_size] float32; 1: off
    seed: torch.Tensor,             # [batch_size] int64
    pos: torch.Tensor,              # [batch_size] int32, sequence length after this step's input
    vocab_offset: int = 0,
    out_pairs: Optional[torch.Tensor] = None,   # [batch_size, 2] float32: (best score, global index) of this shard
    *,
    min_p: Optional[torch.Tensor] = None,           # [batch_size] float32; 0: off
    typical_p: Optional[torch.Tensor] = None,       # [batch_size] float32; 1: off
    xtc_threshold: Optional[torch.Tensor] = None,   # [batch_size] float32
    xtc_probability: Optional[torch.Tensor] = None,  # [batch_size] float32; 0: off
) -> torch.Tensor:
    """Global token ids, int64 [batch_size].  The four filter tensors (all or none) select sllm_sample_tokens_truncated."""
    assert logits.dim() == 2 and logits.stride(1) == 1
    B, V = logits.shape
    filters = (min_p, typical_p, xtc_threshold, xtc_probability)
    truncated = min_p is not None
    assert all((f is not None) == truncated for f in filters), "min_p, typical_p, xtc_threshold, xtc_probability: all or none"
    for t, dt in ((temperature, torch.float32), (top_k, torch.int32), (top_p, torch.float32), (seed, torch.int64),
                  (pos, torch.int32)) + (tuple((f, torch.float32) for f in filters) if truncated else ()):
        assert t.dtype == dt and t.shape == (B,) and t.is_contiguous()
    assert out_pairs is None or (out_pairs.dtype == torch.float32 and out_pairs.shape == (B, 2) and out_pairs.is_contiguous())
    _lib.require_device(logits)
    out = torch.empty((B,), dtype=torch.int64, device=logits.device)
    args = (logits.data_ptr(), B, V, logits.stride(0) if B > 1 else V, vocab_offset, temperature.data_ptr(), top_k.data_ptr(),
            top_p.data_ptr(), seed.data_ptr(), pos.data_ptr(), out.data_ptr(), _lib.ptr(out_pairs))
    if truncated:
        _lib.check(_lib.lib().sllm_sample_tokens_truncated(*args, *(f.data_ptr() for f in filters),
                                                           _lib.dtype_tag(logits.dtype), _lib.stream()), "sample_tokens")
    else:
        _lib.check(_lib.lib().sllm_sample_tokens(*args, _lib.dtype_tag(logits.dtype), _lib.stream()), "sample_tokens")
    return out
