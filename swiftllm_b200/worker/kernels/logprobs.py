"""Token log-probabilities and top-N alternatives (new: the reference returns token ids only).  csrc/logprobs.cu."""
import torch

from swiftllm_b200 import _lib


def token_logprobs(
    logits: torch.Tensor,           # [batch_size, vocab_size] fp16 / bf16, the whole vocabulary, unit column stride
    token_ids: torch.Tensor,        # [batch_size] int64
    top_n: int,                     # 0 .. 20
):
    """log_softmax of the raw logits: (logprob of token_ids fp32 [batch_size], top ids int32 [batch_size, top_n], their
    logprobs fp32 [batch_size, top_n]), the top entries ordered by (logit desc, id asc)."""
    assert logits.dim() == 2 and logits.stride(1) == 1
    B, V = logits.shape
    assert token_ids.dtype == torch.int64 and token_ids.shape == (B,) and token_ids.is_contiguous()
    _lib.require_device(logits)
    dev = logits.device
    token_lp = torch.empty((B,), dtype=torch.float32, device=dev)
    top_ids = torch.empty((B, top_n), dtype=torch.int32, device=dev)
    top_lp = torch.empty((B, top_n), dtype=torch.float32, device=dev)
    _lib.check(_lib.lib().sllm_token_logprobs(
        logits.data_ptr(), B, V, logits.stride(0) if B > 1 else V, token_ids.data_ptr(), top_n, token_lp.data_ptr(),
        top_ids.data_ptr() if top_n else None, top_lp.data_ptr() if top_n else None, _lib.dtype_tag(logits.dtype),
        _lib.stream()), "token_logprobs")
    return token_lp, top_ids, top_lp
