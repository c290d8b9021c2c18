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


def prompt_logprobs(
    logits: torch.Tensor,           # [rows, vocab_size] fp16 / bf16, the whole vocabulary, unit column stride
    target_ids: torch.Tensor,       # [rows] int32
    top_n: int,                     # 0 .. 20
    out=None,                       # optional (logprob fp32 [rows], rank int32 [rows], top ids int32 [rows, top_n], top lp fp32)
):
    """token_logprobs for many rows (csrc/prompt_logprobs.cu), with ranks: (logprob of target_ids fp32 [rows], rank int32 [rows]
    (1 + ids with a larger logit; -1 for an id outside [0, V)), top ids int32 [rows, top_n], their logprobs fp32 [rows, top_n]).
    The values are token_logprobs' bit for bit.  `out` receives the results in place (e.g. slices of larger buffers)."""
    assert logits.dim() == 2 and logits.stride(1) == 1
    R, V = logits.shape
    assert target_ids.dtype == torch.int32 and target_ids.shape == (R,) and target_ids.is_contiguous()
    _lib.require_device(logits)
    dev = logits.device
    if out is None:
        out = (torch.empty((R,), dtype=torch.float32, device=dev), torch.empty((R,), dtype=torch.int32, device=dev),
               torch.empty((R, top_n), dtype=torch.int32, device=dev), torch.empty((R, top_n), dtype=torch.float32, device=dev))
    lp, rank, top_ids, top_lp = out
    assert lp.shape == (R,) and rank.shape == (R,) and lp.is_contiguous() and rank.is_contiguous()
    assert top_ids.shape == (R, top_n) and top_lp.shape == (R, top_n) and top_ids.is_contiguous() and top_lp.is_contiguous()
    _lib.check(_lib.lib().sllm_prompt_logprobs(
        logits.data_ptr(), R, V, logits.stride(0) if R > 1 else V, target_ids.data_ptr(), top_n, lp.data_ptr(), rank.data_ptr(),
        top_ids.data_ptr() if top_n else None, top_lp.data_ptr() if top_n else None, _lib.dtype_tag(logits.dtype),
        _lib.stream()), "prompt_logprobs")
    return lp, rank, top_ids, top_lp
