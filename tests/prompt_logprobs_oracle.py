"""TEST INFRASTRUCTURE: numpy restatement of the prompt log-probability semantics (csrc/prompt_logprobs.cu,
LlamaModel.forward_with_logprobs with SamplingParams.prompt_logprobs).  The values are those of tests/logprobs_oracle.py; this
module adds the rank and the construction of the scored rows and their targets.

    rank       1 + the number of ids whose key (order-preserving 16-bit key, -0 == +0) is strictly greater than the target's;
               -1 for a target outside [0, V).  NaN and inf take their key's place like any other value.
    targets    a prefill entry at prefix p holding x_p .. x_{p+n-1} scores rows j = 0 .. n-2 against x_{p+j+1}, and row n-1
               against the next prompt token when the caller gives it: k = n - 1 (+ 1) rows, first position p + 1."""
from __future__ import annotations

import numpy as np
import torch

import logprobs_oracle as LO
from sampling_oracle import keys_of


def ranks(logits: torch.Tensor, target_ids) -> np.ndarray:
    """int32 [B]."""
    bits = logits.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)
    keys = keys_of(bits).astype(np.int64)
    B, V = keys.shape
    tok = np.asarray(target_ids, dtype=np.int64).reshape(B)
    ok = (tok >= 0) & (tok < V)
    tk = keys[np.arange(B), np.clip(tok, 0, V - 1)]
    return np.where(ok, 1 + (keys > tk[:, None]).sum(axis=1), -1).astype(np.int32)


def prompt_logprobs(logits: torch.Tensor, target_ids, top_n: int):
    """(logprob fp32 [B], rank int32 [B], top ids int32 [B, top_n], top logprobs fp32 [B, top_n])."""
    lp, ids, tlp = LO.token_logprobs(logits, target_ids, top_n)
    return lp, ranks(logits, target_ids), ids, tlp


def entry_targets(ids: list, prefix: int, next_id=None):
    """(first position, rows of the entry (0-based within it), target ids) of one prefill entry."""
    k = len(ids) - 1 + (next_id is not None and len(ids) > 0)
    tgt = [int(x) for x in ids[1:]] + ([int(next_id)] if next_id is not None and len(ids) > 0 else [])
    return prefix + 1, list(range(k)), tgt
