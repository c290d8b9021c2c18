"""TEST INFRASTRUCTURE: numpy restatement of the penalty semantics of csrc/penalties.cu (sllm_apply_penalties).

Per row of 16-bit logits with parameters r (repetition), f (frequency), p (presence) and a history of (id, is_output) tokens:
    c_out(v)   number of output tokens equal to v;  seen(v): v occurs among the prompt or the output tokens;
    seen v     l = fp32(logit); l = l / r if l > 0 else l * r; t = f * fp32(c_out); t = t + p if c_out > 0; l = l - t; every
               operation one IEEE fp32 rounding (np.float32 scalars, no fused multiply-add), then ONE rounding to the storage
               dtype, round to nearest even (torch's .to(float16 / bfloat16));
    other v    unchanged, bit for bit (NaN, +-inf, -0 included);
    ids outside [vocab_offset, vocab_offset + V) are absent.
A row with r == 1, f == 0, p == 0 is unchanged.  The operation is elementwise with one rounding, so the kernel must match this
restatement bit for bit."""
from __future__ import annotations

import numpy as np
import torch


def counts_of(history, vocab_offset: int, V: int):
    """history: iterable of (id, is_output), or a pair of arrays (ids, is_output) -> (seen [V] bool, output counts [V] int64)."""
    if isinstance(history, tuple) and len(history) == 2 and isinstance(history[0], np.ndarray):
        ids, is_out = history
    else:
        h = list(history)
        ids = np.array([int(t) for t, _ in h], dtype=np.int64)
        is_out = np.array([bool(o) for _, o in h], dtype=bool)
    loc = np.asarray(ids, dtype=np.int64) - vocab_offset
    ok = (loc >= 0) & (loc < V)
    seen = np.bincount(loc[ok], minlength=V) > 0
    cnt = np.bincount(loc[ok & np.asarray(is_out, dtype=bool)], minlength=V).astype(np.int64)
    return seen, cnt


def penalize_row(row: torch.Tensor, r: float, f: float, p: float, history, vocab_offset: int = 0) -> torch.Tensor:
    """row: 1-D fp16 / bf16 logits of one row (a shard starting at vocab_offset); returns the penalised copy."""
    out = row.detach().cpu().clone()
    r, f, p = np.float32(r), np.float32(f), np.float32(p)
    if r == 1 and f == 0 and p == 0:
        return out
    V = row.shape[0]
    seen, cnt = counts_of(history, vocab_offset, V)
    ids = np.nonzero(seen)[0]
    if ids.size == 0:
        return out
    l = out[torch.from_numpy(ids)].float().numpy().astype(np.float32)
    c = cnt[ids]
    with np.errstate(all="ignore"):
        l = np.where(l > 0, l / r, l * r).astype(np.float32)
        t = (f * c.astype(np.float32)).astype(np.float32)
        t = np.where(c > 0, (t + p).astype(np.float32), t).astype(np.float32)
        l = (l - t).astype(np.float32)
    out[torch.from_numpy(ids)] = torch.from_numpy(l).to(row.dtype)
    return out


def penalize(logits: torch.Tensor, params, histories, vocab_offset: int = 0) -> torch.Tensor:
    """logits [B, V]; params [(r, f, p)] per row; histories per row (see counts_of)."""
    out = logits.detach().cpu().clone()
    for i, ((r, f, p), h) in enumerate(zip(params, histories)):
        out[i] = penalize_row(out[i], r, f, p, h, vocab_offset)
    return out
