"""TEST INFRASTRUCTURE: numpy restatement of the sampling semantics of csrc/sampling.cu (sllm_sample_tokens).

    key(l)   order-preserving uint16 of the 16-bit logit bits, -0 mapped to +0;
    T == 0   greedy: the first index of the largest key (== torch.argmax);
    top-k    0 < k < V: keep key >= the k-th largest key (boundary ties kept);
    top-p    p < 1: over the survivors, q = exp((l - m) / T) (fp64 here), keep key >= the largest threshold whose mass counted
             from the top is >= p * sum(q);
    draw     x = Philox4x32-10(key (seed_lo, seed_hi), counter (v >> 2, pos, 0, 0)) word v & 3, u = ((x >> 9) + 0.5) * 2^-23,
             score = fp32(l) / T + (-log(-log u)) in fp32, token = first index of the largest score among the kept tokens.
The kernel sums masses in 2^-40 fixed point and uses CUDA's logf, so the tests exempt rows whose top-p boundary or top-2 score
gap is within rounding of those differences (`boundary_margin`, `gap`)."""
from __future__ import annotations

import dataclasses

import numpy as np
import torch

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Vectorised Philox4x32-10 (Random123): uint32 arrays (broadcast) -> four uint32 arrays."""
    c = [np.asarray(x, dtype=np.uint64) for x in (c0, c1, c2, c3)]
    k0, k1 = np.asarray(k0, dtype=np.uint64), np.asarray(k1, dtype=np.uint64)
    mask = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & mask, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & mask]
        k0 = (k0 + np.uint64(W0)) & mask
        k1 = (k1 + np.uint64(W1)) & mask
    return [x.astype(np.uint32) for x in c]


def keys_of(bits: np.ndarray) -> np.ndarray:
    bits = np.where(bits == 0x8000, 0, bits).astype(np.uint32)
    return np.where(bits & 0x8000, ~bits & 0xFFFF, bits | 0x8000).astype(np.uint32)


def gumbel(seed: int, pos: int, gidx: np.ndarray) -> np.ndarray:
    seed = int(seed) & (2 ** 64 - 1)
    w = philox4x32_10(gidx >> 2, np.uint32(pos), 0, 0, seed & 0xFFFFFFFF, seed >> 32)
    x = np.choose((gidx & 3).astype(np.int64), w)
    u = ((x >> 9).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)
    return -np.log(-np.log(u))


@dataclasses.dataclass
class RowResult:
    token: int
    score: float              # the pair value: logit (greedy) or best score
    kept: np.ndarray | None   # bool [V] (None for greedy rows)
    gap: float                # top-1 minus top-2 score among the kept tokens (inf if one token is kept)
    boundary_margin: float    # top-p: distance of p*Z to the nearest cumulative mass at a key boundary, over Z (inf if off)


def sample_row(bits: np.ndarray, vals: np.ndarray, temperature, top_k, top_p, seed, pos, vocab_offset=0) -> RowResult:
    V = bits.shape[0]
    keys = keys_of(bits)
    T = np.float32(temperature)
    if not T > 0:
        i = int(np.argmax(keys))
        return RowResult(vocab_offset + i, float(vals[i]), None, np.inf, np.inf)
    kept = np.ones(V, dtype=bool)
    if 0 < top_k < V:
        tau = np.sort(keys)[::-1][top_k - 1]
        kept = keys >= tau
    margin = np.inf
    p = np.float32(top_p)
    if p < 1:
        m = float(vals[kept].max())
        q = np.where(kept, np.exp((vals.astype(np.float64) - m) / float(T)), 0.0)
        Z = q.sum()
        target = float(p) * Z
        uk = np.unique(keys[kept])[::-1]                          # descending distinct keys
        mass_per_key = np.bincount(keys, weights=q, minlength=65536)[uk]
        cum = np.cumsum(mass_per_key)
        j = int(np.argmax(cum >= target)) if (cum >= target).any() else len(uk) - 1
        kept &= keys >= uk[j]
        margin = min(abs(cum[j] - target), abs(target - cum[j - 1]) if j > 0 else np.inf) / Z
    score = vals.astype(np.float32) / T + gumbel(seed, pos, vocab_offset + np.arange(V, dtype=np.int64))
    s = np.where(kept, score, -np.inf).astype(np.float32)
    i = int(np.argmax(s))
    top2 = np.sort(s[kept])[::-1]
    gap = float(top2[0] - top2[1]) if top2.size > 1 else np.inf
    return RowResult(vocab_offset + i, float(s[i]), kept, gap, margin)


def sample_tokens(logits: torch.Tensor, temperature, top_k, top_p, seed, pos, vocab_offset: int = 0) -> list:
    """logits [B, V] fp16 / bf16 (any device); per-row parameter sequences.  Returns a RowResult per row."""
    lg = logits.detach().cpu().contiguous()
    bits = lg.view(torch.int16).numpy().view(np.uint16)
    vals = lg.float().numpy()
    return [sample_row(bits[r], vals[r], temperature[r], top_k[r], top_p[r], seed[r], pos[r], vocab_offset)
            for r in range(lg.shape[0])]


def merge_pairs(results_per_shard: list) -> list:
    """[shards][rows] RowResult -> merged global tokens: the largest score, then the smallest index."""
    out = []
    for r in range(len(results_per_shard[0])):
        best = max(((res[r].score, -res[r].token) for res in results_per_shard))
        out.append(-best[1])
    return out
