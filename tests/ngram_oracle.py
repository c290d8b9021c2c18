"""TEST INFRASTRUCTURE: numpy restatement of the n-gram controls of csrc/penalties.cu (sllm_apply_penalties_ngram).

One row, history x[0, L) of recorded ids (None: an unmapped position, which matches nothing):
    m(j)   the largest m in [0, min(j, 50)] with x[j - k] == x[L - k] for k = 1 .. m;   M(v) = max m(j) over j with x[j] == v;
    ban    (n >= 1) l = -inf where M(v) >= n - 1;
    DRY    (multiplier > 0) b = the smallest k >= 1 with x[L - k] a breaker (inf if none); for v no breaker, D = min(M(v), b - 1);
           where D >= A: q = multiplier, D - A times q = fp32(q * base), l = fp32(l - q).
Per entry of the shard [vocab_offset, vocab_offset + V): l = fp32(logit); the penalties (tests/penalties_oracle.py formulas)
when the row has any of r, f, p; DRY; the ban; ONE rounding to the storage dtype.  Entries none of these touches keep their
bits."""
from __future__ import annotations

import numpy as np
import torch

MAX_MATCH = 50


def match_lengths(x) -> dict:
    """{id: M(id)} over the ids of the history x (a list of ints, None for unmapped positions)."""
    L = len(x)
    M = {}
    for j in range(L):
        if x[j] is None:
            continue
        m, lim = 0, min(j, MAX_MATCH)
        while m < lim and x[j - m - 1] is not None and x[L - m - 1] is not None and x[j - m - 1] == x[L - m - 1]:
            m += 1
        M[x[j]] = max(M.get(x[j], -1), m)
    return M


def banned_ids(x, n: int) -> set:
    if n <= 0:
        return set()
    return {v for v, m in match_lengths(x).items() if m >= n - 1}


def breaker_distance(x, breakers) -> float:
    br = set(int(t) for t in breakers)
    for k in range(1, len(x) + 1):
        if x[-k] is not None and x[-k] in br:
            return k
    return float("inf")


def dry_penalties(x, multiplier: float, base: float, allowed: int, breakers) -> dict:
    """{id: fp32 q} of the ids DRY penalises."""
    if not multiplier > 0:
        return {}
    b = breaker_distance(x, breakers)
    br = set(int(t) for t in breakers)
    out = {}
    for v, m in match_lengths(x).items():
        if v in br:
            continue
        D = int(min(m, b - 1))
        if D >= allowed:
            q = np.float32(multiplier)
            with np.errstate(over="ignore"):
                for _ in range(D - allowed):
                    q = np.float32(q * np.float32(base))
            out[v] = q
    return out


def apply_row(row: torch.Tensor, x, vocab_offset: int = 0, r: float = 1.0, f: float = 0.0, p: float = 0.0, outputs=None,
              n: int = 0, multiplier: float = 0.0, base: float = 1.75, allowed: int = 2, breakers=()) -> torch.Tensor:
    """row: 1-D fp16 / bf16 logits of one row (a shard starting at vocab_offset); x: the history (ids, None unmapped);
    outputs: per position, whether it is an output token (for the frequency / presence counts).  Returns the new row."""
    out = row.detach().cpu().clone()
    V = row.shape[0]
    r, f, p = np.float32(r), np.float32(f), np.float32(p)
    pen = not (r == 1 and f == 0 and p == 0)
    outputs = [False] * len(x) if outputs is None else list(outputs)
    seen, cnt = {}, {}
    for t, o in zip(x, outputs):
        if t is not None:
            seen[t] = True
            cnt[t] = cnt.get(t, 0) + int(bool(o))
    dry = dry_penalties(x, multiplier, base, allowed, breakers)
    ban = banned_ids(x, n)
    touched = set(dry) | ban | (set(seen) if pen else set())
    vals = out.float().numpy().astype(np.float32)
    with np.errstate(all="ignore"):
        for v in touched:
            loc = v - vocab_offset
            if not 0 <= loc < V:
                continue
            l = np.float32(vals[loc])
            if pen and v in seen:
                l = np.float32(l / r) if l > 0 else np.float32(l * r)
                c = cnt[v]
                t = np.float32(f * np.float32(c))
                if c > 0:
                    t = np.float32(t + p)
                l = np.float32(l - t)
            if v in dry:
                l = np.float32(l - dry[v])
            if v in ban:
                l = np.float32(-np.inf)
            out[loc] = torch.tensor(float(l), dtype=torch.float32).to(row.dtype)
    return out


# ---------------------------------------------------------------- literal transcriptions of the reference algorithms

def hf_banned_tokens(tokens, n: int) -> set:
    """Hugging Face transformers' NoRepeatNGramLogitsProcessor (_get_ngrams / _get_generated_ngrams), one hypothesis."""
    cur_len = len(tokens)
    if cur_len + 1 < n:
        return set()
    generated_ngrams = {}
    gen_tokens = list(tokens)
    for ngram in zip(*[gen_tokens[i:] for i in range(n)]):
        prev_ngram_tuple = tuple(ngram[:-1])
        generated_ngrams[prev_ngram_tuple] = generated_ngrams.get(prev_ngram_tuple, []) + [ngram[-1]]
    start_idx = cur_len + 1 - n
    ngram_idx = tuple(tokens[start_idx:cur_len])
    return set(generated_ngrams.get(ngram_idx, []))


def webui_dry(tokens, multiplier: float, base: float, allowed_length: int, sequence_breakers) -> dict:
    """text-generation-webui's DRYLogitsProcessor loop for one row, without a penalty range: {token: penalty} (float64)."""
    input_ids = list(tokens)
    last_token = input_ids[-1]
    if last_token in sequence_breakers:
        return {}
    match_indices = []
    for idx, val in enumerate(input_ids[:-1]):
        if val == last_token:
            match_indices.append(idx)
    match_lengths = {}
    for i in match_indices:
        next_token = input_ids[i + 1]
        if next_token in sequence_breakers:
            continue
        match_length = 1
        while match_length < 50:
            j = i - match_length
            if j < 0:
                break
            previous_token = input_ids[-(match_length + 1)]
            if input_ids[j] != previous_token:
                break
            if previous_token in sequence_breakers:
                break
            match_length += 1
        if next_token in match_lengths:
            match_lengths[next_token] = max(match_length, match_lengths[next_token])
        else:
            match_lengths[next_token] = match_length
    out = {}
    for token, match_length in match_lengths.items():
        if match_length >= allowed_length:
            out[token] = multiplier * base ** (match_length - allowed_length)
    return out
