"""TEST INFRASTRUCTURE: numpy restatement of the truncation filters of csrc/sampling.cu (sllm_sample_tokens_truncated).

With key(l) and the draw of sampling_oracle, m the row's largest logit, x_v = fp32((m - l_v) / T), q_v = exp(-x_v) and
w_v = round(q_v * 2^40), over the survivors of the previous filter (Z = sum of their w):
    min-p      min_p > 0: keep key >= the smallest key with q >= min_p (runs first);
    top-k      0 < k < V: keep key >= the k-th largest key;
    top-p      p < 1: keep key >= the largest threshold whose mass counted from the top reaches p * Z (Z over min-p and top-k);
    typical-p  typical_p < 1: E = sum round(fp32(q x) * 2^40) (0 where w is 0), c = fp32(E / Z), d = fp32(|x - c|); keep
               d <= delta, the smallest distance whose survivors weigh >= typical_p * Z;
    XTC        u = ((x >> 9) + 0.5) * 2^-23 of Philox4x32-10(key seed, counter (0, pos, 1, 0)) word 0; when u < xtc_probability
               and at least two finite survivors have w >= xtc_threshold * Z: keep key <= the smallest key among those
               (a -inf id is never such a top choice, so threshold 0 stops at the least likely finite survivor).
The kernel's expf and fixed-point sums differ from the fp64 values here in the last bits, so every threshold reports how close
the row came to it (`boundary_margin`, relative); the tests exempt rows within rounding of a boundary, as sampling_oracle does."""
from __future__ import annotations

import numpy as np
import torch

from sampling_oracle import RowResult, gumbel, keys_of, philox4x32_10

SCALE = 2.0 ** 40


def xtc_draw(seed: int, pos: int) -> np.float32:
    seed = int(seed) & (2 ** 64 - 1)
    x = philox4x32_10(0, np.uint32(pos), 1, 0, seed & 0xFFFFFFFF, seed >> 32)[0]
    return (np.float32(int(x) >> 9) + np.float32(0.5)) * np.float32(2.0 ** -23)


def _upper_mass_cut(keys, w, kept, target):
    """The largest key threshold whose survivors counted from the top weigh >= target, and the margin of that cut / Z."""
    uk = np.unique(keys[kept])[::-1]
    per_key = np.bincount(keys[kept], weights=w[kept], minlength=65536)[uk]
    cum = np.cumsum(per_key)
    j = int(np.argmax(cum >= target)) if (cum >= target).any() else len(uk) - 1
    Z = cum[-1]
    margin = min(abs(cum[j] - target), abs(target - cum[j - 1]) if j > 0 else np.inf) / Z
    return uk[j], margin


def sample_row(bits, vals, temperature, top_k, top_p, seed, pos, min_p=0.0, typical_p=1.0, xtc_threshold=0.1,
               xtc_probability=0.0, vocab_offset=0) -> RowResult:
    V = bits.shape[0]
    keys = keys_of(bits)
    T = np.float32(temperature)
    with np.errstate(invalid="ignore"):
        bad = bool(np.isnan(vals).any() or np.isposinf(vals).any() or not (vals > -np.inf).any())
    if not T > 0 or bad:
        i = int(np.argmax(keys))
        return RowResult(vocab_offset + i, float(vals[i]), None, np.inf, np.inf)
    v32 = vals.astype(np.float32)
    m = np.float32(v32.max())
    with np.errstate(over="ignore", invalid="ignore"):
        x = ((m - v32).astype(np.float32) / T).astype(np.float32)
        q = np.exp(-x.astype(np.float64))
    w = np.rint(q * SCALE)
    kept = np.ones(V, dtype=bool)
    margin = np.inf
    mp = np.float32(min_p)
    if mp > 0:
        lo = keys[q >= float(mp)].min()
        kept &= keys >= lo
        below = q[x > 0]                                                    # q of the maximum is exactly 1 on both sides
        margin = min(margin, (float(np.min(np.abs(below - float(mp)))) if below.size else np.inf) / float(mp))
    if 0 < top_k < V:
        kept &= keys >= np.sort(keys)[::-1][top_k - 1]
    p = np.float32(top_p)
    if p < 1:
        Z = w[kept].sum()
        thr, mg = _upper_mass_cut(keys, w, kept, float(p) * Z)
        kept &= keys >= thr
        margin = min(margin, mg)
    tp = np.float32(typical_p)
    if tp < 1:
        Z = w[kept].sum()
        with np.errstate(invalid="ignore"):
            e = np.where(kept & (w > 0), np.rint((q.astype(np.float32) * x).astype(np.float64) * SCALE), 0.0)
        c = np.float32(e.sum() / Z)
        with np.errstate(invalid="ignore"):
            d = np.abs((x - c).astype(np.float32))
        ud, inv = np.unique(d[kept], return_inverse=True)                  # ascending distinct distances
        per_d = np.bincount(inv, weights=w[kept], minlength=ud.size)
        cum = np.cumsum(per_d)
        target = float(tp) * Z
        j = int(np.argmax(cum >= target))
        delta = ud[j]
        surv = kept.copy()
        kept &= d <= delta
        margin = min(margin, min(abs(cum[j] - target), abs(target - cum[j - 1]) if j > 0 else np.inf) / Z)
        # a shift of c moves the distances on either side of it in opposite directions: distances near delta may swap
        near = np.abs(d[surv & (d != delta) & (w > 0)] - delta)
        margin = min(margin, (float(near.min()) if near.size else np.inf) / max(1.0, abs(float(c))))
    xp = np.float32(xtc_probability)
    if xp > 0 and xtc_draw(seed, pos) < xp:
        Z = w[kept].sum()
        bar = float(np.float32(xtc_threshold)) * Z
        top = kept & np.isfinite(v32) & (w >= bar)                          # -inf ids are never top choices
        if bar > 0:                                                          # bar 0: every finite survivor is one, exactly
            margin = min(margin, float(np.min(np.abs(w[kept] - bar))) / Z)
        if top.sum() >= 2:
            kept &= keys <= keys[top].min()
    score = vals.astype(np.float32) / T + gumbel(seed, pos, vocab_offset + np.arange(V, dtype=np.int64))
    s = np.where(kept, score, -np.inf).astype(np.float32)
    i = int(np.argmax(s))
    top2 = np.sort(s[kept])[::-1]
    gap = float(top2[0] - top2[1]) if top2.size > 1 else np.inf
    return RowResult(vocab_offset + i, float(s[i]), kept, gap, margin)


def sample_tokens(logits: torch.Tensor, temperature, top_k, top_p, seed, pos, min_p, typical_p, xtc_threshold, xtc_probability,
                  vocab_offset: int = 0) -> list:
    """logits [B, V] fp16 / bf16 (any device); per-row parameter sequences.  Returns a RowResult per row."""
    lg = logits.detach().cpu().contiguous()
    bits = lg.view(torch.int16).numpy().view(np.uint16)
    vals = lg.float().numpy()
    return [sample_row(bits[r], vals[r], temperature[r], top_k[r], top_p[r], seed[r], pos[r], min_p[r], typical_p[r],
                       xtc_threshold[r], xtc_probability[r], vocab_offset) for r in range(lg.shape[0])]
