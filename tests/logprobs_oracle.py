"""TEST INFRASTRUCTURE: numpy restatement of the log-probability semantics of csrc/logprobs.cu (sllm_token_logprobs), and the
fp64 reference both are held to.

Per row of 16-bit logits l (full vocabulary, V entries):
    key(l)     order-preserving uint16 of the bits, -0 mapped to +0 (tests/sampling_oracle.keys_of);
    m          the value of the largest key;
    Z          sum over v of rint(fp32(exp(fp32(l_v - m))) * 2^40) as uint64 - exact, so the order of additions is irrelevant;
    lse        fp32(m + fp32(log(fp32(Z) * 2^-40)));  logprob(v) = fp32(l_v - lse);
    top-N      the min(N, V) ids with the largest keys, ordered by (key desc, id asc); later slots id -1 and NaN;
    token      logprob(token), NaN for a token outside [0, V);
    bad rows   a NaN or +inf anywhere, or a largest logit of -inf: every logprob NaN (the top ids still follow the keys).

Tolerance.  The fp64 reference is log_softmax of the 16-bit values computed in float64: exact to ~1e-15.  Against it, the fp32
computation above (the kernel's, and this restatement's) makes these rounding steps, for |l| <= 64 and V <= 2^20:
    exp        CUDA expf is within 2 ulp (numpy's float32 exp within 1): a relative error <= 2^-22 in every term, so in Z;
    fixed point each term is rounded to a multiple of 2^-40 (<= 2^-41 each) while Z >= 1 (the max term is expf(0) = 1 exactly):
               a relative error <= V * 2^-41 <= 2^-21;
    fp32(Z)    2^-24 relative.  Relative errors of Z become absolute errors of log Z: together <= 2^-22 + 2^-21 + 2^-24 < 8e-7;
    logf       <= 1 ulp of log Z <= log(2^20) < 16: 2^-20 < 1e-6;
    m + log Z  rounding to fp32 of a value below 64 + 16 < 128: half an ulp, 2^-18 < 3.9e-6;
    l - lse    rounding of a value below 128 + 16 < 256: half an ulp, 2^-17 < 7.7e-6.
The sum is below 1.35e-5, so TOL = 2e-5 absolute holds with margin for any |l| <= 64.  Two fp32 results (kernel and
restatement) may therefore differ by up to 2 * TOL; both are held to the fp64 reference instead of to each other.  The ids do
not depend on any rounding and must match bit for bit."""
from __future__ import annotations

import numpy as np
import torch

from sampling_oracle import keys_of

TOL = 2e-5
MAX_TOP_N = 20


def _bits_vals(logits: torch.Tensor):
    lg = logits.detach().cpu().contiguous()
    bits = lg.view(torch.int16).numpy().view(np.uint16)
    return bits, lg.float().numpy(), lg.dtype


def _bad_rows(keys: np.ndarray, dtype) -> np.ndarray:
    pos, neg = (0xFC00, 0x03FF) if dtype == torch.float16 else (0xFF80, 0x007F)
    return ((keys >= pos) | (keys < neg)).any(axis=1)


def value_of_keys(keys: np.ndarray, dtype) -> np.ndarray:
    bits = np.where(keys & 0x8000, keys ^ 0x8000, ~keys & 0xFFFF).astype(np.uint16)
    return torch.from_numpy(bits.view(np.int16).copy()).view(dtype).float().numpy()


def top_ids(keys: np.ndarray, n: int) -> np.ndarray:
    """int32 [B, n]: the ids of the min(n, V) largest keys, (key desc, id asc); -1 beyond V."""
    B, V = keys.shape
    out = np.full((B, n), -1, dtype=np.int32)
    k = min(n, V)
    if k == 0:
        return out
    comp = (keys.astype(np.int64) << 32) | (0xFFFFFFFF - np.arange(V, dtype=np.int64))[None]     # larger = better, unique
    part = np.argpartition(-comp, k - 1, axis=1)[:, :k]
    order = np.argsort(-np.take_along_axis(comp, part, axis=1), axis=1)
    out[:, :k] = np.take_along_axis(part, order, axis=1)
    return out


def token_logprobs(logits: torch.Tensor, token_ids, top_n: int):
    """The kernel's semantics in numpy: (token logprob fp32 [B], top ids int32 [B, top_n], top logprobs fp32 [B, top_n])."""
    bits, vals, dtype = _bits_vals(logits)
    B, V = bits.shape
    keys = keys_of(bits)
    bad = _bad_rows(keys, dtype)
    m = value_of_keys(keys.max(axis=1), dtype).astype(np.float32)
    bad |= m == -np.inf
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        d = (vals.astype(np.float32) - m[:, None]).astype(np.float32)
        q = np.exp(d).astype(np.float32) * np.float32(2.0 ** 40)
        q = np.where(bad[:, None], 0, q)
        Z = np.rint(q).astype(np.uint64).sum(axis=1, dtype=np.uint64)
        lse = (m + np.log(Z.astype(np.float32) * np.float32(2.0 ** -40)).astype(np.float32)).astype(np.float32)
    lse = np.where(bad, np.float32(np.nan), lse).astype(np.float32)
    lv = value_of_keys(keys, dtype).astype(np.float32)                 # -0 read as +0, like the kernel
    tok = np.asarray(token_ids, dtype=np.int64).reshape(B)
    ok = (tok >= 0) & (tok < V)
    tl = np.where(ok, lv[np.arange(B), np.clip(tok, 0, V - 1)] - lse, np.float32(np.nan)).astype(np.float32)
    ids = top_ids(keys, top_n)
    tlp = np.where(ids >= 0, np.take_along_axis(lv, np.clip(ids, 0, V - 1), axis=1) - lse[:, None], np.float32(np.nan))
    return tl, ids, tlp.astype(np.float32)


def log_softmax64(logits: torch.Tensor) -> np.ndarray:
    """fp64 reference [B, V]."""
    return torch.log_softmax(logits.detach().cpu().double(), dim=1).numpy()
