"""Numpy restatement of csrc/constraints.cu (allowed-token masks and logit bias), the reference of the CPU and GPU tests.

For a constrained row of 16-bit logits l (a vocabulary shard starting at global id vocab_offset):
  mask   every id whose bit (mask[v // 32] >> (v % 32)) & 1 is 0 becomes -inf; allowed ids keep their bits (NaN, -0 included);
  bias   then every allowed id v with a bias b becomes round_to_storage(float32(l) + float32(b)): one IEEE fp32 add, one rounding
         to nearest even.  A bias on a masked id leaves it -inf; a biased NaN becomes the canonical NaN 0x7fff (the device's fp32
         add returns the canonical fp32 NaN, which converts to 0x7fff in fp16 and bf16);
  other  rows with neither are untouched."""
import numpy as np
import torch

CANONICAL_NAN = 0x7fff              # a NaN produced by the device's arithmetic, in fp16 and bf16


def allowed_ids(mask, lo: int, hi: int) -> np.ndarray:
    """bool [hi - lo]: the bits of global ids [lo, hi) of a packed mask."""
    words = np.asarray(mask).view(np.uint32)
    v = np.arange(lo, hi, dtype=np.int64)
    return ((words[v >> 5] >> (v & 31).astype(np.uint32)) & 1).astype(bool)


def constrain_row(row: torch.Tensor, mask=None, bias: dict = None, vocab_offset: int = 0) -> torch.Tensor:
    """One row (fp16 / bf16 CPU tensor of this shard's V ids): mask (packed int32 / uint32 words of global ids, or None) and bias
    ({global id: bias}, or None), as the kernel applies them."""
    out = row.clone()
    V = row.shape[0]
    ok = np.ones((V,), dtype=bool) if mask is None else allowed_ids(mask, vocab_offset, vocab_offset + V)
    if mask is not None:
        out[torch.from_numpy(~ok)] = float("-inf")
    for v, b in (bias or {}).items():
        local = int(v) - vocab_offset
        if 0 <= local < V and ok[local]:
            s = np.float32(np.float32(out[local].float().item()) + np.float32(b))
            out[local] = torch.tensor(float(s), dtype=torch.float32).to(row.dtype)
            if np.isnan(s):
                out.view(torch.int16)[local] = CANONICAL_NAN
    return out


def constrain(logits: torch.Tensor, masks: list, biases: list, vocab_offset: int = 0) -> torch.Tensor:
    """[rows, V] logits; masks / biases: per row None or as in constrain_row."""
    out = logits.clone()
    for i, (m, b) in enumerate(zip(masks, biases)):
        if m is not None or b:
            out[i] = constrain_row(logits[i], m, b, vocab_offset)
    return out


def constrain_staged(logits: torch.Tensor, mask_index, masks, bias_index, bias_starts, bias_ids, bias_values,
                     vocab_offset: int = 0) -> torch.Tensor:
    """The same semantics over the kernel's argument form (numpy / CPU arrays; see sllm_constrain_logits), vectorised for large
    batches: row r uses mask row mask_index[r] (-1: none) and bias entry bias_index[r] (-1: none) of the CSR arrays."""
    out = logits.clone()
    B, V = logits.shape
    mask_index, bias_index = np.asarray(mask_index), np.asarray(bias_index)
    bias_starts, bias_ids, bias_values = np.asarray(bias_starts), np.asarray(bias_ids), np.asarray(bias_values, np.float32)
    words = np.asarray(masks).view(np.uint32)
    ok = np.ones((B, V), dtype=bool)
    rows = np.flatnonzero(mask_index >= 0)
    if rows.size:
        v = np.arange(vocab_offset, vocab_offset + V, dtype=np.int64)
        ok[rows] = ((words[mask_index[rows]][:, v >> 5] >> (v & 31).astype(np.uint32)) & 1).astype(bool)
        out[torch.from_numpy(~ok)] = float("-inf")
    for r in np.flatnonzero(bias_index >= 0):
        e = bias_index[r]
        ids = bias_ids[bias_starts[e]:bias_starts[e + 1]].astype(np.int64) - vocab_offset
        vals = bias_values[bias_starts[e]:bias_starts[e + 1]]
        keep = (ids >= 0) & (ids < V)
        ids, vals = ids[keep], vals[keep]
        keep = ok[r, ids]
        ids, vals = torch.from_numpy(ids[keep]), torch.from_numpy(vals[keep])
        s = out[r, ids].float() + vals                                    # fp32 add, one rounding
        o = s.to(logits.dtype)
        o.view(torch.int16)[torch.isnan(s)] = CANONICAL_NAN
        out[r, ids] = o
    return out
