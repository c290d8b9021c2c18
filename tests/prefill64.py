"""The fp64 definitions of packed and prefix-aware prefill attention (oracle/kernels.py: prefill_attention_exact,
prefix_prefill_attention_exact), evaluated on whatever device the inputs live on.

The CPU oracles build the whole [heads, rows, keys] score tensor of a sequence, which a 16384-token prompt does not fit
(32 heads x 16384^2 x 8 bytes = 64 GiB).  Here each kv head's GQA group of query heads is processed in slabs of SLAB
query rows against the keys those rows can see (causal: at most prefix + the slab's last row + 1), so the largest
temporary of a 16384-token prompt with GQA group 4 is 4 x 1024 x 16384 fp64 values (512 MiB).
tests/test_prefill64_cpu.py holds both functions to the CPU oracles."""
import torch

SLAB = 1024


def _attend(out, Q, K, V, pre, scale, slab):
    """out[t] = softmax(Q[t] K[:pre + t + 1]^T * scale) V[:pre + t + 1] for the n rows of one sequence, in fp64.
    Q [n, nq, D], K / V [nkv, >= pre + n, D]; out [n, nq, D]."""
    n, nq, _ = Q.shape
    nkv = K.shape[0]
    g = nq // nkv
    dev = Q.device
    for h in range(nkv):
        Qh = Q[:, h * g:(h + 1) * g]
        for r0 in range(0, n, slab):
            r1 = min(n, r0 + slab)
            L = pre + r1
            s = torch.einsum("rgd,kd->grk", Qh[r0:r1], K[h, :L]) * scale
            pos = pre + torch.arange(r0, r1, device=dev)
            s.masked_fill_(torch.arange(L, device=dev)[None, None, :] > pos[None, :, None], float("-inf"))
            out[r0:r1, h * g:(h + 1) * g] = torch.einsum("grk,kd->rgd", torch.softmax(s, dim=-1), V[h, :L])


def prefill_attention(q, k, v, start_locs, seq_lens, softmax_scale, slab=SLAB):
    """prefill_attention_exact: causal attention of each packed sequence over its own rows of k / v.
    q [T, nq, D], k / v [T, nkv, D] -> fp64 [T, nq, D] on q's device; rows outside every sequence are zero."""
    T, nq, D = q.shape
    out = torch.zeros((T, nq, D), dtype=torch.float64, device=q.device)
    for s0, n in zip(start_locs, seq_lens):
        s0, n = int(s0), int(n)
        if n == 0:
            continue
        K = k[s0:s0 + n].to(torch.float64).transpose(0, 1)
        V = v[s0:s0 + n].to(torch.float64).transpose(0, 1)
        _attend(out[s0:s0 + n], q[s0:s0 + n].to(torch.float64), K, V, 0, softmax_scale, slab)
    return out


def _gather(cache, row, L, block_size, layer):
    """Positions 0 .. L-1 of one sequence from a paged cache [blocks, layers, nkv, bs, D] -> fp64 [nkv, L, D]."""
    npg = (L + block_size - 1) // block_size
    blocks = torch.as_tensor(row[:npg]).to(device=cache.device, dtype=torch.long)
    pages = cache[blocks, layer].to(torch.float64)                          # [npg, nkv, bs, D]
    return pages.permute(1, 0, 2, 3).reshape(pages.shape[1], npg * block_size, -1)[:, :L]


def prefix_prefill_attention(q, k_cache, v_cache, block_table, seq_ids, start_locs, chunk_lens, prefix_lens,
                             softmax_scale, block_size, cur_layer, slab=SLAB):
    """prefix_prefill_attention_exact: chunk b holds positions prefix_lens[b] .. prefix_lens[b] + chunk_lens[b] - 1 of
    sequence seq_ids[b] and attends to every position up to its own, read from the paged caches through block_table.
    q [Tp, nq, D] -> fp64 [Tp, nq, D] on q's device; rows outside every chunk are zero."""
    T, nq, D = q.shape
    out = torch.zeros((T, nq, D), dtype=torch.float64, device=q.device)
    for b in range(len(chunk_lens)):
        s0, n, pre = int(start_locs[b]), int(chunk_lens[b]), int(prefix_lens[b])
        if n == 0:
            continue
        row = block_table[int(seq_ids[b])]
        K = _gather(k_cache, row, pre + n, block_size, cur_layer)
        V = _gather(v_cache, row, pre + n, block_size, cur_layer)
        _attend(out[s0:s0 + n], q[s0:s0 + n].to(torch.float64), K, V, pre, softmax_scale, slab)
    return out
