"""CPU: the slabbed fp64 prefill references of tests/prefill64.py (which the long-prompt GPU tests use) against the
oracle's definitions, at small ragged shapes with slabs smaller than the sequences so that slab edges are crossed."""
import numpy as np
import pytest
import torch

import prefill64
from oracle import kernels as K


@pytest.mark.parametrize("slab", [1, 5, 64, 1024])
@pytest.mark.parametrize("nq,nkv", [(4, 4), (8, 2), (12, 4)])
def test_packed_matches_oracle(slab, nq, nkv):
    D = 32
    lens = [1, 7, 0, 33, 64, 65, 2]
    starts = list(np.cumsum([0] + lens[:-1]))
    T = sum(lens) + 3                                          # trailing rows outside every sequence stay zero
    g = torch.Generator().manual_seed(nq * 10 + slab)
    q = torch.randn(T, nq, D, generator=g, dtype=torch.float64)
    k = torch.randn(T, nkv, D, generator=g, dtype=torch.float64)
    v = torch.randn(T, nkv, D, generator=g, dtype=torch.float64)
    ref = K.prefill_attention_exact(q, k, v, starts, lens, D ** -0.5)
    got = prefill64.prefill_attention(q, k, v, starts, lens, D ** -0.5, slab=slab)
    assert got.dtype == torch.float64 and got.shape == ref.shape
    assert (got - ref).abs().max() <= 1e-12 * ref.abs().max()
    assert (got[sum(lens):] == 0).all()


@pytest.mark.parametrize("slab", [1, 5, 64, 1024])
@pytest.mark.parametrize("nq,nkv", [(4, 4), (8, 2), (12, 4)])
def test_prefix_matches_oracle(slab, nq, nkv):
    D, bs, layers, layer = 32, 16, 2, 1
    prefix = [0, 13, 16, 40, 3, 100]
    chunk = [5, 20, 1, 0, 47, 17]
    starts = list(np.cumsum([0] + chunk[:-1]))
    g = torch.Generator().manual_seed(nq * 10 + slab + 1)
    need = [(p + c + bs - 1) // bs for p, c in zip(prefix, chunk)]
    nblk = sum(need) + 4
    perm = torch.randperm(nblk, generator=g).tolist()
    sids = [5, 0, 3, 1, 6, 2]                                  # block-table rows in another order than the chunks
    bt = torch.full((7, max(need) + 1), -1, dtype=torch.int32)
    p = 0
    for s, n in zip(sids, need):
        bt[s, :n] = torch.tensor(perm[p:p + n], dtype=torch.int32); p += n
    kc = torch.randn(nblk, layers, nkv, bs, D, generator=g, dtype=torch.float64)
    vc = torch.randn(nblk, layers, nkv, bs, D, generator=g, dtype=torch.float64)
    T = sum(chunk) + 2
    q = torch.randn(T, nq, D, generator=g, dtype=torch.float64)
    ref = K.prefix_prefill_attention_exact(q, kc, vc, bt.numpy(), sids, starts, chunk, prefix, D ** -0.5, bs, layer)
    for table in (bt, bt.numpy()):
        got = prefill64.prefix_prefill_attention(q, kc, vc, table, sids, starts, chunk, prefix, D ** -0.5, bs, layer,
                                                 slab=slab)
        assert got.dtype == torch.float64 and got.shape == ref.shape
        assert (got - ref).abs().max() <= 1e-12 * ref.abs().max()
        assert (got[sum(chunk):] == 0).all()


def test_half_precision_inputs_are_widened_exactly():
    """Inputs in the storage dtypes are evaluated in fp64 (as the oracle does), not in their own precision."""
    nq, nkv, D = 8, 2, 64
    lens = [50, 17]
    starts = [0, 50]
    g = torch.Generator().manual_seed(3)
    for dt in (torch.float16, torch.bfloat16):
        q = torch.randn(67, nq, D, generator=g).to(dt)
        k = torch.randn(67, nkv, D, generator=g).to(dt)
        v = torch.randn(67, nkv, D, generator=g).to(dt)
        ref = K.prefill_attention_exact(q, k, v, starts, lens, D ** -0.5)
        got = prefill64.prefill_attention(q, k, v, starts, lens, D ** -0.5, slab=16)
        assert (got - ref).abs().max() <= 1e-12 * ref.abs().max()
