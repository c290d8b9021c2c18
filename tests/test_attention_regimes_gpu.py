"""GPU: attention in the regimes and at the cache edges the product reaches, against the fp64 definition
(tests/attention_check.py), both kernel generations wherever a shape is served by both:
  * decode planner regimes (csrc/paged_attn.cu choose_split_tokens), each asserted through the workspace size, which is 0
    iff a launch has one split: single pass (batch x kv heads >= 6 x SMs), a sequence longer than PA_MAX_SPLIT_TOKENS
    (16384) inside it, and the bench regime (batch 64 x 4096, 8 kv heads: two splits of 2048);
  * decode rows dominated by one "sink" key in the first tile, the last tile and the last split;
  * decode over a cache with NaN in every page it does not own and NaN K / huge V past the end of its last pages;
  * element offsets past 2^31 in decode, chunked prefill and store_kvcache (two 4 GiB caches);
  * row-strided (fused-QKV) q for GQA group 3 in decode and both prefills;
  * speculative verification (sllm_paged_attention_verify) in the same regimes: single pass, rows straddling split
    boundaries over a NaN workspace, sink keys at draft positions, poisoned pages with more items than SMs, element offsets
    past 2^31, and bit-exact repeats and block permutations."""
import functools

import numpy as np
import pytest
import torch

from attention_check import check_attention
from oracle import kernels as K
from test_chunked_prefill_gpu import i32
from test_kernels_gpu import NS, _paged_run, check_fused_qkv_column_slices, paged_gen, prefill_gen  # noqa: F401 (fixtures)
from test_speculative_gpu import verify_gen  # noqa: F401 (fixture)
from verify_shapes import random_kv_q, verify_np

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.float16, torch.bfloat16]
D, BS = 128, 16
PA_MAX_SPLIT_TOKENS = 16384


def num_splits(B, nq, nkv, max_len):
    """Splits of a decode launch, read back from the planner through the workspace it asks for."""
    from swiftllm_b200 import _lib
    ws = _lib.lib().sllm_paged_attention_workspace_bytes(B, nq, D, max_len, 0, nkv)
    if ws == 0:
        return 1
    per_split = B * nq * (D + 1) * 4
    assert ws % per_split == 0, ws
    return ws // per_split


def _table(g, lens, extra_blocks=0, base=0):
    """Block table over randomly permuted blocks base .. base + sum(pages) + extra_blocks - 1, sequence i in row i."""
    need = [(n + BS - 1) // BS for n in lens]
    nblk = sum(need) + extra_blocks
    perm = (torch.randperm(nblk, generator=g) + base).tolist()
    bt = torch.full((len(lens), max(need) + 1), -1, dtype=torch.int32)
    p = 0
    for s, n in enumerate(need):
        bt[s, :n] = torch.tensor(perm[p:p + n], dtype=torch.int32); p += n
    return bt, nblk


@functools.lru_cache(maxsize=3)           # shared by the two kernel generations
def _decode_case(lens, nq, nkv, dtype, seed):
    """Random decode batch (CPU tensors, sequence i in block-table row i) and its fp64 output."""
    g = torch.Generator().manual_seed(seed)
    bt, nblk = _table(g, lens)
    kc = torch.randn(nblk, 1, nkv, BS, D, generator=g).to(dtype); vc = torch.randn(nblk, 1, nkv, BS, D, generator=g).to(dtype)
    q = torch.randn(len(lens), nq, D, generator=g).to(dtype)
    o64 = K.paged_attention_exact(q, kc, vc, bt, range(len(lens)), lens, D ** -0.5, BS, 0)
    return q, kc, vc, bt, o64


def _single_pass_lens(nkv, longest):
    """Enough sequences that batch x kv heads >= 6 x SMs; mixed lengths, page and tile edges, one `longest` row."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = -(-6 * sms // nkv) + 3
    rng = np.random.default_rng(B)
    lens = rng.integers(1, 700, size=B)
    lens[:9] = [longest, 1, 15, 16, 17, 127, 128, 129, 2049]
    return tuple(int(x) for x in lens)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("longest,splits", [(PA_MAX_SPLIT_TOKENS, 1), (PA_MAX_SPLIT_TOKENS + 4007, 2)])
def test_decode_single_pass_regime(dtype, longest, splits, paged_gen):
    """The regime of large-batch serving: each persistent CTA handles several (sequence, kv head) items and writes o
    directly, rolling over its Q double buffer and its K / V rings.  With one row longer than 16384 tokens the launch
    still uses 16384-token splits; every other row's second split item is then empty."""
    nq, nkv = 24, 8                                                   # GQA group 3: padded to 8 heads by the wgmma kernel
    lens = _single_pass_lens(nkv, longest)
    B = len(lens)
    assert num_splits(B, nq, nkv, PA_MAX_SPLIT_TOKENS) == 1, "the batch alone must select the single-pass regime"
    assert num_splits(B, nq, nkv, longest) == splits, f"expected {splits} split(s) of {PA_MAX_SPLIT_TOKENS} tokens"
    q, kc, vc, bt, o64 = _decode_case(lens, nq, nkv, dtype, seed=longest)
    o = _paged_run(q, kc, vc, bt, list(range(B)), list(lens), D ** -0.5, BS, 0)
    check_attention(o, o64, nq, lens, what="decode")


def test_decode_bench_regime(paged_gen):
    """bench.py's shape (Llama-3-8B heads, bf16, batch 64, up to 4096 tokens): the planner makes two splits of 2048 tokens.
    Rows of 2048 or fewer tokens leave their second split item empty; 2049 puts one token in it."""
    nq, nkv, B = 32, 8, 64
    rng = np.random.default_rng(64)
    lens = rng.integers(1, 4097, size=B)
    lens[:12] = [4096, 4096, 4095, 2049, 2048, 2047, 1, 17, 128, 129, 2176, 3968]
    lens = tuple(int(x) for x in lens)
    # two splits at 4096 tokens means the planner aimed at 2 items per (sequence, kv head): split_tokens = 4096 / 2
    assert num_splits(B, nq, nkv, 4096) == 2, "expected two splits of 2048 tokens"
    q, kc, vc, bt, o64 = _decode_case(lens, nq, nkv, torch.bfloat16, seed=4096)
    o = _paged_run(q, kc, vc, bt, list(range(B)), list(lens), D ** -0.5, BS, 0)
    check_attention(o, o64, nq, lens, what="decode")


@pytest.mark.parametrize("dtype", DTYPES)
def test_decode_peaked_rows(dtype, paged_gen):
    """One key per (sequence, kv head) dominates its row by more than 150 in log2 units, so every other p is exactly 0
    and the output is that key's V up to the output rounding.  The sink sits in the first tile, in the last tile (the
    last token), in the last split but not in its last tile, and mid-sequence; the planner splits this small batch."""
    nq, nkv = 32, 8
    lens = [4096, 4096, 4096, 777, 300, 1000]
    sink = [3, 4095, 3850, 776, 130, 640]
    assert num_splits(len(lens), nq, nkv, max(lens)) > 1
    g = torch.Generator().manual_seed(150)
    bt, nblk = _table(g, lens)
    kc = torch.randn(nblk, 1, nkv, BS, D, generator=g); vc = torch.randn(nblk, 1, nkv, BS, D, generator=g)
    u = torch.randint(0, 2, (len(lens), nkv, D), generator=g).float() * 2 - 1            # one +-1 direction per kv head
    q = 0.3 * torch.randn(len(lens), nq, D, generator=g) + u.repeat_interleave(nq // nkv, dim=1)
    for s, (n, j) in enumerate(zip(lens, sink)):
        kc[int(bt[s, j // BS]), 0, :, j % BS] = 16 * u[s]
    q, kc, vc = q.to(dtype), kc.to(dtype), vc.to(dtype)
    o64 = K.paged_attention_exact(q, kc, vc, bt, range(len(lens)), lens, D ** -0.5, BS, 0)
    c = D ** -0.5 * K.LOG2E
    for s, (n, j) in enumerate(zip(lens, sink)):                      # the premise: a gap of more than 150 (log2 units)
        keys = torch.cat([kc[int(b), 0] for b in bt[s, :(n + BS - 1) // BS]], dim=1)[:, :n].double()   # [nkv, n, D]
        sc = torch.einsum("khd,knd->khn", q[s].double().view(nkv, nq // nkv, D), keys) * c
        others = torch.cat([sc[..., :j], sc[..., j + 1:]], dim=-1)
        assert float((sc[..., j] - others.amax(-1)).min()) > 150
    o = _paged_run(q, kc, vc, bt, list(range(len(lens))), lens, D ** -0.5, BS, 0).view(len(lens), nq, D)
    check_attention(o, o64, nq, lens, what="decode")
    u_out = 2.0 ** -11 if dtype == torch.float16 else 2.0 ** -8
    for s, j in enumerate(sink):
        v = vc[int(bt[s, j // BS]), 0, :, j % BS].float().repeat_interleave(nq // nkv, dim=0)   # [nq, D]
        assert ((o[s].float() - v).abs() <= u_out * v.abs()).all(), f"sequence {s}: output is not the sink's V"


@pytest.mark.parametrize("dtype", DTYPES)
def test_decode_poisoned_pages_are_harmless(dtype, paged_gen):
    """The decode counterpart of test_prefill_attention_paged_nan_in_unowned_pages_is_harmless: blocks (and layers) a
    sequence does not own hold NaN; slots of its last page past the end hold NaN K and V = 3e4.  The wgmma kernel loads
    whole pages, so the tail must be masked before the softmax and multiplied by P = 0 exactly."""
    nq, nkv, L, layer = 24, 8, 2, 1
    lens = [1, 15, 17, 91, 300, 777, 4091]
    g = torch.Generator().manual_seed(91)
    bt, nblk = _table(g, lens, extra_blocks=7)
    kc = torch.randn(nblk, L, nkv, BS, D, generator=g).to(dtype); vc = torch.randn(nblk, L, nkv, BS, D, generator=g).to(dtype)
    q = torch.randn(len(lens), nq, D, generator=g).to(dtype)
    sids = list(range(len(lens)))
    o64 = K.paged_attention_exact(q, kc, vc, bt, sids, lens, D ** -0.5, BS, layer)
    owned = set()
    for s, n in enumerate(lens):
        npg = (n + BS - 1) // BS
        owned |= set(bt[s, :npg].tolist())
        last = int(bt[s, npg - 1])
        kc[last, layer, :, n - (npg - 1) * BS:] = float("nan"); vc[last, layer, :, n - (npg - 1) * BS:] = 3.0e4
    kc[:, 1 - layer] = float("nan"); vc[:, 1 - layer] = float("nan")
    for b in range(nblk):
        if b not in owned:
            kc[b] = float("nan"); vc[b] = float("nan")
    o = _paged_run(q, kc, vc, bt, sids, lens, D ** -0.5, BS, layer)
    assert torch.isfinite(o.float()).all()
    check_attention(o, o64, nq, lens, what="decode")


# ----------------------------------------------------------------------------- element offsets past 2^31
BIG_NKV, BIG_NQ = 8, 24
BIG_BLOCK_ELEMS = BIG_NKV * BS * D                                    # one layer
FIRST_BIG = 2 ** 31 // BIG_BLOCK_ELEMS                                # first block whose element offset is 2^31
BIG_BLOCKS = FIRST_BIG + 512


@pytest.fixture(scope="module")
def big_cache():
    """K and V caches of 4 GiB each ([blocks, 1 layer, 8 kv heads, 16, 128] bf16): blocks >= FIRST_BIG start at element
    offsets >= 2^31.  Only the blocks a test touches are ever written or read."""
    nbytes = 2 * BIG_BLOCKS * BIG_BLOCK_ELEMS * 2
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + (1 << 30):
        pytest.skip(f"needs {nbytes / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free (the GPU is shared)")
    kc = torch.empty(BIG_BLOCKS, 1, BIG_NKV, BS, D, dtype=torch.bfloat16, device=DEV)
    vc = torch.empty_like(kc)
    yield kc, vc
    del kc, vc
    torch.cuda.empty_cache()


def _big_layout(g, lens, kc, vc):
    """Block table over blocks straddling FIRST_BIG (most of them above), those blocks filled with random data.
    Returns the device table, the touched block ids and the same table remapped onto CPU copies of those blocks."""
    bt, nblk = _table(g, lens, base=FIRST_BIG - 16)
    assert FIRST_BIG - 16 + nblk <= BIG_BLOCKS
    ids = torch.arange(FIRST_BIG - 16, FIRST_BIG - 16 + nblk)
    kc[ids.to(DEV)] = torch.randn(nblk, 1, BIG_NKV, BS, D, generator=g).to(torch.bfloat16).to(DEV)
    vc[ids.to(DEV)] = torch.randn(nblk, 1, BIG_NKV, BS, D, generator=g).to(torch.bfloat16).to(DEV)
    bt_small = torch.where(bt >= 0, bt - (FIRST_BIG - 16), bt)
    return bt, ids, bt_small


def test_decode_element_offsets_past_2pow31(big_cache, paged_gen):
    """Pages on both sides of element offset 2^31, most of them above it."""
    kc, vc = big_cache
    lens = [1000, 333, 17, 2049, 1]
    g = torch.Generator().manual_seed(31)
    bt, ids, bt_small = _big_layout(g, lens, kc, vc)
    assert int(bt.max()) * BIG_BLOCK_ELEMS >= 2 ** 31
    q = torch.randn(len(lens), BIG_NQ, D, generator=g).to(torch.bfloat16)
    sids = list(range(len(lens)))
    o = _paged_run(q, kc, vc, bt, sids, lens, D ** -0.5, BS, 0)
    o64 = K.paged_attention_exact(q, kc[ids.to(DEV)].cpu(), vc[ids.to(DEV)].cpu(), bt_small, sids, lens, D ** -0.5, BS, 0)
    check_attention(o, o64, BIG_NQ, lens, what="decode")


def test_paged_prefill_element_offsets_past_2pow31(big_cache, prefill_gen):
    from swiftllm_b200.worker.kernels.prefill_attn import prefill_attention_paged
    kc, vc = big_cache
    prefix, chunk = [700, 0, 13], [300, 129, 64]
    g = torch.Generator().manual_seed(32)
    bt, ids, bt_small = _big_layout(g, [p + c for p, c in zip(prefix, chunk)], kc, vc)
    starts = list(np.cumsum([0] + chunk[:-1]))
    q = torch.randn(sum(chunk), BIG_NQ, D, generator=g).to(torch.bfloat16)
    st = NS(num_prefill_seqs=3, seq_ids=i32([0, 1, 2]), prefill_seq_start_locs=i32(starts), prefill_seq_lens=i32(chunk),
            prefill_prefix_lens=i32(prefix), max_prefill_len=max(chunk), softmax_scale=D ** -0.5)
    o = torch.zeros(q.shape, dtype=q.dtype, device=DEV)
    prefill_attention_paged(q.to(DEV), kc, vc, bt.to(DEV), o, None, None, st, 0)
    o64 = K.prefix_prefill_attention_exact(q, kc[ids.to(DEV)].cpu(), vc[ids.to(DEV)].cpu(), bt_small.numpy(), [0, 1, 2], starts,
                                           chunk, prefix, D ** -0.5, BS, 0)
    check_attention(o, o64, BIG_NQ, chunk, starts=starts, prefix=prefix, what="paged_prefill")


def test_store_kvcache_element_offsets_past_2pow31(big_cache):
    """Prefill and decode rows stored into blocks past 2^31 elements, bit-exact with the oracle on CPU copies."""
    from swiftllm_b200.worker.kernels.kvcache_mgmt import store_kvcache
    kc, vc = big_cache
    plens, dlens = [300, 37], [900, 17]
    g = torch.Generator().manual_seed(33)
    bt, ids, bt_small = _big_layout(g, plens + dlens, kc, vc)
    kc0, vc0 = kc[ids.to(DEV)].cpu(), vc[ids.to(DEV)].cpu()
    Tp = sum(plens)
    k = torch.randn(Tp + len(dlens), BIG_NKV, D, generator=g).to(torch.bfloat16)
    v = torch.randn(Tp + len(dlens), BIG_NKV, D, generator=g).to(torch.bfloat16)
    starts = [0, plens[0]]
    K.store_kvcache_inplace(k, v, kc0, vc0, bt_small, [0, 1, 2, 3], starts, plens, dlens, 2, Tp, BS, 0)
    st = NS(seq_ids=i32([0, 1, 2, 3]), num_prefill_seqs=2, num_decoding_seqs=2, num_prefill_tokens=Tp,
            prefill_seq_start_locs=i32(starts), prefill_seq_lens=i32(plens), max_prefill_len=max(plens),
            decoding_seq_lens=i32(dlens))
    store_kvcache(k.to(DEV), v.to(DEV), kc, vc, bt.to(DEV), None, None, st, 0)
    assert torch.equal(kc[ids.to(DEV)].cpu().view(torch.int16), kc0.view(torch.int16))
    assert torch.equal(vc[ids.to(DEV)].cpu().view(torch.int16), vc0.view(torch.int16))


# ----------------------------------------------------------------------------- row-strided q
@pytest.mark.parametrize("dtype", DTYPES)
def test_fused_qkv_column_slices_gqa3(dtype, paged_gen, prefill_gen):
    """q as a column slice of the fused QKV output for GQA group 3 (24 / 8 heads): the wgmma decode kernel's 16-head Q
    box then covers the heads of the next kv heads, and for the last kv head runs past q head 23 (zero-filled)."""
    check_fused_qkv_column_slices(dtype, 24, 8)


# ----------------------------------------------------------------------------- speculative verification
# sllm_paged_attention_verify: entry i has rows j < rows_i at positions prefix_i + j, row j sees positions <= prefix_i + j.
# Splits come from the decode planner over entries x kv heads; each test asserts the regime it claims.
def verify_plan(B, T, nq, nkv, max_len):
    """(splits, candidate split lengths) of a verify launch, read back from its workspace ([T, nq, splits] partials of
    D + 1 floats, then T int32 row lengths; 0 bytes iff one split).  The planner's split length is a multiple of 128 in
    [256, 16384]; the candidates are those that give this many splits of max_len tokens."""
    from swiftllm_b200 import _lib
    ws = _lib.lib().sllm_paged_attention_verify_workspace_bytes(B, T, nq, nkv, D, max_len)
    if ws == 0:
        return 1, [PA_MAX_SPLIT_TOKENS]
    per_split = T * nq * (D + 1) * 4
    assert (ws - 4 * T) % per_split == 0, ws
    ns = (ws - 4 * T) // per_split
    return ns, [s for s in range(256, PA_MAX_SPLIT_TOKENS + 1, 128) if -(-max_len // s) == ns]


def verify_split_tokens(B, T, nq, nkv, max_len):
    """The split length of a launch whose split count pins it down (asserted)."""
    ns, cand = verify_plan(B, T, nq, nkv, max_len)
    assert ns > 1 and len(cand) == 1, f"{ns} split(s) of {max_len} tokens do not determine the split length: {cand}"
    return cand[0]


def _verify_raw(q, kc, vc, bt, rows, prefix, layer=0, ws=None):
    """sllm_paged_attention_verify through the C ABI into a NaN-filled output, entry i in block-table row i.  `ws` replaces
    the workspace the launch asks for (same size)."""
    from swiftllm_b200 import _lib
    l = _lib.lib()
    T, nq, _ = q.shape
    nblk, nl, nkv, bs, _ = kc.shape
    B, max_len = len(rows), max(p + n for p, n in zip(prefix, rows))
    need = l.sllm_paged_attention_verify_workspace_bytes(B, T, nq, nkv, D, max_len)
    if ws is None and need > 0:
        ws = torch.empty(need // 4, dtype=torch.float32, device=DEV)
    assert (0 if ws is None else 4 * ws.numel()) == need
    meta = [i32(range(B)), i32(np.cumsum([0] + list(rows[:-1]))), i32(rows), i32(prefix)]
    o = torch.full(q.shape, float("nan"), dtype=q.dtype, device=DEV)
    _lib.check(l.sllm_paged_attention_verify(
        q.data_ptr(), kc.data_ptr(), vc.data_ptr(), o.data_ptr(), bt.data_ptr(), *[t.data_ptr() for t in meta], _lib.ptr(ws),
        need, D ** -0.5, B, max(rows), max_len, T, layer, nl, nq, nkv, bs, D, bt.shape[1], nblk, _lib.row_stride(q),
        _lib.dtype_tag(q.dtype), _lib.stream()), "paged_attention_verify")
    torch.cuda.synchronize()
    return o


def _verify_case(g, rows, prefix, nq, nkv, dtype, layers=1, extra_blocks=0):
    """Random caches, a block table over permuted blocks (entry i in row i) and packed q, all on the CPU."""
    bt, nblk = _table(g, [p + n for p, n in zip(prefix, rows)], extra_blocks)
    kc, vc, q = random_kv_q(g, nblk, layers, nkv, sum(rows), nq, D, BS, dtype)
    return q, kc, vc, bt


def _verify_exact(q, kc, vc, bt, rows, prefix, layer=0):
    starts = list(np.cumsum([0] + list(rows[:-1])))
    return K.prefix_prefill_attention_exact(q, kc, vc, bt.numpy(), range(len(rows)), starts, rows, prefix, D ** -0.5, BS, layer)


def _check_verify(o, o64, nq, rows, prefix, what):
    starts = list(np.cumsum([0] + list(rows[:-1])))
    return check_attention(o, o64, nq, rows, starts=starts, prefix=prefix, what=what)


def _dev(*ts):
    return [t.to(DEV) for t in ts]


def _what(verify_gen, nq, nkv, rows):
    """Kernel label of a check: the wgmma verify kernel with the N its launch uses, or the paged-prefill fallback."""
    if verify_gen != "wgmma":
        return "paged_attention_verify(fallback)"
    npad = verify_np(nq // nkv, max(rows))
    assert npad is not None, "a shape the wgmma verify kernel serves"
    return f"paged_attention_verify(wgmma, np{npad})"


@pytest.fixture
def wgmma_verify(monkeypatch):
    """sllm_paged_attention_verify must be served by the wgmma verify kernel (anything else is an error)."""
    monkeypatch.setenv("SLLM_PAGED_ATTN_GEN", "2")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("long_prefix,splits", [(None, 1), (PA_MAX_SPLIT_TOKENS - 3, 2)], ids=["one-split", "two-splits"])
def test_verify_single_pass_regime(dtype, long_prefix, splits, wgmma_verify):
    """Entries x kv heads >= 6 x SMs: each persistent CTA runs several (entry, kv head) items and writes o directly (no
    workspace).  With one entry at prefix 16384 - 3 and 8 rows the launch has two 16384-token splits: rows 0-2 of that entry
    see only split 0 (the merge must read no partial of split 1 for them), rows 3-7 also see split 1."""
    nq, nkv = 32, 8                                                      # g4 x 8 rows: N = 32
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = -(-6 * sms // nkv) + 3
    rng = np.random.default_rng(B)
    rows = [1 + i % 8 for i in range(B)]
    prefix = rng.integers(0, 700, size=B).tolist()
    prefix[:8] = [0, 1, 15, 16, 120, 127, 128, 2040]
    if long_prefix is not None:
        rows[0], prefix[0] = 8, long_prefix
    T, max_len = sum(rows), max(p + n for p, n in zip(prefix, rows))
    assert verify_plan(B, T, nq, nkv, PA_MAX_SPLIT_TOKENS)[0] == 1, "the batch alone must select the single-pass regime"
    assert verify_plan(B, T, nq, nkv, max_len)[0] == splits
    if long_prefix is not None:                      # single pass: the planner's split length is PA_MAX_SPLIT_TOKENS
        seen = [-(-(long_prefix + j + 1) // PA_MAX_SPLIT_TOKENS) for j in range(8)]
        assert seen == [1, 1, 1, 2, 2, 2, 2, 2]
    g = torch.Generator().manual_seed(B + splits)
    q, kc, vc, bt = _verify_case(g, rows, prefix, nq, nkv, dtype)
    o64 = _verify_exact(q, kc, vc, bt, rows, prefix)
    o = _verify_raw(*_dev(q, kc, vc, bt), rows, prefix)
    _check_verify(o, o64, nq, rows, prefix, _what("wgmma", nq, nkv, rows))


@pytest.mark.parametrize("dtype", DTYPES)
def test_verify_split_straddle_with_poisoned_workspace(dtype, wgmma_verify):
    """Entries whose rows straddle split boundaries k * split_tokens (split length read back from the workspace size), run
    with a workspace full of NaN (row lengths -1): the output is finite and within tolerance of fp64, so the kernel wrote
    every row's length and the merge read no partial of a split the row does not see (whether such a partial is also
    written is not observable here: the merge never reads that slot).  An entry ending exactly at a boundary has no item
    past it."""
    nq, nkv = 24, 8                                                      # g3 x 8 rows: N = 32, 8 dead columns
    rows = [8, 8, 8, 6, 8]
    last = 4000 - 8                                                      # fixes max_len, hence the split length
    B, T = len(rows), sum(rows)
    st = verify_split_tokens(B, T, nq, nkv, last + 8)
    prefix = [st - 3, 5 * st - 1, 3 * st - 8, 7 * st - 5, last]
    assert max(p + n for p, n in zip(prefix, rows)) == last + 8
    for i in (0, 1, 3):                                                  # the premise: rows of one entry see different splits
        seen = {-(-(prefix[i] + j + 1) // st) for j in range(rows[i])}
        assert len(seen) == 2, (i, st, seen)
    assert (prefix[2] + rows[2]) % st == 0
    g = torch.Generator().manual_seed(st)
    q, kc, vc, bt = _verify_case(g, rows, prefix, nq, nkv, dtype)
    o64 = _verify_exact(q, kc, vc, bt, rows, prefix)
    ns = verify_plan(B, T, nq, nkv, last + 8)[0]
    ws = torch.full((T * nq * ns * (D + 1) + T,), float("nan"), dtype=torch.float32, device=DEV)
    ws[T * nq * ns * (D + 1):].view(torch.int32).fill_(-1)        # an unwritten row length makes its row NaN, never a wild read
    o = _verify_raw(*_dev(q, kc, vc, bt), rows, prefix, ws=ws)
    assert torch.isfinite(o.float()).all()
    _check_verify(o, o64, nq, rows, prefix, _what("wgmma", nq, nkv, rows))


@pytest.mark.parametrize("dtype", DTYPES)
def test_verify_peaked_rows(dtype, verify_gen):
    """The verify counterpart of test_decode_peaked_rows: per (entry, kv head) one key at draft position prefix + j0
    dominates by more than 150 (log2 units).  Rows below j0 do not see it and match fp64 (a causal leak inside the entry would
    be a gross error); rows j0 and above return its V up to the output rounding.  Sinks: in the first tile, in the last split
    but not its last tile, at a split's first token, and at the entry's last position."""
    nq, nkv = 24, 8
    rows = [8, 8, 8, 6]
    last = 4000 - 8
    B, T = len(rows), sum(rows)
    st = verify_split_tokens(B, T, nq, nkv, last + 8)
    s1 = 10 * st + 126                                                   # first tile of the last split of entry 1
    prefix = [3, s1 - 3, last, 8 * st - 4]
    j0 = [2, 3, 7, 4]
    sink = [p + j for p, j in zip(prefix, j0)]
    n1 = prefix[1] + rows[1]
    assert sink[1] // st == (n1 - 1) // st and (sink[1] % st) // 128 != ((n1 - 1) % st) // 128
    assert sink[0] < 128 and sink[2] == prefix[2] + rows[2] - 1 and sink[3] % st == 0
    g = torch.Generator().manual_seed(151)
    bt, nblk = _table(g, [p + n for p, n in zip(prefix, rows)])
    kc = torch.randn(nblk, 1, nkv, BS, D, generator=g); vc = torch.randn(nblk, 1, nkv, BS, D, generator=g)
    u = torch.randint(0, 2, (B, nkv, D), generator=g).float() * 2 - 1
    q = 0.3 * torch.randn(T, nq, D, generator=g) + u.repeat_interleave(nq // nkv, dim=1).repeat_interleave(torch.tensor(rows), dim=0)
    for e, j in enumerate(sink):
        kc[int(bt[e, j // BS]), 0, :, j % BS] = 16 * u[e]
    q, kc, vc = q.to(dtype), kc.to(dtype), vc.to(dtype)
    o64 = _verify_exact(q, kc, vc, bt, rows, prefix)
    c = D ** -0.5 * K.LOG2E
    starts = list(np.cumsum([0] + rows[:-1]))
    for e in range(B):                                                   # the premise: a gap of more than 150 (log2 units)
        n = prefix[e] + rows[e]
        keys = torch.cat([kc[int(b), 0] for b in bt[e, :(n + BS - 1) // BS]], dim=1)[:, :n].double()   # [nkv, n, D]
        for j in range(j0[e], rows[e]):
            qe = q[starts[e] + j].double().view(nkv, nq // nkv, D)
            sc = torch.einsum("khd,knd->khn", qe, keys[:, :prefix[e] + j + 1]) * c
            others = torch.cat([sc[..., :sink[e]], sc[..., sink[e] + 1:]], dim=-1)
            assert float((sc[..., sink[e]] - others.amax(-1)).min()) > 150
    o = _verify_raw(*_dev(q, kc, vc, bt), rows, prefix).cpu()
    _check_verify(o, o64, nq, rows, prefix, _what(verify_gen, nq, nkv, rows))
    # the output rounding; the fallback's lazy reference point also rounds the sink's own weight p before P.V
    u_out = (2.0 ** -11 if dtype == torch.float16 else 2.0 ** -8) * (1 if verify_gen == "wgmma" else 2)
    for e, j in enumerate(sink):
        v = vc[int(bt[e, j // BS]), 0, :, j % BS].float().repeat_interleave(nq // nkv, dim=0)   # [nq, D]
        for r in range(j0[e], rows[e]):
            got = o[starts[e] + r].float()
            assert ((got - v).abs() <= u_out * v.abs()).all(), f"entry {e} row {r}: output is not the sink's V"


@pytest.mark.parametrize("dtype", DTYPES)
def test_verify_poisoned_pages_are_harmless(dtype, verify_gen):
    """NaN in every block the batch does not own and in the other layer; slots of an entry's last page past its last
    position hold NaN K and V = 3e4.  More work items than SMs, so the wgmma kernel's CTAs reuse their K / V rings across
    items and short tail tiles meet slots an earlier item loaded."""
    nq, nkv, layer = 24, 8, 1
    B = 40
    rng = np.random.default_rng(40)
    rows = [1 + i % 8 for i in range(B)]
    prefix = rng.integers(0, 900, size=B).tolist()
    prefix[:6] = [0, 16 - 2, 129, 511, 1000, 2047]
    T, max_len = sum(rows), max(p + n for p, n in zip(prefix, rows))
    ns = verify_plan(B, T, nq, nkv, max_len)[0]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert B * nkv * ns > sms, "every CTA must run more than one item"
    g = torch.Generator().manual_seed(41)
    q, kc, vc, bt = _verify_case(g, rows, prefix, nq, nkv, dtype, layers=2, extra_blocks=7)
    o64 = _verify_exact(q, kc, vc, bt, rows, prefix, layer)
    owned = set()
    for e, (p, r) in enumerate(zip(prefix, rows)):
        n = p + r
        npg = (n + BS - 1) // BS
        owned |= set(bt[e, :npg].tolist())
        lastb = int(bt[e, npg - 1])
        kc[lastb, layer, :, n - (npg - 1) * BS:] = float("nan"); vc[lastb, layer, :, n - (npg - 1) * BS:] = 3.0e4
    kc[:, 1 - layer] = float("nan"); vc[:, 1 - layer] = float("nan")
    for b in range(kc.shape[0]):
        if b not in owned:
            kc[b] = float("nan"); vc[b] = float("nan")
    o = _verify_raw(*_dev(q, kc, vc, bt), rows, prefix, layer)
    assert torch.isfinite(o.float()).all()
    _check_verify(o, o64, nq, rows, prefix, _what(verify_gen, nq, nkv, rows))


def test_verify_element_offsets_past_2pow31(big_cache, verify_gen):
    """Pages on both sides of element offset 2^31, most of them above it (g3 x 8 rows: N = 32)."""
    kc, vc = big_cache
    rows, prefix = [8, 3, 8, 5, 1], [1000, 333, 17, 2049, 0]
    g = torch.Generator().manual_seed(34)
    bt, ids, bt_small = _big_layout(g, [p + n for p, n in zip(prefix, rows)], kc, vc)
    assert int(bt.max()) * BIG_BLOCK_ELEMS >= 2 ** 31
    q = torch.randn(sum(rows), BIG_NQ, D, generator=g).to(torch.bfloat16)
    o = _verify_raw(q.to(DEV), kc, vc, bt.to(DEV), rows, prefix)
    o64 = _verify_exact(q, kc[ids.to(DEV)].cpu(), vc[ids.to(DEV)].cpu(), bt_small, rows, prefix)
    _check_verify(o, o64, BIG_NQ, rows, prefix, _what(verify_gen, BIG_NQ, BIG_NKV, rows))


@pytest.mark.parametrize("dtype", DTYPES)
def test_verify_bit_exact_repeat_and_block_permutation(dtype, verify_gen):
    """A second call gives the same bits, and so does the same cache stored in permuted physical blocks with the block
    table remapped: the result depends on the tokens, not on where their pages live (g7 x 4 rows: N = 32, split launch)."""
    nq, nkv = 28, 4
    rows, prefix = [4, 1, 3, 4], [2999, 0, 1500, 700]
    g = torch.Generator().manual_seed(7)
    q, kc, vc, bt = _verify_case(g, rows, prefix, nq, nkv, dtype)
    assert verify_plan(len(rows), sum(rows), nq, nkv, max(p + n for p, n in zip(prefix, rows)))[0] > 1
    o1 = _verify_raw(*_dev(q, kc, vc, bt), rows, prefix)
    o2 = _verify_raw(*_dev(q, kc, vc, bt), rows, prefix)
    perm = torch.randperm(kc.shape[0], generator=g)
    kp, vp = torch.empty_like(kc), torch.empty_like(vc)
    kp[perm] = kc; vp[perm] = vc
    btp = torch.where(bt >= 0, perm.to(torch.int32)[bt.clamp_min(0).long()], bt)
    o3 = _verify_raw(*_dev(q, kp, vp, btp), rows, prefix)
    assert torch.equal(o1.view(torch.int16), o2.view(torch.int16))
    assert torch.equal(o1.view(torch.int16), o3.view(torch.int16))
    _check_verify(o1, _verify_exact(q, kc, vc, bt, rows, prefix), nq, rows, prefix, _what(verify_gen, nq, nkv, rows))
