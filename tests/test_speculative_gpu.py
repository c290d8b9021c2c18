"""GPU: speculative verification - the multi-query paged-attention kernel (sllm_paged_attention_verify) against the fp64
definition for every (entry, q head, row), and LlamaModel.forward_speculative end to end."""
import functools
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import sampling_oracle as SO
from attention_check import TOL, check_attention
from oracle import kernels as K
from oracle.model import OracleLlama, OracleWeights
from test_model_gpu import ENG2, TINY2, _make_model
from verify_shapes import LAYOUTS, VERIFY_GEOMS, geom_id, random_kv_q, verify_layout, verify_np

pytestmark = pytest.mark.gpu
DEV = "cuda"
D, BS, LAYERS, LAYER = 128, 16, 2, 1


def _i32(x):
    return torch.tensor(list(x), dtype=torch.int32, device=DEV)


@pytest.fixture(params=["wgmma", "fallback"])
def verify_gen(request, monkeypatch):
    """Which kernel serves sllm_paged_attention_verify: the wgmma verify kernel (SLLM_PAGED_ATTN_GEN=2, where a shape it does
    not serve is an error) or the paged-prefill kernel it falls back to (=1).  The 1-row decode comparisons then run the
    wgmma decode kernel and the mma.sync decode kernel respectively."""
    monkeypatch.setenv("SLLM_PAGED_ATTN_GEN", "2" if request.param == "wgmma" else "1")
    return request.param


def fused_q(q, nkv):
    """q [T, nq, D] as the column slice of a [T, (nq + 2 nkv) D] buffer (the fused QKV GEMM's output) whose k / v columns
    hold NaN: the kernel sees q's row stride (nq + 2 nkv) D and must never read past q's own columns."""
    T, nq, D_ = q.shape
    buf = torch.full((T, (nq + 2 * nkv) * D_), float("nan"), dtype=q.dtype, device=q.device)
    buf[:, :nq * D_] = q.reshape(T, -1)
    return buf[:, :nq * D_].unflatten(1, (nq, D_))


def _case(g_, nkv, rows, prefix, dtype, seed, mbps=None):
    """Random caches (2 layers, layer 1 used), a block table over randomly permuted block ids with entry i in table row 2 i + 1,
    packed q; returns the device tensors, the metadata and the fp64 output.  rows / prefix: tuples."""
    c = _inputs(g_, nkv, rows, prefix, dtype, seed, mbps)
    o64 = _exact(g_, nkv, rows, prefix, dtype, seed, mbps)
    return dict(c, q=c["q"].to(DEV), kc=c["kc"].to(DEV), vc=c["vc"].to(DEV), bt=c["bt"].to(DEV), o64=o64)


@functools.lru_cache(maxsize=None)        # the fp64 outputs (small) are shared by the two kernels
def _exact(*key):
    c = _inputs(*key)
    return K.prefix_prefill_attention_exact(c["q"], c["kc"], c["vc"], c["bt"].numpy(), c["sids"], c["starts"], c["rows"],
                                            c["prefix"], D ** -0.5, BS, LAYER)


def _inputs(g_, nkv, rows, prefix, dtype, seed, mbps):
    gen = torch.Generator().manual_seed(seed)
    nq = nkv * g_
    need = [(p + n + BS - 1) // BS for p, n in zip(prefix, rows)]
    mbps = mbps or max(need) + 1
    nblk = sum(need) + 5
    perm = torch.randperm(nblk, generator=gen)
    bt = torch.full((2 * len(rows) + 1, mbps), -1, dtype=torch.int32)
    at = 0
    for i, n in enumerate(need):
        bt[2 * i + 1, :n] = perm[at:at + n].to(torch.int32); at += n
    kc, vc, q = random_kv_q(gen, nblk, LAYERS, nkv, sum(rows), nq, D, BS, dtype)
    starts = list(np.cumsum([0] + list(rows[:-1])))
    sids = [2 * i + 1 for i in range(len(rows))]
    return dict(q=q, kc=kc, vc=vc, bt=bt, sids=sids, starts=starts, rows=list(rows), prefix=list(prefix), nq=nq)


def _verify(c, q=None):
    """paged_attention_verify on the case (q defaults to the case's contiguous q) into a NaN-filled output."""
    from swiftllm_b200.worker.kernels.prefill_attn import paged_attention_verify
    q = c["q"] if q is None else q
    st = SimpleNamespace(seq_ids=_i32(c["sids"]), prefill_prefix_lens=_i32(c["prefix"]), num_prefill_seqs=len(c["rows"]),
                         max_prefill_kv_len=max(p + n for p, n in zip(c["prefix"], c["rows"])),
                         prefill_seq_start_locs=_i32(c["starts"]), prefill_seq_lens=_i32(c["rows"]), max_prefill_len=max(c["rows"]),
                         softmax_scale=D ** -0.5)
    o = torch.full(q.shape, float("nan"), dtype=q.dtype, device=DEV)
    paged_attention_verify(q, c["kc"], c["vc"], c["bt"], o, None, None, st, LAYER)
    torch.cuda.synchronize()
    return o


def _paged_rows(c):
    """sllm_paged_attention with every row as a decode sequence: row j of entry i at length prefix_i + j + 1."""
    from swiftllm_b200.worker.kernels.paged_attn import paged_attention
    sids = [s for s, n in zip(c["sids"], c["rows"]) for _ in range(n)]
    lens = [p + j + 1 for p, n in zip(c["prefix"], c["rows"]) for j in range(n)]
    st = SimpleNamespace(paged_attn_seq_block_size=0, seq_ids=_i32(sids), num_prefill_seqs=0,
                         decoding_seq_lens=_i32(lens), max_decoding_len=max(lens), softmax_scale=D ** -0.5)
    q = c["q"].contiguous()
    o = torch.empty((q.shape[0], c["nq"] * D), dtype=q.dtype, device=DEV)
    paged_attention(q, c["kc"], c["vc"], c["bt"], None, SimpleNamespace(block_size=BS), st, LAYER, o)
    torch.cuda.synchronize()
    return o, lens


def _workspace_splits(c, nkv):
    from swiftllm_b200 import _lib
    T = sum(c["rows"])
    ws = _lib.lib().sllm_paged_attention_verify_workspace_bytes(len(c["rows"]), T, c["nq"], nkv, D,
                                                                 max(p + n for p, n in zip(c["prefix"], c["rows"])))
    return 1 if ws == 0 else (ws - 4 * T) // (T * c["nq"] * (D + 1) * 4)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("geom", VERIFY_GEOMS, ids=geom_id)
@pytest.mark.parametrize("regime", LAYOUTS)
def test_verify_kernel_vs_fp64(dtype, geom, regime, verify_gen):
    """Every (entry, q head, row) within the decode-attention tolerance of fp64, under both kernels; under `wgmma` a shape of
    more than 32 columns must be refused.  q is a column slice of a fused QKV buffer (NaN k / v columns) in short_many and
    contiguous in long_few.  Row j of every entry also agrees with sllm_paged_attention at length prefix + j + 1."""
    g_, nkv, max_rows, npad = geom
    rows, prefix = verify_layout(regime, g_, max_rows)
    rows = tuple(rows)
    assert verify_np(g_, max(rows)) == npad, "the rows must give the launch the intended wgmma width"
    mbps = 256 if regime == "long_few" else None
    c = _case(g_, nkv, rows, tuple(prefix), dtype, seed=3, mbps=mbps)
    if regime == "long_few":
        assert _workspace_splits(c, nkv) > 1
    q = fused_q(c["q"], nkv) if regime == "short_many" else c["q"]
    if verify_gen == "wgmma" and npad is None:
        with pytest.raises(RuntimeError, match="SLLM_PAGED_ATTN_GEN=2"):
            _verify(c, q)
        return
    o = _verify(c, q)
    check_attention(o, c["o64"], c["nq"], c["rows"], starts=c["starts"], prefix=c["prefix"],
                    what=f"paged_attention_verify(wgmma, np{npad})" if verify_gen == "wgmma" else "paged_attention_verify(fallback)")
    op, lens = _paged_rows(c)
    check_attention(o.reshape(len(lens), -1), op.double(), c["nq"], lens, tol=2 * TOL[dtype], what="verify vs paged_attention")


def _oracle(w, tdt, cfg=TINY2):
    return OracleLlama(cfg, w, block_size=16, num_blocks=ENG2["num_blocks"], num_cpu_blocks=4, max_seqs_in_block_table=16,
                       max_blocks_per_seq=16, attn="exact", dtype=tdt)


# GQA group 3 at head_dim 128 (12 q / 4 kv heads): the verify kernel runs with 8 dead columns at 8 rows (N = 32) and one at
# 5 rows (N = 16), on q sliced from the fused QKV output
TINY3 = dict(TINY2, num_attention_heads=12, num_key_value_heads=4, hidden_size=1536)
E2E_CASES = {"g4-np32": (TINY2, [8, 1, 5], 32), "g3-np32": (TINY3, [8, 1, 5], 32), "g3-np16": (TINY3, [5, 1, 3], 16)}


@pytest.mark.parametrize("dtype", ["bfloat16", "float16"])
@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "sampled"])
@pytest.mark.parametrize("model", list(E2E_CASES))
def test_forward_speculative_end_to_end(dtype, sampled, model, monkeypatch):
    """Per-row logits within test_model_gpu's tolerance of the oracle fed the rows one at a time; greedy tokens equal the
    oracle's where the top-1 margin is clear; sampled tokens equal the sampling restatement applied to the product's own logits
    rows with pos = prefix + j + 1 (exact); the device block state matches the host mirror and ceil(len / bs) afterwards.
    The verify attention must be served by the wgmma verify kernel at the intended width."""
    from swiftllm_b200 import SamplingParams
    cfg, rows, npad = E2E_CASES[model]
    assert verify_np(cfg["num_attention_heads"] // cfg["num_key_value_heads"], max(rows)) == npad
    monkeypatch.setenv("SLLM_PAGED_ATTN_GEN", "2")           # a shape the wgmma kernels do not serve is an error
    tdt = dict(bfloat16=torch.bfloat16, float16=torch.float16)[dtype]
    tol = 2 ** -5 if dtype == "bfloat16" else 4e-3
    w = OracleWeights.random(cfg, dtype=tdt, seed=3, std=0.05)
    m, o = _make_model(cfg, ENG2, w, dtype=dtype), _oracle(w, tdt, cfg)
    rng = np.random.default_rng(2)
    plens = [15, 16, 33]
    sids = [7, 1, 4]
    prompts = [rng.integers(0, 1000, size=n).tolist() for n in plens]
    first = o.forward(prompts, sids, [])
    m.forward(prompts, sids, [])
    entries = [[x] + rng.integers(0, 1000, size=n - 1).tolist() for x, n in zip(first, rows)]
    params = [SamplingParams(0.8, top_k=(0, 50, 0)[i], seed=9 + i) for i in range(3)] if sampled else None
    out = m.forward_speculative(entries, sids, plens, params)
    got = m.post_layer.last_logits.float().cpu()
    ref = []
    for e, s, p in zip(entries, sids, plens):
        for j, t in enumerate(e):
            o.forward([[t]], [s], [], prefill_prefix_lens_list=[p + j])
            ref.append(o.last_logits[0].float())
    ref = torch.stack(ref)
    assert float((got - ref).abs().max() / ref.abs().max()) <= tol
    if sampled:
        rep = np.repeat(np.arange(3), rows)
        pos = [p + j + 1 for p, n in zip(plens, rows) for j in range(n)]
        y = [r.token for r in SO.sample_tokens(m.post_layer.last_logits, [params[i].temperature for i in rep],
                                               [params[i].top_k for i in rep], [params[i].top_p for i in rep],
                                               [params[i].seed for i in rep], pos)]
    else:
        top2 = ref.topk(2, dim=1).values
        clear = (top2[:, 0] - top2[:, 1]) > 2 * tol * ref.abs().max()
        y = torch.argmax(got, dim=1).tolist()
        assert torch.equal(torch.argmax(got, dim=1)[clear], torch.argmax(ref, dim=1)[clear])
    s = 0
    for e, n, res in zip(entries, rows, out):
        k = 0
        while k < n - 1 and e[k + 1] == y[s + k]:
            k += 1
        assert res == y[s:s + k + 1]
        s += n
    bm = m.gpu_block_manager
    nsab = bm.num_seq_allocated_blocks.cpu().numpy()
    free = bm.is_block_free.cpu().numpy()
    for sid, p, res in zip(sids, plens, out):
        assert nsab[sid] == bm._host_nsab[sid] == (p + len(res) + BS - 1) // BS
    assert int(free.sum()) == bm.num_free_blocks
    used = np.concatenate([bm.block_table[sid, :nsab[sid]].cpu().numpy() for sid in sids])
    assert not free[used].any()


def _agrees(tokens, expected, logits, tol):
    """True when the tokens equal the plain run's.  A first difference is only allowed at a row whose top-1 margin is not
    clear (the verify step's GEMMs round differently from a decode step's); the comparison of the run then stops."""
    for i, (a, b) in enumerate(zip(tokens, expected)):
        if a != b:
            row = logits[i].float()
            top2 = row.topk(2).values
            assert float(top2[0] - top2[1]) <= 2 * tol * float(row.abs().max()), (i, a, b)
            return False
    return True


def test_greedy_speculation_reproduces_plain_greedy_run():
    """Drafts from a plain greedy run with one wrong draft per step: every call returns the plain run's tokens (accepted
    prefix + the correction), and plain decoding continues the sequence to the same tokens, up to a near-tie."""
    tol = 4e-3
    w = OracleWeights.random(TINY2, dtype=torch.float16, seed=5, std=0.05)
    rng = np.random.default_rng(4)
    prompt = rng.integers(0, 1000, size=29).tolist()
    plain_m = _make_model(TINY2, ENG2, w, dtype="float16")
    plain = plain_m.forward([prompt], [2], [])
    for j in range(30):
        plain += plain_m.forward([[plain[-1]]], [2], [len(prompt) + j + 1])
    m = _make_model(TINY2, ENG2, w, dtype="float16")
    got = m.forward([prompt], [2], [])
    L = len(prompt)
    for k, wrong in [(7, 4), (3, None), (5, 0), (6, 5)]:
        drafts = plain[len(got):len(got) + k]
        if wrong is not None:
            drafts[wrong] = (drafts[wrong] + 1) % 1000
        out = m.forward_speculative([[got[-1]] + drafts], [2], [L])[0]
        if not _agrees(out, plain[len(got):], m.post_layer.last_logits, tol):
            return
        assert len(out) == (k if wrong is None else wrong) + 1
        got += out
        L += len(out)
        assert m.gpu_block_manager.num_seq_allocated_blocks[2].item() == (L + BS - 1) // BS
    while len(got) < len(plain):
        t = m.forward([[got[-1]]], [2], [L + 1])
        if not _agrees(t, plain[len(got):], m.post_layer.last_logits, tol):
            return
        got += t
        L += 1
    assert got == plain
