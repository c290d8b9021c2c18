"""GPU: chunked ("prefix-aware") prefill - SURVEY.md §8 f-1 - through the C ABI:
  sllm_store_kvcache_chunked      bit-exact vs the oracle (pages entered in the middle, ragged chunks, mixed with decode rows)
  sllm_prefill_attention_paged    both kernel generations vs the fp64 definition; with prefix 0 vs sllm_prefill_attention
  LlamaModel.forward(..., prefill_prefix_lens_list=...)   chunked == whole-prompt (tokens exact, logits within tolerance)

Part of the default `-m gpu` suite."""
import types

import numpy as np
import pytest
import torch

from attention_check import check_attention
from oracle import kernels as K
from oracle.model import OracleLlama, OracleWeights

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.float16, torch.bfloat16]


def NS(**kw):
    return types.SimpleNamespace(**kw)


def i32(x):
    return torch.as_tensor(np.asarray(x), dtype=torch.int32).to(DEV)


@pytest.fixture(params=["gen2-tcgen05", "gen1-mma.sync"])
def prefill_gen(request, monkeypatch):
    monkeypatch.setenv("SLLM_PREFILL_ATTN_GEN", "1" if request.param.startswith("gen1") else "0")
    return request.param


def _layout(g, prefix, chunk, bs, extra_seqs=3, extra_blocks=5):
    """Random block table for sequences of length prefix_i + chunk_i (+ unused rows / blocks)."""
    need = [(p + c + bs - 1) // bs for p, c in zip(prefix, chunk)]
    nblk = sum(need) + extra_blocks
    perm = torch.randperm(nblk, generator=g).tolist()
    sids = torch.randperm(len(chunk) + extra_seqs, generator=g)[: len(chunk)].tolist()
    bt = torch.full((len(chunk) + extra_seqs, max(need) + 2), -1, dtype=torch.int32)
    p = 0
    for s, n in zip(sids, need):
        bt[s, :n] = torch.tensor(perm[p:p + n], dtype=torch.int32); p += n
    return bt, sids, nblk


# ----------------------------------------------------------------------------- store
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("bs", [16, 32])
def test_store_kvcache_chunked_bit_exact(dtype, bs):
    from swiftllm_b200.worker.kernels.kvcache_mgmt import store_kvcache
    nkv, D, L, layer = 2, 128, 3, 1
    prefix = [0, 13, 16, 31, 100, 7]
    chunk = [5, 20, 16, 1, 77, 64]
    dec_lens = [9, 33]                                         # two decoding rows after the prefill tokens
    g = torch.Generator().manual_seed(bs)
    bt, sids, nblk = _layout(g, prefix + [0, 0], chunk + dec_lens, bs)
    starts = list(np.cumsum([0] + chunk[:-1]))
    Tp = sum(chunk); Tn = Tp + len(dec_lens)
    k = torch.randn(Tn, nkv, D, generator=g).to(dtype); v = torch.randn(Tn, nkv, D, generator=g).to(dtype)
    kc = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype); vc = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype)
    kc_o, vc_o = kc.clone(), vc.clone()
    K.store_kvcache_inplace(k, v, kc_o, vc_o, bt.numpy(), sids, starts, chunk, dec_lens, len(chunk), Tp, bs, layer,
                            prefill_prefix_lens=prefix)
    st = NS(seq_ids=i32(sids), prefill_seq_start_locs=i32(starts), prefill_seq_lens=i32(chunk), decoding_seq_lens=i32(dec_lens),
            num_prefill_seqs=len(chunk), num_decoding_seqs=len(dec_lens), num_prefill_tokens=Tp, max_prefill_len=max(chunk),
            prefill_prefix_lens=i32(prefix))
    kd, vd = kc.to(DEV), vc.to(DEV)
    store_kvcache(k.to(DEV), v.to(DEV), kd, vd, bt.to(DEV), None, None, st, layer)
    assert torch.equal(kd.cpu().view(torch.int16), kc_o.view(torch.int16))
    assert torch.equal(vd.cpu().view(torch.int16), vc_o.view(torch.int16))


# ----------------------------------------------------------------------------- attention
def _paged_prefill_run(q, kc, vc, bt, sids, starts, chunk, prefix, scale, layer):
    from swiftllm_b200.worker.kernels.prefill_attn import prefill_attention_paged
    st = NS(num_prefill_seqs=len(chunk), seq_ids=i32(sids), prefill_seq_start_locs=i32(starts), prefill_seq_lens=i32(chunk),
            prefill_prefix_lens=i32(prefix), max_prefill_len=int(max(chunk)), softmax_scale=scale)
    o = torch.zeros(q.shape, dtype=q.dtype, device=DEV)
    prefill_attention_paged(q.to(DEV), kc.to(DEV), vc.to(DEV), bt.to(DEV), o, None, None, st, layer)
    torch.cuda.synchronize()
    return o.cpu()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("geom", [dict(nq=4, nkv=2, D=64, bs=16), dict(nq=8, nkv=2, D=128, bs=16), dict(nq=4, nkv=4, D=128, bs=16),
                                  dict(nq=8, nkv=2, D=128, bs=32),
                                  # GQA groups that are not powers of two: 3 (head_dim 64 and 128), 5, 6, 7, 12
                                  dict(nq=12, nkv=4, D=64, bs=16), dict(nq=24, nkv=8, D=128, bs=16), dict(nq=40, nkv=8, D=128, bs=16),
                                  dict(nq=12, nkv=2, D=128, bs=16), dict(nq=28, nkv=4, D=128, bs=16), dict(nq=24, nkv=2, D=128, bs=16)])
def test_prefill_attention_paged_vs_exact_oracle(dtype, geom, prefill_gen):
    nq, nkv, D, bs = geom["nq"], geom["nkv"], geom["D"], geom["bs"]
    if (D == 64 or bs != 16) and prefill_gen.startswith("gen2"):
        pytest.skip("the wgmma kernel serves head_dim 128 / block_size 16; other shapes run gen 1")
    L, layer = 2, 1
    #          no prefix | mid-page prefix | page-aligned | 1-token chunk deep in a sequence | chunk > 256 rows (several CTAs) | tiny
    prefix = [0,   13,  64, 500, 100, 3, 255, 0]
    chunk = [37, 200, 64,   1, 513, 2, 257, 300]
    g = torch.Generator().manual_seed(nq * 100 + D + bs)
    bt, sids, nblk = _layout(g, prefix, chunk, bs)
    starts = list(np.cumsum([0] + chunk[:-1]))
    Tn = sum(chunk) + 5                                        # trailing rows (decode tokens of a mixed batch) stay untouched
    q = torch.randn(Tn, nq, D, generator=g).to(dtype)
    kc = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype); vc = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype)
    o64 = K.prefix_prefill_attention_exact(q, kc, vc, bt.numpy(), sids, starts, chunk, prefix, D ** -0.5, bs, layer)
    o = _paged_prefill_run(q, kc, vc, bt, sids, starts, chunk, prefix, D ** -0.5, layer)
    assert torch.isfinite(o.float()).all()
    check_attention(o, o64, nq, chunk, starts=starts, prefix=prefix, what="paged_prefill")
    assert (o[sum(chunk):] == 0).all()


@pytest.mark.parametrize("dtype", DTYPES)
def test_prefill_attention_paged_nan_in_unowned_pages_is_harmless(dtype, prefill_gen):
    """Blocks the sequence does not own may hold anything (NaN here): they are never loaded.  Slots of the LAST owned page past the
    sequence end are loaded by the TMA kernel (whole pages): their K may be NaN (the tail mask is a select), their V is multiplied by
    P = 0 exactly, so it must be finite - as it always is in a cache that is zero-initialised and only receives finite K/V - but may
    be huge (3e4 here).  tests/test_kernel_logic_mirror_cpu.py holds the same contract on CPU."""
    nq, nkv, D, bs, L = 8, 2, 128, 16, 1
    prefix, chunk = [70], [21]                                 # kv length 91: last page holds 11 valid slots
    g = torch.Generator().manual_seed(9)
    bt, sids, nblk = _layout(g, prefix, chunk, bs)
    q = torch.randn(chunk[0], nq, D, generator=g).to(dtype)
    kc = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype); vc = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype)
    o64 = K.prefix_prefill_attention_exact(q, kc, vc, bt.numpy(), sids, [0], chunk, prefix, D ** -0.5, bs, 0)
    last = int(bt[sids[0], 5])
    kc[last, :, :, 11:] = float("nan"); vc[last, :, :, 11:] = 3.0e4
    owned = set(bt[sids[0], :6].tolist())
    for b in range(nblk):
        if b not in owned:
            kc[b] = float("nan"); vc[b] = float("nan")
    o = _paged_prefill_run(q, kc, vc, bt, sids, [0], chunk, prefix, D ** -0.5, 0)
    assert torch.isfinite(o.float()).all()
    check_attention(o, o64, nq, chunk, starts=[0], prefix=prefix, what="paged_prefill")


@pytest.mark.parametrize("dtype", DTYPES)
def test_prefill_attention_paged_zero_prefix_equals_packed_kernel(dtype, prefill_gen):
    """With every prefix 0 the paged kernel sees exactly the keys the packed kernel sees, in the same 64-token steps: the two
    must agree to the last bit (same MMA shapes, same softmax code; only the producer differs)."""
    from swiftllm_b200.worker.kernels.prefill_attn import prefill_attention
    from swiftllm_b200.worker.kernels.kvcache_mgmt import store_kvcache
    nq, nkv, D, bs, L = 8, 2, 128, 16, 2
    chunk = [300, 64, 1, 129]
    prefix = [0] * len(chunk)
    g = torch.Generator().manual_seed(3)
    bt, sids, nblk = _layout(g, prefix, chunk, bs)
    starts = list(np.cumsum([0] + chunk[:-1]))
    Tn = sum(chunk)
    q = torch.randn(Tn, nq, D, generator=g).to(dtype); k = torch.randn(Tn, nkv, D, generator=g).to(dtype)
    v = torch.randn(Tn, nkv, D, generator=g).to(dtype)
    kc = torch.zeros(nblk, L, nkv, bs, D, dtype=dtype, device=DEV); vc = torch.zeros_like(kc)
    st = NS(seq_ids=i32(sids), prefill_seq_start_locs=i32(starts), prefill_seq_lens=i32(chunk), decoding_seq_lens=i32([]),
            num_prefill_seqs=len(chunk), num_decoding_seqs=0, num_prefill_tokens=Tn, max_prefill_len=max(chunk),
            prefill_prefix_lens=i32(prefix), softmax_scale=D ** -0.5)
    store_kvcache(k.to(DEV), v.to(DEV), kc, vc, bt.to(DEV), None, None, st, 1)
    o_paged = _paged_prefill_run(q, kc.cpu(), vc.cpu(), bt, sids, starts, chunk, prefix, D ** -0.5, 1)
    o_packed = torch.zeros(q.shape, dtype=dtype, device=DEV)
    prefill_attention(q.to(DEV), k.to(DEV), v.to(DEV), o_packed, None, None, st)
    assert torch.equal(o_paged.view(torch.int16), o_packed.cpu().view(torch.int16))


def test_prefill_attention_paged_sarathi_shape_property(prefill_gen):
    """BASELINE configs[2] geometry: a 512-token chunk at the end of a 4096-token prompt (Llama-3-8B heads, bf16).  The last
    row of the chunk equals decode attention over the same 4096 keys (paged decode kernel and fp64 definition)."""
    from swiftllm_b200.worker.kernels.paged_attn import paged_attention
    dtype, nq, nkv, D, bs = torch.bfloat16, 32, 8, 128, 16
    prefix, chunk = [3584], [512]
    g = torch.Generator().manual_seed(5)
    bt, sids, nblk = _layout(g, prefix, chunk, bs, extra_seqs=0, extra_blocks=0)
    q = torch.randn(512, nq, D, generator=g).to(dtype)
    kc = torch.randn(nblk, 1, nkv, bs, D, generator=g).to(dtype); vc = torch.randn(nblk, 1, nkv, bs, D, generator=g).to(dtype)
    o = _paged_prefill_run(q, kc, vc, bt, sids, [0], chunk, prefix, D ** -0.5, 0)
    for r in (0, 1, 255, 256, 511):
        ref = K.paged_attention_exact(q[r:r + 1], kc, vc, bt.numpy(), sids, [3584 + r + 1], D ** -0.5, bs, 0)
        check_attention(o[r], ref[0], nq, [3584 + r + 1], what="paged_prefill")
    st = NS(num_decoding_seqs=1, num_prefill_seqs=0, seq_ids=i32(sids), decoding_seq_lens=i32([4096]), softmax_scale=D ** -0.5,
            max_decoding_len=4096, paged_attn_seq_block_size=0)
    od = torch.zeros(1, nq * D, dtype=dtype, device=DEV)
    paged_attention(q[-1:].to(DEV), kc.to(DEV), vc.to(DEV), bt.to(DEV), None, NS(block_size=bs), st, 0, od)
    assert (od.cpu().float() - o[-1].reshape(1, -1).float()).abs().max() <= 2 ** -5 * float(o[-1].float().abs().max())   # two bf16 kernels, each within 8e-3 of fp64


# ----------------------------------------------------------------------------- model level
CFG = dict(model_type="llama", num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, hidden_size=512,
           vocab_size=320, max_position_embeddings=1024, intermediate_size=768, rope_theta=10000.0, rms_norm_eps=1e-5,
           hidden_act="silu")          # head_dim 128: the wgmma kernels serve it
ENG = dict(block_size=16, num_blocks=96, num_cpu_blocks=2, max_seqs_in_block_table=8, max_blocks_per_seq=48)


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_model_chunked_prefill_matches_whole_prompt_and_oracle(dtype, prefill_gen):
    """A SARATHI-style schedule (chunks of two prompts + a piggybacked decode) through LlamaModel.forward on the GPU:
    logits vs the CPU oracle fed the same calls; final tokens equal the whole-prompt prefill's; block tables identical."""
    from test_model_gpu import _make_model
    tdt = torch.float16 if dtype == "float16" else torch.bfloat16
    w = OracleWeights.random(CFG, dtype=tdt, seed=8, std=0.06)
    rng = np.random.default_rng(2)
    pa, pb, pc = (rng.integers(0, 320, size=n).tolist() for n in (600, 130, 9))
    m = _make_model(CFG, ENG, w, dtype=dtype)
    o = OracleLlama(CFG, w, block_size=16, num_blocks=96, num_cpu_blocks=2, max_seqs_in_block_table=8, max_blocks_per_seq=48,
                    attn="exact", dtype=tdt)
    tol = 2e-2 if dtype == "float16" else 2 ** -4          # of max|logit|: 2 layers of fp16 / bf16 rounding (cf. test_model_gpu.py)

    def step(ids, sids, dlens, prefix):
        tm = m.forward(ids, sids, dlens, prefill_prefix_lens_list=prefix)
        to = o.forward(ids, sids, dlens, prefill_prefix_lens_list=prefix)
        got, ref = m.post_layer.last_logits.float().cpu(), o.last_logits.float()
        assert float((got - ref).abs().max()) <= tol * float(ref.abs().max())
        n = o.gpu_block_manager.num_seq_allocated_blocks
        bt = m.gpu_block_manager.block_table.cpu().numpy()
        assert np.array_equal(m.gpu_block_manager.num_seq_allocated_blocks.cpu().numpy(), n)
        for s in range(len(n)):
            assert np.array_equal(bt[s, : n[s]], o.gpu_block_manager.block_table[s, : n[s]])
        return tm, to

    (tm, to) = step([pc], [4], [], None)
    lc = len(pc)
    lc += 1; tm, to = step([pa[:256], pb[:100], [to[0]]], [1, 6, 4], [lc], [0, 0])
    lc += 1; tm, to = step([pa[256:519], pb[100:], [to[2]]], [1, 6, 4], [lc], [256, 100])
    tb = to[1]
    lc += 1; tm, to = step([pa[519:], [tb], [to[2]]], [1, 6, 4], [len(pb) + 1, lc], [519])
    whole = OracleLlama(CFG, w, block_size=16, num_blocks=96, num_cpu_blocks=2, max_seqs_in_block_table=8, max_blocks_per_seq=48,
                        attn="exact", dtype=tdt)
    assert whole.forward([pa, pb], [1, 6], []) == [to[0], tb]


def test_model_chunked_replay_of_the_reference_golden_trace(golden):
    """The recorded trace of the UNMODIFIED reference (tests/golden/model_tiny.npz, fp16, head_dim 64 -> the mma.sync paged
    prefill kernel) replayed with every prefill issued in 7-token chunks: greedy tokens equal the reference's wherever its top-1
    margin is clear, logits within the tolerance of the whole-prompt GPU test (tests/test_model_gpu.py)."""
    import json
    from test_model_gpu import _make_model
    z = golden("model_tiny")
    cfg = json.loads(str(z["config"])); eng = json.loads(str(z["engine"]))
    w = OracleWeights.from_golden(z, cfg["num_hidden_layers"])
    m = _make_model(cfg, eng, w)
    calls = json.loads(str(z["calls"]))
    for i, c in enumerate(calls):
        if c["op"] == "forward":
            nd = len(c["dec_lens"])
            prompts = c["input_ids"][: len(c["input_ids"]) - nd]
            psids = c["seq_ids"][: len(prompts)]
            for p, s in zip(prompts, psids):
                for pos in range(0, max(len(p) - 7, 0), 7):
                    if pos + 7 < len(p):
                        m.forward([p[pos:pos + 7]], [s], [], prefill_prefix_lens_list=[pos])
            last_start = [((len(p) - 1) // 7) * 7 if len(p) > 7 else 0 for p in prompts]
            ids = [p[a:] for p, a in zip(prompts, last_start)] + c["input_ids"][len(prompts):]
            toks = m.forward(ids, c["seq_ids"], c["dec_lens"], prefill_prefix_lens_list=last_start if prompts else None)
            ref = torch.from_numpy(z[f"t{i}_logits"]).float()
            got = m.post_layer.last_logits.float().cpu()
            assert float((got - ref).abs().max()) <= 4e-3 * float(ref.abs().max())
            top2 = ref.topk(2, dim=1).values
            clear = ((top2[:, 0] - top2[:, 1]) > 8e-3 * ref.abs().max()).tolist()
            for a, b, ok in zip(toks, z[f"t{i}_tokens"].tolist(), clear):
                assert (not ok) or a == b
        elif c["op"] == "swap_out":
            m.swap_out_seqs(c["seq_ids"])
        elif c["op"] == "swap_in":
            m.swap_in_seqs(c["seq_ids"])
        else:
            m.free_seqs_resources(c["seq_ids"])
