"""GPU: decode-step fusion - rotary embedding + KV store of the new rows in one launch (sllm_rotary_store_kvcache_decode,
csrc/rotary_store.cu; EngineConfig.fuse_rotary_store) against the two separate kernels (bit for bit) and the oracle.

Part of the default `-m gpu` suite."""
import numpy as np
import pytest
import torch

from oracle import kernels as K
from oracle.model import OracleWeights
from test_chunked_prefill_gpu import CFG, DEV, DTYPES, NS, _layout, i32

pytestmark = pytest.mark.gpu


# ----------------------------------------------------------------------------- fused rotary + KV store (decode rows)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("geom", [dict(nq=4, nkv=2, D=64, bs=16), dict(nq=32, nkv=8, D=128, bs=16), dict(nq=8, nkv=1, D=128, bs=32)])
def test_rotary_store_decode_equals_separate_kernels_and_oracle(dtype, geom):
    """sllm_rotary_store_kvcache_decode == rotary_embedding_inplace followed by store_kvcache, bit for bit (q, k, both caches), on
    row-strided q/k/v slices of one fused-QKV buffer; and both equal the oracle."""
    from swiftllm_b200.worker.kernels.kvcache_mgmt import rotary_store_kvcache_decode, store_kvcache
    from swiftllm_b200.worker.kernels.rotary_emb import rotary_embedding_inplace
    nq, nkv, D, bs = geom["nq"], geom["nkv"], geom["D"], geom["bs"]
    L, layer = 3, 2
    lens = [1, 16, 17, 33, 100, 250, 64]
    Bd = len(lens)
    g = torch.Generator().manual_seed(nq + D)
    bt, sids, nblk = _layout(g, [0] * Bd, lens, bs)
    qkv = torch.randn(Bd, (nq + 2 * nkv) * D, generator=g).to(dtype)
    cos = torch.randn(Bd, D // 2, generator=g).to(dtype); sin = torch.randn(Bd, D // 2, generator=g).to(dtype)
    kc = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype); vc = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype)

    def views(buf):
        return (buf[:, : nq * D].unflatten(1, (nq, D)), buf[:, nq * D:(nq + nkv) * D].unflatten(1, (nkv, D)),
                buf[:, (nq + nkv) * D:].unflatten(1, (nkv, D)))
    st = NS(seq_ids=i32(sids), prefill_seq_start_locs=i32([]), prefill_seq_lens=i32([]), decoding_seq_lens=i32(lens),
            num_prefill_seqs=0, num_decoding_seqs=Bd, num_prefill_tokens=0, max_prefill_len=0,
            position_cos=cos.to(DEV), position_sin=sin.to(DEV), prefill_prefix_lens=None)
    a_buf, b_buf = qkv.to(DEV), qkv.to(DEV)
    ka, va, kb, vb = kc.to(DEV), vc.to(DEV), kc.to(DEV), vc.to(DEV)
    q, k, v = views(a_buf)
    rotary_store_kvcache_decode(q, k, v, ka, va, bt.to(DEV), st, layer)
    q2, k2, v2 = views(b_buf)
    rotary_embedding_inplace(q2, k2, st)
    store_kvcache(k2, v2, kb, vb, bt.to(DEV), None, None, st, layer)
    torch.cuda.synchronize()
    for x, y in ((a_buf, b_buf), (ka, kb), (va, vb)):
        assert torch.equal(x.view(torch.int16), y.view(torch.int16))
    qo, ko = K.rotary_embedding(*views(qkv)[:2], cos, sin)
    kc_o, vc_o = kc.clone(), vc.clone()
    K.store_kvcache_inplace(ko, views(qkv)[2], kc_o, vc_o, bt.numpy(), sids, [], [], lens, 0, 0, bs, layer)
    assert torch.equal(ka.cpu().view(torch.int16), kc_o.view(torch.int16)) and torch.equal(va.cpu().view(torch.int16), vc_o.view(torch.int16))
    assert torch.equal(views(a_buf.cpu())[0].contiguous().view(torch.int16), qo.contiguous().view(torch.int16))


def test_model_decode_with_fused_rotary_store_equals_unfused():
    """LlamaModel with fuse_rotary_store=True (eager and CUDA-graph decode) produces the tokens, logits and KV cache of the
    unfused model exactly."""
    import swiftllm_b200
    from swiftllm_b200.worker.weight import dict_getter
    from test_model_gpu import _hf_tensors
    w = OracleWeights.random(CFG, dtype=torch.bfloat16, seed=8, std=0.06)

    def make(**kw):
        ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=2,
                                        max_seqs_in_block_table=8, max_blocks_per_seq=48, max_batch_size=4, max_tokens_in_batch=256,
                                        dtype="bfloat16", **kw)
        m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(CFG))
        m.load_weights(dict_getter(_hf_tensors(w, CFG["intermediate_size"])))
        m.init_kvcache_and_swap(96)
        m.post_layer.keep_logits = True
        return m
    ref, fused, fused_g = make(), make(fuse_rotary_store=True), make(fuse_rotary_store=True, use_cuda_graph=True)
    rng = np.random.default_rng(4)
    prompts = [rng.integers(0, 320, size=n).tolist() for n in (33, 5, 130)]
    sids = [2, 0, 5]
    t = [m.forward(prompts, sids, []) for m in (ref, fused, fused_g)]
    assert t[0] == t[1] == t[2]
    lens = [len(p) for p in prompts]
    for _ in range(5):
        lens = [l + 1 for l in lens]
        ids = [[x] for x in t[0]]
        t = [m.forward(ids, sids, lens) for m in (ref, fused, fused_g)]
        assert t[0] == t[1] == t[2]
        assert torch.equal(ref.post_layer.last_logits, fused.post_layer.last_logits)
        assert torch.equal(ref.post_layer.last_logits, fused_g.post_layer.last_logits)
    assert torch.equal(ref.k_cache, fused.k_cache) and torch.equal(ref.v_cache, fused.v_cache)
    assert torch.equal(ref.k_cache, fused_g.k_cache) and torch.equal(ref.v_cache, fused_g.v_cache)
