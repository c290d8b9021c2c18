"""GPU: swap with device-resident id lists (sllm_swap_blocks_gathered, csrc/swap_gather.cu; EngineConfig.device_swap) against the
oracle and the memcpy path (swiftllm_c.swap_blocks): exact bytes, K and V, scattered and consecutive ids, both directions.

Part of the default `-m gpu` suite."""
import numpy as np
import pytest
import torch

from oracle import kernels as K
from oracle.model import OracleWeights

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_swap_blocks_device_ids_exact(dtype):
    from swiftllm_b200 import swiftllm_c
    g = torch.Generator().manual_seed(1)
    shape_g, shape_c = (20, 3, 2, 16, 64), (12, 3, 2, 16, 64)
    kc, vc = torch.randn(shape_g, generator=g).to(dtype), torch.randn(shape_g, generator=g).to(dtype)
    ks, vs = torch.randn(shape_c, generator=g).to(dtype), torch.randn(shape_c, generator=g).to(dtype)
    src, dst = [3, 4, 5, 17, 0, 9], [0, 1, 2, 7, 11, 4]
    kco, vco, kso, vso = kc.clone(), vc.clone(), ks.clone(), vs.clone()
    kcd, vcd = kc.to(DEV), vc.to(DEV)
    ksd, vsd = ks.clone().pin_memory(), vs.clone().pin_memory()
    i64 = lambda x: torch.tensor(x, dtype=torch.int64, device=DEV)
    K.swap_blocks_inplace(src, dst, False, kco, vco, kso, vso)
    swiftllm_c.swap_blocks_device(i64(src), i64(dst), False, kcd, vcd, ksd, vsd); torch.cuda.synchronize()
    assert torch.equal(ksd.view(torch.int16), kso.view(torch.int16)) and torch.equal(vsd.view(torch.int16), vso.view(torch.int16))
    kcd.zero_(); vcd.zero_(); kco.zero_(); vco.zero_()
    K.swap_blocks_inplace(dst, src, True, kco, vco, kso, vso)
    swiftllm_c.swap_blocks_device(i64(dst), i64(src), True, kcd, vcd, ksd, vsd); torch.cuda.synchronize()
    assert torch.equal(kcd.cpu().view(torch.int16), kco.view(torch.int16)) and torch.equal(vcd.cpu().view(torch.int16), vco.view(torch.int16))
    swiftllm_c.swap_blocks_device(i64([]), i64([]), True, kcd, vcd, ksd, vsd)       # empty is a no-op
    with pytest.raises(AssertionError, match="pinned"):
        swiftllm_c.swap_blocks_device(i64(src), i64(dst), False, kcd, vcd, ks.clone(), vs.clone())


@pytest.mark.parametrize("variant", [dict(device_swap=True), dict(swap_on_copy_stream=True),
                                     dict(device_swap=True, swap_on_copy_stream=True)],
                         ids=["device-ids", "copy-stream", "device-ids+copy-stream"])
def test_model_swap_with_device_ids_equals_memcpy_path(variant):
    """Preempt / resume through LlamaModel.swap_out_seqs / swap_in_seqs with device_swap=True (ids stay on the device, one
    gather kernel) and / or swap_on_copy_stream=True (the copy runs on a dedicated stream, the next forward waits for it on the
    device): block tables, free maps, swap space and cache contents equal the memcpy path's; decoding between and after the swaps
    gives the same tokens."""
    from test_chunked_prefill_gpu import CFG
    from test_model_gpu import _hf_tensors
    import swiftllm_b200
    from swiftllm_b200.worker.weight import dict_getter
    w = OracleWeights.random(CFG, dtype=torch.bfloat16, seed=8, std=0.06)

    def make(**kw):
        ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=24,
                                        max_seqs_in_block_table=8, max_blocks_per_seq=48, max_batch_size=4, max_tokens_in_batch=256,
                                        dtype="bfloat16", **kw)
        m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(CFG))
        m.load_weights(dict_getter(_hf_tensors(w, CFG["intermediate_size"])))
        m.init_kvcache_and_swap(96)
        return m
    a, b = make(), make(**variant)
    rng = np.random.default_rng(6)
    prompts = [rng.integers(0, 320, size=n).tolist() for n in (70, 5, 33)]
    sids = [2, 0, 5]
    ta, tb = a.forward(prompts, sids, []), b.forward(prompts, sids, [])
    assert ta == tb
    for m in (a, b):
        m.swap_out_seqs([2, 5])
    torch.cuda.synchronize()
    assert torch.equal(a.k_swap, b.k_swap) and torch.equal(a.v_swap, b.v_swap)
    for name in ("gpu_block_manager", "cpu_block_manager"):
        x, y = getattr(a, name), getattr(b, name)
        assert torch.equal(x.is_block_free, y.is_block_free) and torch.equal(x.num_seq_allocated_blocks, y.num_seq_allocated_blocks)
        assert x.num_free_blocks == y.num_free_blocks
    ta, tb = a.forward([[ta[1]]], [0], [6]), b.forward([[tb[1]]], [0], [6])
    assert ta == tb
    for m in (a, b):
        m.swap_in_seqs([5, 2])
    lens = [71, 7, 34]
    ta2 = a.forward([[1], [2], [3]], sids, lens); tb2 = b.forward([[1], [2], [3]], sids, lens)
    assert ta2 == tb2
    n = a.gpu_block_manager.num_seq_allocated_blocks.tolist()
    for s in sids:
        assert torch.equal(a.gpu_block_manager.block_table[s, : n[s]], b.gpu_block_manager.block_table[s, : n[s]])
    assert torch.equal(a.k_cache, b.k_cache) and torch.equal(a.v_cache, b.v_cache)
