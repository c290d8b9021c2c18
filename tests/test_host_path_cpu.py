"""CPU: the product's host path (swiftllm_b200.LlamaModel and everything under it except the CUDA kernels) against
oracle.model.OracleLlama.  Kernel wrappers are replaced by the oracle's restatements (tests/cpu_shim.py), so any difference
comes from the host code: metadata staging, positions, block allocation + host mirror, layer sequencing with the fused QKV
GEMM, last-token gather, swap and free.  The GPU parity of the kernels themselves is tests/test_kernels_gpu.py."""
import numpy as np
import torch

from oracle.model import OracleLlama, OracleWeights
from cpu_shim import product_on_cpu            # tests/ is on sys.path (rootdir conftest, no package)

CFG = dict(model_type="llama", num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, hidden_size=128,
           vocab_size=300, max_position_embeddings=256, intermediate_size=192, rope_theta=10000.0, rms_norm_eps=1e-5,
           hidden_act="silu")
ENG = dict(block_size=16, num_blocks=24, num_cpu_blocks=6, max_seqs_in_block_table=8, max_blocks_per_seq=8)


def _hf_tensors(w: OracleWeights, F: int):
    d = {"model.embed_tokens.weight": w.wte, "lm_head.weight": w.lm_head, "model.norm.weight": w.final_norm}
    for i, lw in enumerate(w.layers):
        p = f"model.layers.{i}."
        d[p + "input_layernorm.weight"] = lw.attn_norm; d[p + "post_attention_layernorm.weight"] = lw.ffn_norm
        d[p + "self_attn.q_proj.weight"] = lw.q_proj; d[p + "self_attn.k_proj.weight"] = lw.k_proj
        d[p + "self_attn.v_proj.weight"] = lw.v_proj; d[p + "self_attn.o_proj.weight"] = lw.o_proj
        d[p + "mlp.up_proj.weight"] = lw.up_gate_proj[:F]; d[p + "mlp.gate_proj.weight"] = lw.up_gate_proj[F:]
        d[p + "mlp.down_proj.weight"] = lw.down_proj
    return d


def _product(w, **ec_kw):
    import swiftllm_b200
    from swiftllm_b200.worker.weight import dict_getter
    ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=ENG["block_size"], gpu_mem_utilization=0.9,
                                    num_cpu_blocks=ENG["num_cpu_blocks"], max_seqs_in_block_table=ENG["max_seqs_in_block_table"],
                                    max_blocks_per_seq=ENG["max_blocks_per_seq"], max_batch_size=8, max_tokens_in_batch=256,
                                    dtype="float16", **ec_kw)
    m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(CFG))
    m.load_weights(dict_getter(_hf_tensors(w, CFG["intermediate_size"])))
    m.init_kvcache_and_swap(ENG["num_blocks"])
    m.post_layer.keep_logits = True
    return m


def _oracle(w):
    return OracleLlama(CFG, w, block_size=ENG["block_size"], num_blocks=ENG["num_blocks"], num_cpu_blocks=ENG["num_cpu_blocks"],
                       max_seqs_in_block_table=ENG["max_seqs_in_block_table"], max_blocks_per_seq=ENG["max_blocks_per_seq"],
                       attn="exact", dtype=torch.float16)


def _same_state(m, o):
    for name in ("gpu_block_manager", "cpu_block_manager"):
        bm, ob = getattr(m, name), getattr(o, name)
        n = ob.num_seq_allocated_blocks
        assert np.array_equal(bm.num_seq_allocated_blocks.numpy(), n)
        assert np.array_equal(bm._host_nsab, n)                                   # host mirror
        assert np.array_equal(bm.is_block_free.numpy(), ob.is_block_free)
        assert bm.num_free_blocks == int(ob.is_block_free.sum())
        bt = bm.block_table.numpy()
        for s in range(len(n)):
            assert np.array_equal(bt[s, : n[s]], ob.block_table[s, : n[s]])


import pytest


@pytest.mark.parametrize("fuse_rotary_store,device_swap", [(False, False), (True, True)], ids=["reference-shaped", "fused-rotary-store+device-swap"])
def test_product_host_path_matches_oracle_on_cpu(fuse_rotary_store, device_swap):
    """Prefill, decode, a mixed batch, swap out / in, free.  Same oracle kernels on both sides, so the only arithmetic difference
    is the fused QKV GEMM: logits within 1e-5 of max|logit|, greedy tokens, every block id, free map and host mirror identical.
    fuse_rotary_store: pure-decode steps take the one-launch rotary + KV-store path, mixed / prefill steps the separate calls;
    device_swap: swap_out / swap_in hand device-resident id tensors to the gather/scatter swap entry (no .tolist())."""
    torch.manual_seed(0)
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=2, std=0.08)
    rng = np.random.default_rng(5)
    with product_on_cpu():
        m, o = _product(w, fuse_rotary_store=fuse_rotary_store, device_swap=device_swap), _oracle(w)

        def step(*a):
            tm, to = m.forward(*a), o.forward(*a)
            assert tm == to
            ref = o.last_logits
            assert float((m.post_layer.last_logits - ref).abs().max()) <= 1e-5 * float(ref.abs().max())
            _same_state(m, o)
            return to

        prompts = [rng.integers(0, 300, size=n).tolist() for n in (37, 5, 16)]
        sids = [5, 0, 3]
        t = step(prompts, sids, [])
        lens = [len(p) for p in prompts]
        for _ in range(3):
            lens = [l + 1 for l in lens]
            t = step([[x] for x in t], sids, lens)
        # mixed batch: two new prompts + the three decoding sequences
        newp = [rng.integers(0, 300, size=n).tolist() for n in (20, 1)]
        lens = [l + 1 for l in lens]
        t = step(newp + [[x] for x in t[:3]], [7, 2] + sids, lens)
        # preempt sequence 5 (swap out), keep decoding the others, bring it back
        m.swap_out_seqs([5]); o.swap_out_seqs([5]); _same_state(m, o)
        lens_b = [lens[1] + 1, lens[2] + 1]
        t2 = step([[t[3]], [t[4]]], [0, 3], lens_b)
        m.swap_in_seqs([5]); o.swap_in_seqs([5]); _same_state(m, o)
        step([[t[2]], [t2[0]], [t2[1]]], [5, 0, 3], [lens[0] + 1, lens_b[0] + 1, lens_b[1] + 1])
        m.free_seqs_resources([0, 7]); o.free_seqs_resources([0, 7]); _same_state(m, o)
        assert float((m.k_cache - o.k_cache).abs().max()) <= 1e-5 and float((m.v_cache - o.v_cache).abs().max()) <= 1e-5


def test_product_block_exhaustion_raises_like_the_reference():
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=3, std=0.08)
    with product_on_cpu():
        m = _product(w)
        import pytest
        with pytest.raises(RuntimeError, match="No enough free blocks"):
            m.forward([[1] * 120, [2] * 120, [3] * 120, [4] * 120], [0, 1, 2, 3], [])      # 4 x 8 blocks > 24
        assert m.gpu_block_manager.num_free_blocks == ENG["num_blocks"]                     # nothing was taken


def test_block_manager_random_operation_sequences_match_the_oracle():
    """Seeded random walks over the product BlockManager's API (allocate to a larger target - as decode and chunked prefill do -,
    free, gather-and-free, exhaustion) against the numpy restatement of the reference's BlockManager (block_manager.py:5-103):
    block ids handed out, tables, free map, free count and the host mirror must agree after every operation, and a failed
    allocation must change nothing."""
    from swiftllm_b200.worker.block_manager import BlockManager
    from oracle.kernels import BlockManagerOracle
    import pytest
    with product_on_cpu():
        for seed in range(6):
            rng = np.random.default_rng(seed)
            nblk, nseq, mbps, bs = int(rng.integers(8, 40)), 10, 12, 16
            bm = BlockManager("GPU", nblk, nseq, mbps, bs, device="cpu")
            ob = BlockManagerOracle(nblk, nseq, mbps, bs)
            lens = np.zeros(nseq, dtype=np.int64)
            for _ in range(120):
                op = rng.choice(["alloc", "alloc", "alloc", "free", "gather"])
                k = int(rng.integers(1, 5))
                sids = rng.choice(nseq, size=k, replace=False).tolist()
                t_s = torch.tensor(sids, dtype=torch.int32)
                if op == "alloc":
                    grow = rng.integers(0, 40, size=k)
                    target = np.minimum(lens[sids] + grow, mbps * bs).tolist()
                    t_l = torch.tensor(target, dtype=torch.int32)
                    need = int(sum((t + bs - 1) // bs for t in target) - ob.num_seq_allocated_blocks[sids].sum())
                    if need > ob.num_free_blocks:
                        free_before = bm.is_block_free.clone()
                        with pytest.raises(RuntimeError, match="No enough free blocks"):
                            bm.allocate_blocks_for_seqs(t_s, t_l, seq_ids_list=sids, target_lens_list=target)
                        with pytest.raises(RuntimeError):
                            ob.allocate_blocks_for_seqs(sids, target)
                        assert torch.equal(bm.is_block_free, free_before)
                    else:
                        new = bm.allocate_blocks_for_seqs(t_s, t_l, seq_ids_list=sids, target_lens_list=target)
                        ref = ob.allocate_blocks_for_seqs(sids, target)
                        assert new.tolist() == ref.tolist()
                        lens[sids] = target
                elif op == "free":
                    bm.free_blocks_for_seqs(t_s, seq_ids_list=sids); ob.free_blocks_for_seqs(sids); lens[sids] = 0
                else:
                    got = bm.gather_allocated_blocks_and_free(t_s, seq_ids_list=sids)
                    assert got.tolist() == ob.gather_allocated_blocks_and_free(sids).tolist()
                    lens[sids] = 0
                n = ob.num_seq_allocated_blocks
                assert np.array_equal(bm.num_seq_allocated_blocks.numpy(), n) and np.array_equal(bm._host_nsab, n)
                assert np.array_equal(bm.is_block_free.numpy(), ob.is_block_free) and bm.num_free_blocks == ob.num_free_blocks
                for s in range(nseq):
                    assert np.array_equal(bm.block_table.numpy()[s, : n[s]], ob.block_table[s, : n[s]])


def test_block_reservation_refuses_without_changing_anything():
    """BlockManager.reserve_blocks_for_seqs, the host half with which every step path (eager, CUDA graph, speculative) counts its
    blocks: it counts only the new blocks into the mirror and the free count, touches no device table, and a sequence past
    max_blocks_per_seq or more new blocks than are free raises RuntimeError and changes nothing."""
    from swiftllm_b200.worker.block_manager import BlockManager
    import pytest
    bm = BlockManager("GPU", 6, 4, 3, 16, device="cpu")
    assert bm.reserve_blocks_for_seqs([0, 1], [40, 1]) == 4
    assert bm._host_nsab.tolist() == [3, 1, 0, 0] and bm.num_free_blocks == 2
    assert bm.reserve_blocks_for_seqs([0, 1], [48, 16]) == 0                   # already held
    assert bm.reserve_blocks_for_seqs([], []) == 0
    before = bm._host_nsab.copy()
    with pytest.raises(RuntimeError, match=r"^sequence needs 4 blocks > max_blocks_per_seq=3$"):
        bm.reserve_blocks_for_seqs([2, 0], [16, 49])
    with pytest.raises(RuntimeError, match=r"^No enough free blocks available on GPU \(6 in total, 2 free, 4 requested\)$"):
        bm.reserve_blocks_for_seqs([2, 3], [16, 48])
    assert np.array_equal(bm._host_nsab, before) and bm.num_free_blocks == 2
    assert not bm.num_seq_allocated_blocks.any() and bool(bm.is_block_free.all())
