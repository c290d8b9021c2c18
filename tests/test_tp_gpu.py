"""GPU (needs >= 2 devices; skipped otherwise): tensor-parallel LlamaModel (heads / FFN columns sharded, one NCCL
all-reduce after o_proj and down_proj) against the TP=1 model on the same synthetic weights: identical KV-block
indices, greedy tokens equal where the top-1 margin is clear, logits within bf16 tolerance."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

CFG = dict(model_type="llama", num_hidden_layers=3, num_attention_heads=8, num_key_value_heads=4, hidden_size=1024,
           vocab_size=1000, max_position_embeddings=512, intermediate_size=1536, rope_theta=500000.0, rms_norm_eps=1e-5,
           hidden_act="silu")


# 8 kv heads (head_dim stays 128): shards down to 1 kv head / 2 q heads per rank at world 8
CFG8 = dict(CFG, hidden_size=2048, num_attention_heads=16, num_key_value_heads=8)

# (name, fused_allreduce, shard_lm_head, fuse_rotary_store): every exchange / sharding variant of the TP data plane
MODES = [("nccl", False, False, False),
         ("fused-one-shot", True, False, False),
         ("fused-two-shot", "two_shot", False, False),
         ("fused-two-shot-nvls", "two_shot_nvls", False, False),
         ("fused-ll", "ll", False, False),
         ("fused-ll-nvls", "ll_nvls", False, False),
         ("nccl+sharded-lm-head+rotary-store", False, True, True),
         ("two-shot+sharded-lm-head+rotary-store", "two_shot", True, True),
         ("ll-nvls+sharded-lm-head+rotary-store", "ll_nvls", True, True),
         ("nvls+sharded-lm-head+rotary-store", "two_shot_nvls", True, True),      # the library default at TP 8
         ("default", None, None, True)]                                              # whatever the library picks for this TP degree


def _run(rank, world, port, q, mode_names):
    """One process per GPU; ALL requested modes run in this one process group (one NCCL init per world size instead of one
    per mode: multi-GPU box time is charged per GPU)."""
    import numpy as np
    import torch.distributed as dist
    import swiftllm_b200
    from swiftllm_b200.worker.weight import synthetic_getter
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    cfg = CFG8 if world > 4 else CFG

    def make(tp, r, graph=False, fused=False, shard=False, frs=False):
        ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=2,
                                        max_seqs_in_block_table=8, max_blocks_per_seq=16, max_batch_size=4, max_tokens_in_batch=256,
                                        dtype="bfloat16", tp_size=tp, tp_rank=r, use_cuda_graph=graph, fused_allreduce=fused,
                                        shard_lm_head=shard, fuse_rotary_store=frs)
        m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(cfg))
        m.load_weights(synthetic_getter(seed=11, std=0.05, device=f"cuda:{rank}"))
        m.init_kvcache_and_swap(40)
        m.post_layer.keep_logits = True
        return m

    results = {}
    import sys
    import time
    for name, fused, shard, frs in [m for m in MODES if m[0] in mode_names]:
        t_mode = time.perf_counter()
        if rank == 0:
            print(f"[tp parity world {world}] mode `{name}` ...", file=sys.stderr, flush=True)
        tp = make(world, rank, fused=fused, shard=shard, frs=frs)
        tpg = make(world, rank, graph=True, fused=fused, shard=shard, frs=frs)
        ref = make(1, 0) if rank == 0 else None
        rng = np.random.default_rng(3)
        prompts = [rng.integers(0, 1000, size=n).tolist() for n in (40, 7, 129)]
        sids = [5, 0, 2]
        worst = 0.0
        toks = tp.forward(prompts, sids, []); tg = tpg.forward(prompts, sids, [])
        assert toks == tg, name
        lens = [len(p) for p in prompts]
        rt = ref.forward(prompts, sids, []) if ref else None
        for step in range(6):
            if ref:
                a, b = tp.post_layer.last_logits.float(), ref.post_layer.last_logits.float()
                rel = float((a - b).abs().max() / b.abs().max()); worst = max(worst, rel)
                top2 = b.topk(2, dim=1).values
                clear = ((top2[:, 0] - top2[:, 1]) > 2 * 2 ** -5 * b.abs().max()).tolist()
                assert rel <= 2 ** -5, (name, rel)
                for x, y, c in zip(toks, rt, clear):
                    if c:
                        assert x == y, name
                n = ref.gpu_block_manager.num_seq_allocated_blocks
                assert torch.equal(tp.gpu_block_manager.num_seq_allocated_blocks, n), name
                for s in sids:
                    k = int(n[s])
                    assert torch.equal(tp.gpu_block_manager.block_table[s, :k], ref.gpu_block_manager.block_table[s, :k]), name
            # all ranks must feed the same tokens: use rank 0's reference tokens
            feed = [rt if ref else None]
            dist.broadcast_object_list(feed, src=0)
            lens = [l + 1 for l in lens]
            ids = [[t] for t in feed[0]]
            toks = tp.forward(ids, sids, lens); tg = tpg.forward(ids, sids, lens)
            assert toks == tg, name                            # CUDA-graph decode with the exchange inside == eager
            if ref:
                rt = ref.forward(ids, sids, lens)
        results[name] = worst
        if rank == 0:
            ex = "nccl" if tp.comm is None else ("ll" if tp.comm.ll else "two_shot_nvls" if tp.comm.nvls else "two_shot" if tp.comm.two_shot else "one_shot")
            print(f"[tp parity world {world}] mode `{name}` ok: worst logit rel. err. {worst:.4f}, exchange {ex}, "
                  f"lm_head sharded {tp.weight.lm_head_sharded}, {time.perf_counter() - t_mode:.1f} s", file=sys.stderr, flush=True)
        # NCCL kernels captured in live CUDA graphs make later collectives / teardown block: drop the graphs first
        tpg._graphs.clear(); torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
        del tp, tpg, ref
    if rank == 0:
        q.put(results)
    time.sleep(0.5)            # let the parent drain the queue
    os._exit(0)


def _spawn(world, mode_names, port):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_run, args=(r, world, port, q, mode_names)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        results = q.get(timeout=420)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.exitcode is None:
                p.kill()
    for p in procs:
        assert p.exitcode == 0
    return results


@pytest.mark.parametrize("world", [2, 4])
def test_tp_matches_single_gpu(world):
    """NCCL all-reduce + add/norm kernel, the one-shot fused peer-memory exchange, and the library's default configuration for
    this TP degree (exchange, lm_head sharding, fused rotary / store), against TP = 1 (eager and CUDA graph)."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    res = _spawn(world, ["nccl", "fused-one-shot", "default"], 29650 + world)
    print("TP parity (worst logit rel. err. vs TP=1):", world, res)
    assert set(res) == {"nccl", "fused-one-shot", "default"} and max(res.values()) <= 2 ** -5


@pytest.mark.parametrize("world", [2, 4])
def test_tp_two_shot_exchange_and_sharded_lm_head_match_single_gpu(world):
    """fused_allreduce="two_shot" (row owner reduces + adds + normalises, pushes the row to every rank; residual sharded by
    rows) with peer loads / stores and with the NVSwitch doing the reduction and the broadcast (multimem.ld_reduce /
    multimem.st); vocabulary-sharded lm_head (+ fused rotary / KV store) with both exchanges - against TP = 1, eager and inside
    CUDA graphs.  Prompts of 40 / 7 / 129 tokens exercise rows without an owner CTA on some ranks and T not divisible by the
    world size."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    names = ["fused-two-shot", "fused-two-shot-nvls", "nccl+sharded-lm-head+rotary-store", "two-shot+sharded-lm-head+rotary-store"]
    res = _spawn(world, names, 29690 + world)
    print("TP parity (worst logit rel. err. vs TP=1):", world, res)
    assert set(res) == set(names) and max(res.values()) <= 2 ** -5


@pytest.mark.parametrize("world", [2, 4])
def test_tp_ll_push_exchange_matches_single_gpu(world):
    """fused_allreduce="ll" / "ll_nvls": the barrier-free push exchange (csrc/allreduce_ll.cu; data lines carry their epoch tag)
    for decode-sized steps - prompts of 40 + 7 + 129 = 176 rows (not divisible by the world size; some ranks own one row more)
    and 3-row decode steps (fewer rows than ranks at world 4 / 8: ranks that own nothing), eager and in CUDA graphs."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    names = ["fused-ll", "fused-ll-nvls", "ll-nvls+sharded-lm-head+rotary-store"]
    res = _spawn(world, names, 29730 + world)
    print("TP parity (worst logit rel. err. vs TP=1):", world, res)
    assert set(res) == set(names) and max(res.values()) <= 2 ** -5


def test_tp_world8_matches_single_gpu():
    """World 8 (1 kv head / 2 q heads per rank; 3-row decode steps leave five ranks without a row to own): the library default for
    TP 8 (two-shot exchange with in-switch reduction + sharded lm_head + fused rotary / store), the NCCL path and the P2P two-shot
    kernel against TP = 1, in ONE process group.  SLLM_TP8_MODES=<comma list | all> selects others (all eleven modes in one
    process group means 22 tensor-parallel models and ~80 symmetric-memory buffers with multicast bindings)."""
    if torch.cuda.device_count() < 8:
        pytest.skip("needs 8 GPUs")
    want = os.environ.get("SLLM_TP8_MODES", "default,nccl,fused-two-shot")
    names = [m[0] for m in MODES] if want == "all" else [n for n in (m[0] for m in MODES) if n in want.split(",")]
    res = _spawn(8, names, 29760)
    print("TP parity (worst logit rel. err. vs TP=1):", 8, res)
    assert set(res) == set(names) and max(res.values()) <= 2 ** -5
