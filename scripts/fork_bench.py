#!/usr/bin/env python
"""Cost of shared KV blocks (LlamaModel.fork_seqs; csrc/kvcache.cu fork_blocks_kernel, copy_block_tails_kernel,
release_blocks_kernel) on one GPU, Llama-3-8B geometry (32 layers, 8 kv heads, head_dim 128, block_size 16, bf16: 1 MiB of K and
1 MiB of V per block).

1. Fork of a 4096-token parent into 1 / 8 / 64 children, P = 4096 (aligned: no tail) and P = 4095 (one tail block per child):
   the whole fork_seqs call (host + fork kernel + allocator + tail copy, then a release of the children; CUDA events over --iters
   repetitions, after one warm-up), against prefilling the same prompts (4 prompts of 4096 tokens per call); and the tail-copy
   kernel alone for 1 / 8 / 64 tails from distinct source blocks (repeated on the same state) with its achieved bytes/s over the
   roofline 4 * block_bytes per tail (read + write of K and V), as a fraction of the H100 SXM data-sheet 3.35 TB/s.
2. KV blocks held by 8 samples of a 4096-token prompt after 256 graph-replayed decode steps: forked (one prefill, 7 forks at
   P = 4096) against unshared (8 prefills).
3. Graph-replayed decode step of a forked batch (64 forks of one 4095-token sequence) against an unshared batch of the same
   lengths, alternating the arms in blocks of --steps steps.  Pages are still read per sequence, so they should be equal.

    python scripts/fork_bench.py [--iters 20] [--steps 20]

Prints one JSON line per measurement, with the GPU name and power limit."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from sampling_bench import gpu_info, time_ms  # noqa: E402

HBM = 3.35e12
BS, CTX = 16, 4096


def _i32(x):
    return torch.tensor(list(x), dtype=torch.int32, device="cuda")


def _model(num_blocks, max_seqs, mbps):
    import swiftllm_b200
    from bench import model_dict
    from swiftllm_b200.worker.weight import synthetic_getter
    mc = swiftllm_b200.LlamaModelConfig(model_dict("llama3-8b"))
    ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=BS, gpu_mem_utilization=0.97, num_cpu_blocks=0,
                                    max_seqs_in_block_table=max_seqs, max_blocks_per_seq=mbps, max_batch_size=64,
                                    max_tokens_in_batch=16384, dtype="bfloat16", use_cuda_graph=True)
    m = swiftllm_b200.LlamaModel(ec, mc)
    m.load_weights(synthetic_getter(seed=0, std=0.02, device="cuda"))
    m.init_kvcache_and_swap(num_blocks)
    return m


def _events(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def fork_cost(m, iters, info):
    from swiftllm_b200.worker.kernels.block_mgmt import copy_block_tails
    bm = m.gpu_block_manager
    block_bytes = m.k_cache[0].numel() * m.k_cache.element_size()
    prompt = [(7 * i) % 128000 for i in range(CTX)]
    m.forward([prompt], [0], [])
    for n in (1, 8, 64):
        kids = list(range(1, n + 1))
        for P in (CTX, CTX - 1):
            def fork_and_free():
                m.fork_seqs([0] * n, kids, [P] * n)
                m.free_seqs_resources(kids)
            fork_and_free()             # warm-up
            ms_fork = _events(fork_and_free, iters)
            row = {"what": "fork", "children": n, "P": P, "gpu": info, "fork_and_release_ms": ms_fork}
            print(json.dumps(row), flush=True)
        # prefilling the same prompts instead, 4 per call
        def prefill_all():
            for c in range(0, n, 4):
                sids = kids[c:c + 4]
                m.forward([prompt] * len(sids), sids, [])
            m.free_seqs_resources(kids)
        if n == 1:
            prefill_all()               # warm-up
        ms = _events(prefill_all, 1)
        print(json.dumps({"what": "prefill_instead", "children": n, "gpu": info, "prefill_ms": ms}), flush=True)
    m.free_seqs_resources([0])
    # the tail copy alone, every tail from a DIFFERENT source block (one source read by all children would be served by L2):
    # n one-block parents forked at P = bs - 1, the copy repeated on the same state
    for n in (1, 8, 64):
        parents, kids = list(range(1, n + 1)), list(range(65, 65 + n))
        bm.allocate_blocks_for_seqs(_i32(parents), _i32([BS - 1] * n), seq_ids_list=parents, target_lens_list=[BS - 1] * n,
                                    want_new_blocks=False)
        m.fork_seqs(parents, kids, [BS - 1] * n)
        s, d, lens = _i32(parents), _i32(kids), _i32([BS - 1] * n)
        ms = time_ms(lambda: copy_block_tails(m.k_cache, m.v_cache, m.token_cache, bm.block_table, s, d, lens, BS), iters)
        moved = 4 * block_bytes * n
        print(json.dumps({"what": "tail_copy_kernel", "tails": n, "block_bytes": block_bytes, "gpu": info, "ms": ms,
                          "roofline_bytes": moved, "tb_per_s": moved / ms / 1e9, "of_hbm_peak": moved / ms / 1e9 / (HBM / 1e12)}),
                         flush=True)
        m.free_seqs_resources(parents + kids)


def blocks_held(m, info):
    from swiftllm_b200 import SamplingParams
    bm = m.gpu_block_manager
    prompt = [(11 * i) % 128000 for i in range(CTX)]
    out = {}
    for shared in (True, False):
        free0 = bm.num_free_blocks
        t = m.forward([prompt], [0], [])[0]
        if shared:
            m.fork_seqs([0] * 7, list(range(1, 8)), [CTX] * 7)
        else:
            for s in range(1, 8):
                m.forward([prompt], [s], [])
        last, L = [t] * 8, CTX
        for _ in range(256):
            L += 1
            last = m.forward([[x] for x in last], list(range(8)), [L] * 8,
                             sampling_params_list=[SamplingParams(0.8, seed=i) for i in range(8)])
        out["forked" if shared else "unshared"] = free0 - bm.num_free_blocks
        m.free_seqs_resources(list(range(8)))
    print(json.dumps({"what": "blocks_held", "samples": 8, "prompt": CTX, "decode_steps": 256, "gpu": info, **out}), flush=True)


def step_time(m, steps, info):
    B, S = 64, CTX
    unshared, forked = list(range(B)), list(range(B, 2 * B))
    bm = m.gpu_block_manager
    bm.allocate_blocks_for_seqs(_i32(unshared), _i32([S - 1] * B), seq_ids_list=unshared, target_lens_list=[S - 1] * B,
                                want_new_blocks=False)
    bm.allocate_blocks_for_seqs(_i32([forked[0]]), _i32([S - 1]), seq_ids_list=forked[:1], target_lens_list=[S - 1],
                                want_new_blocks=False)
    g = torch.Generator(device="cuda").manual_seed(1234)
    with torch.inference_mode():
        nb = m.k_cache.shape[0]
        for s in range(0, nb, 64):
            m.k_cache[s:s + 64].normal_(generator=g)
            m.v_cache[s:s + 64].normal_(generator=g)
    m.fork_seqs([forked[0]] * (B - 1), forked[1:], [S - 1] * (B - 1))
    ids = [[1000 + i] for i in range(B)]
    arms = {"unshared": lambda n: [m.forward(ids, unshared, [S] * B) for _ in range(n)],
            "forked": lambda n: [m.forward(ids, forked, [S] * B) for _ in range(n)]}
    res = {k: [] for k in arms}
    for fn in arms.values():
        fn(3)
    for _ in range(5):
        for k, fn in arms.items():
            res[k].append(_events(lambda: fn(steps), 1) / steps)
    print(json.dumps({"what": "decode_step", "B": B, "seqlen": S, "gpu": info, "ms": res, "best_ms": {k: min(v) for k, v in res.items()},
                      "spread_ms": {k: max(v) - min(v) for k, v in res.items()}}), flush=True)
    m.free_seqs_resources(unshared + forked)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "fork_bench.py measures on a GPU"
    info = gpu_info()
    # 64 unshared sequences of 4096 tokens, plus one 4096-token parent and 64 tails (34 GiB of KV cache)
    m = _model(num_blocks=65 * (CTX // BS) + 512, max_seqs=2 * 64 + 1, mbps=CTX // BS + 32)
    fork_cost(m, args.iters, info)
    blocks_held(m, info)
    step_time(m, args.steps, info)


if __name__ == "__main__":
    main()
