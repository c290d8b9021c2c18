#!/usr/bin/env python
"""Cost of sampling (csrc/sampling.cu) on the GPU.

1. Kernel time (CUDA events, mean over --iters launches) at B in {1, 8, 64, 256}, V = 128256 bf16, for greedy (torch.argmax),
   temperature only, top-k 50, top-p 0.95 (T = 0.8), next to a torch implementation of the top-p filter (sort + softmax +
   cumsum + multinomial).
2. The bench.py decode step (Llama-3-8B shapes, batch 64 x 4096 tokens, CUDA-graph replay): greedy against sampled
   (T = 0.8, top-p 0.95), alternating blocks of --steps steps.

    python scripts/sampling_bench.py [--iters 200] [--steps 30] [--skip-model]

Prints one JSON line per measurement, with the GPU name and power limit."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def time_ms(fn, iters):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def torch_top_p(logits, T, p, gen):
    probs = torch.softmax(logits.float() / T, dim=-1)
    sp, si = probs.sort(dim=-1, descending=True)
    cum = sp.cumsum(dim=-1)
    sp[(cum - sp) > p] = 0
    pick = torch.multinomial(sp, 1, generator=gen)
    return si.gather(1, pick).squeeze(1)


def kernel_bench(iters, info):
    from swiftllm_b200.worker.kernels.sampling import sample_tokens
    V = 128256
    gen = torch.Generator(device="cuda").manual_seed(0)
    for B in (1, 8, 64, 256):
        logits = (torch.randn((B, V), device="cuda", generator=gen) * 3).to(torch.bfloat16)
        z = lambda v, dt: torch.full((B,), v, dtype=dt, device="cuda")
        seed = torch.arange(B, dtype=torch.int64, device="cuda")
        pos = z(4096, torch.int32)
        row = {"what": "sampling_kernel", "B": B, "V": V, "dtype": "bf16", "gpu": info,
               "bytes": B * V * 2, "argmax_us": 1e3 * time_ms(lambda: torch.argmax(logits, dim=1), iters)}
        for name, T, k, p in (("greedy", 0.0, 0, 1.0), ("temperature", 0.8, 0, 1.0), ("top_k50", 0.8, 50, 1.0),
                              ("top_p0.95", 0.8, 0, 0.95), ("top_k50_top_p0.95", 0.8, 50, 0.95)):
            t, kk, pp = z(T, torch.float32), z(k, torch.int32), z(p, torch.float32)
            row[f"{name}_us"] = 1e3 * time_ms(lambda: sample_tokens(logits, t, kk, pp, seed, pos), iters)
        row["torch_top_p0.95_us"] = 1e3 * time_ms(lambda: torch_top_p(logits, 0.8, 0.95, gen), max(10, iters // 10))
        print(json.dumps(row), flush=True)


def model_bench(steps, info):
    import swiftllm_b200
    from bench import model_dict
    from swiftllm_b200.worker.weight import synthetic_getter
    B, S, bs = 64, 4096, 16
    mc = swiftllm_b200.LlamaModelConfig(model_dict("llama3-8b"))
    bps = (S + bs - 1) // bs
    ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=bs, gpu_mem_utilization=0.97, num_cpu_blocks=0,
                                    max_seqs_in_block_table=B, max_blocks_per_seq=bps + 8, max_batch_size=B,
                                    max_tokens_in_batch=16384, dtype="bfloat16", use_cuda_graph=True)
    m = swiftllm_b200.LlamaModel(ec, mc)
    m.load_weights(synthetic_getter(seed=0, std=0.02, device="cuda"))
    nb = B * bps + 64
    m.init_kvcache_and_swap(nb)
    g = torch.Generator(device="cuda").manual_seed(1234)
    with torch.inference_mode():
        for s in range(0, nb, max(1, nb // 64)):
            m.k_cache[s:s + nb // 64].normal_(generator=g)
            m.v_cache[s:s + nb // 64].normal_(generator=g)
    sids = list(range(B))
    lens = [S] * B
    ids = [[i % 1000] for i in range(B)]
    sp = [swiftllm_b200.SamplingParams(0.8, top_p=0.95, seed=i) for i in range(B)]

    def run(params, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            m.forward(ids, sids, lens, sampling_params_list=params)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    run(None, 3); run(sp, 3)
    greedy, sampled = [], []
    for _ in range(3):
        greedy.append(run(None, steps))
        sampled.append(run(sp, steps))
    gm, sm = min(greedy), min(sampled)
    print(json.dumps({"what": "decode_step", "B": B, "seqlen": S, "graph": True, "gpu": info, "greedy_ms": greedy,
                      "sampled_T0.8_p0.95_ms": sampled, "overhead_ms_best": sm - gm, "overhead_pct_best": 100 * (sm - gm) / gm}),
          flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--skip-model", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "sampling_bench.py measures on the GPU; there is nothing to measure without one"
    info = gpu_info()
    with torch.inference_mode():
        kernel_bench(args.iters, info)
    if not args.skip_model:
        model_bench(args.steps, info)


if __name__ == "__main__":
    main()
