#!/usr/bin/env python
"""Cost of the min-p, typical-p and XTC filters (csrc/sampling.cu, sllm_sample_tokens_truncated) on the GPU.

1. Kernel time (CUDA events, mean over --iters launches) at B in {1, 8, 64, 256}, V = 128256 bf16, T = 0.8: top-p 0.95 through
   the plain kernel, then through the truncated kernel min-p 0.05, typical-p 0.95, XTC (threshold 0.1, probability 1) and all
   three with top-p 0.95.
2. The bench.py decode step (Llama-3-8B shapes, batch 64 x 4096 tokens, CUDA-graph replay): a top-p 0.95 step against a
   min-p 0.05 + typical-p 0.95 step, alternating blocks of --steps steps.

    python scripts/truncation_bench.py [--iters 200] [--steps 30] [--skip-model]

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

# (name, top_p, min_p, typical_p, xtc_threshold, xtc_probability); None: the plain kernel
KINDS = (("top_p0.95", 0.95, None, None, None, None), ("min_p0.05", 1.0, 0.05, 1.0, 0.1, 0.0),
         ("typical_p0.95", 1.0, 0.0, 0.95, 0.1, 0.0), ("xtc0.1_p1", 1.0, 0.0, 1.0, 0.1, 1.0),
         ("all_top_p0.95", 0.95, 0.05, 0.95, 0.1, 1.0))


def kernel_bench(iters, info):
    from swiftllm_b200.worker.kernels.sampling import sample_tokens
    V = 128256
    gen = torch.Generator(device="cuda").manual_seed(0)
    for B in (1, 8, 64, 256):
        logits = (torch.randn((B, V), device="cuda", generator=gen) * 3).to(torch.bfloat16)
        z = lambda v, dt: torch.full((B,), v, dtype=dt, device="cuda")      # noqa: E731
        seed = torch.arange(B, dtype=torch.int64, device="cuda")
        pos, t, k = z(4096, torch.int32), z(0.8, torch.float32), z(0, torch.int32)
        row = {"what": "truncation_kernel", "B": B, "V": V, "dtype": "bf16", "T": 0.8, "gpu": info, "bytes": B * V * 2}
        for name, p, *filt in KINDS:
            pp = z(p, torch.float32)
            kw = {} if filt[0] is None else dict(zip(("min_p", "typical_p", "xtc_threshold", "xtc_probability"),
                                                     (z(f, torch.float32) for f in filt)))
            row[f"{name}_us"] = 1e3 * time_ms(lambda: sample_tokens(logits, t, k, pp, seed, pos, **kw), iters)
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
    top_p = [swiftllm_b200.SamplingParams(0.8, top_p=0.95, seed=i) for i in range(B)]
    trunc = [swiftllm_b200.SamplingParams(0.8, min_p=0.05, typical_p=0.95, seed=i) for i in range(B)]

    def run(params, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            m.forward(ids, sids, lens, sampling_params_list=params)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    run(top_p, 3); run(trunc, 3)
    a, b = [], []
    for _ in range(3):
        a.append(run(top_p, steps))
        b.append(run(trunc, steps))
    am, bm = min(a), min(b)
    print(json.dumps({"what": "decode_step", "B": B, "seqlen": S, "graph": True, "gpu": info, "top_p0.95_ms": a,
                      "min_p0.05_typical_p0.95_ms": b, "overhead_ms_best": bm - am, "overhead_pct_best": 100 * (bm - am) / am}),
          flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--skip-model", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "truncation_bench.py measures on the GPU; there is nothing to measure without one"
    info = gpu_info()
    with torch.inference_mode():
        kernel_bench(args.iters, info)
    if not args.skip_model:
        model_bench(args.steps, info)


if __name__ == "__main__":
    main()
