#!/usr/bin/env python
"""Cost of log-probabilities (csrc/logprobs.cu) on the GPU.

1. Kernel time (CUDA events, mean over --iters launches) at B in {1, 8, 64, 256}, V = 128256 bf16, top-N in {0, 5, 20}, next to
   the torch equivalent (log_softmax in fp32 + gather + topk).
2. The bench.py decode step (Llama-3-8B shapes, batch 64 x 4096 tokens, CUDA-graph replay, greedy): forward() against
   forward_with_logprobs() with logprobs = 5 on every row, alternating blocks of --steps steps.

    python scripts/logprobs_bench.py [--iters 200] [--steps 30] [--skip-model]

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


def torch_logprobs(logits, tokens, n):
    lp = torch.log_softmax(logits.float(), dim=-1)
    tok = lp.gather(1, tokens[:, None])
    return (tok, torch.topk(lp, n, dim=-1)) if n else (tok,)


def kernel_bench(iters, info):
    from swiftllm_b200.worker.kernels.logprobs import token_logprobs
    V = 128256
    gen = torch.Generator(device="cuda").manual_seed(0)
    for B in (1, 8, 64, 256):
        logits = (torch.randn((B, V), device="cuda", generator=gen) * 3).to(torch.bfloat16)
        tokens = torch.argmax(logits, dim=1)
        row = {"what": "logprobs_kernel", "B": B, "V": V, "dtype": "bf16", "gpu": info, "bytes": B * V * 2}
        for n in (0, 5, 20):
            row[f"kernel_top{n}_us"] = 1e3 * time_ms(lambda: token_logprobs(logits, tokens, n), iters)
            row[f"torch_top{n}_us"] = 1e3 * time_ms(lambda: torch_logprobs(logits, tokens, n), iters)
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
    sp = [swiftllm_b200.SamplingParams(logprobs=5) for _ in range(B)]

    def run(with_lp, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            if with_lp:
                m.forward_with_logprobs(ids, sids, lens, sampling_params_list=sp)
            else:
                m.forward(ids, sids, lens)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    same = [r.token for r in m.forward_with_logprobs(ids, sids, lens, sampling_params_list=sp)] == m.forward(ids, sids, lens)
    run(False, 3); run(True, 3)
    plain, with_lp = [], []
    for _ in range(3):
        plain.append(run(False, steps))
        with_lp.append(run(True, steps))
    pm, lm = min(plain), min(with_lp)
    print(json.dumps({"what": "decode_step", "B": B, "seqlen": S, "graph": True, "gpu": info, "same_tokens": same,
                      "greedy_ms": plain, "greedy_logprobs5_ms": with_lp, "overhead_ms_best": lm - pm,
                      "overhead_pct_best": 100 * (lm - pm) / pm}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--skip-model", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "logprobs_bench.py measures on the GPU; there is nothing to measure without one"
    info = gpu_info()
    with torch.inference_mode():
        kernel_bench(args.iters, info)
    if not args.skip_model:
        model_bench(args.steps, info)


if __name__ == "__main__":
    main()
