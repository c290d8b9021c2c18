#!/usr/bin/env python
"""Cost of prompt log-probabilities (csrc/prompt_logprobs.cu) on the GPU.

1. Kernel time (CUDA events, mean over --iters launches) at rows in {64, 256, 1024, 4096, 16384}, V = 128256 bf16, top-N in
   {0, 5, 20}, next to sllm_token_logprobs on the same rows and the torch equivalent (fp32 log_softmax + gather + topk +
   (l > l_target).sum); the outputs are asserted identical to both.  Also the share of the data-sheet HBM bandwidth
   (3.35 TB/s) the kernel reaches on rows * V * 2 bytes of logits.
2. A whole-prompt prefill step at Llama-3-8B shapes (synthetic weights, 1 x 4096 and 4 x 4096 tokens, ignore_kvcache): forward()
   against forward_with_logprobs() with prompt_logprobs in {0, 5} on every entry, alternating blocks of --steps steps, next to
   the lm_head GEMM over the same rows.

    python scripts/prompt_logprobs_bench.py [--iters 50] [--steps 5] [--skip-model] [--skip-kernel]

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

HBM_BYTES_PER_S = 3.35e12


def torch_prompt_logprobs(logits, targets, n):
    lf = logits.float()
    lp = torch.log_softmax(lf, dim=-1)
    tok = lp.gather(1, targets[:, None])
    rank = 1 + (lf > lf.gather(1, targets[:, None])).sum(dim=1)
    return (tok, rank, torch.topk(lp, n, dim=-1)) if n else (tok, rank)


def kernel_bench(iters, info):
    from swiftllm_b200.worker.kernels.logprobs import prompt_logprobs, token_logprobs
    V = 128256
    gen = torch.Generator(device="cuda").manual_seed(0)
    for R in (64, 256, 1024, 4096, 16384):
        logits = (torch.randn((R, V), device="cuda", generator=gen) * 3).to(torch.bfloat16)
        targets = torch.randint(0, V, (R,), device="cuda", generator=gen, dtype=torch.int32)
        t64 = targets.long()
        row = {"what": "prompt_logprobs_kernel", "rows": R, "V": V, "dtype": "bf16", "gpu": info, "bytes": R * V * 2}
        for n in (0, 5, 20):
            lp, rank, ids, tlp = prompt_logprobs(logits, targets, n)
            t_lp, t_ids, t_tlp = token_logprobs(logits, t64, n)
            assert torch.equal(lp.view(torch.int32), t_lp.view(torch.int32)), "logprobs differ from token_logprobs"
            assert torch.equal(ids, t_ids) and torch.equal(tlp.view(torch.int32), t_tlp.view(torch.int32))
            ref = torch_prompt_logprobs(logits, t64, n)
            assert torch.equal(rank.long(), ref[1]), "ranks differ from torch"
            if n:                                            # torch.topk orders ties arbitrarily: compare the logits
                assert torch.equal(logits.gather(1, ids.long()), logits.gather(1, ref[2].indices))
            assert float((lp - ref[0][:, 0]).abs().max()) <= 2e-5
            del ref
            us = 1e3 * time_ms(lambda: prompt_logprobs(logits, targets, n), iters)
            row[f"kernel_top{n}_us"] = us
            row[f"kernel_top{n}_hbm_share"] = R * V * 2 / (us * 1e-6) / HBM_BYTES_PER_S
            row[f"token_kernel_top{n}_us"] = 1e3 * time_ms(lambda: token_logprobs(logits, t64, n), max(3, iters // 4))
            row[f"torch_top{n}_us"] = 1e3 * time_ms(lambda: torch_prompt_logprobs(logits, t64, n), max(3, iters // 4))
        print(json.dumps(row), flush=True)
        del logits


def model_bench(steps, info):
    import swiftllm_b200
    from bench import model_dict
    from swiftllm_b200.worker.kernels.linear import linear
    from swiftllm_b200.worker.weight import synthetic_getter
    S, bs = 4096, 16
    mc = swiftllm_b200.LlamaModelConfig(model_dict("llama3-8b"))
    ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=bs, gpu_mem_utilization=0.9, num_cpu_blocks=0,
                                    max_seqs_in_block_table=8, max_blocks_per_seq=S // bs + 8, max_batch_size=4,
                                    max_tokens_in_batch=4 * S, dtype="bfloat16")
    m = swiftllm_b200.LlamaModel(ec, mc)
    m.load_weights(synthetic_getter(seed=0, std=0.02, device="cuda"))
    m.init_kvcache_and_swap(64)
    gen = torch.Generator().manual_seed(1)

    def timed(fn, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    for B in (1, 4):
        prompts = [torch.randint(0, mc.vocab_size, (S,), generator=gen).tolist() for _ in range(B)]
        sids = list(range(B))
        x = torch.randn((B * S, mc.hidden_size), device="cuda").to(torch.bfloat16)
        timed(lambda: linear(x, m.weight.lm_head), 2)                   # GEMM heuristics and workspace for this shape
        gemm_ms = min(timed(lambda: linear(x, m.weight.lm_head), steps) for _ in range(3))
        del x
        for n in (0, 5):
            sp = [swiftllm_b200.SamplingParams(prompt_logprobs=n) for _ in range(B)]
            plain = lambda: m.forward(prompts, sids, [], ignore_kvcache=True)
            asked = lambda: m.forward_with_logprobs(prompts, sids, [], ignore_kvcache=True, sampling_params_list=sp)
            same = [r.token for r in asked()] == plain()
            timed(plain, 1); timed(asked, 1)
            pl, wl = [], []
            for _ in range(3):
                pl.append(timed(plain, steps))
                wl.append(timed(asked, steps))
            print(json.dumps({"what": "prefill_step", "prompts": B, "prompt_len": S, "prompt_logprobs": n, "gpu": info,
                              "same_tokens": same, "forward_ms": pl, "with_prompt_logprobs_ms": wl,
                              "added_ms_best": min(wl) - min(pl), "lm_head_gemm_ms_same_rows": gemm_ms,
                              "block_rows": m._prompt_block_rows()}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--skip-model", action="store_true")
    ap.add_argument("--skip-kernel", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "prompt_logprobs_bench.py measures on the GPU; there is nothing to measure without one"
    info = gpu_info()
    with torch.inference_mode():
        if not args.skip_kernel:
            kernel_bench(args.iters, info)
        if not args.skip_model:
            model_bench(args.steps, info)


if __name__ == "__main__":
    main()
