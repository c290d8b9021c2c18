#!/usr/bin/env python
"""Cost of the no-repeat n-gram ban and DRY (the penalty kernel's n-gram launch, csrc/penalties.cu) on the GPU.

1. Kernel time (CUDA events, mean over --iters launches) at B in {1, 8, 64, 256}, V = 128256 bf16, history 4096 and 32768 tokens
   in the token pages (decode rows): penalties only (the plain launch), penalties + DRY + ban on a Zipf-like history, and the
   same on the adversarial history of one repeated token (every position matches 50 deep).
2. The bench.py decode step (Llama-3-8B shapes, batch 64 x 4096 tokens, CUDA-graph replay) in alternating blocks of --steps
   steps: greedy, penalties only, and penalties + DRY + ban on every row.

    python scripts/ngram_bench.py [--iters 50] [--steps 30] [--skip-model]

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


def _pages(ids, out):
    w = (ids | (out.long() << 31)).remainder(1 << 32)
    return torch.where(w >= (1 << 31), w - (1 << 32), w).to(torch.int32)


def kernel_bench(iters, info):
    from swiftllm_b200.worker.kernels.penalties import apply_penalties
    V, bs = 128256, 16
    gen = torch.Generator(device="cuda").manual_seed(0)
    zipf = 1.0 / torch.arange(1, V + 1, dtype=torch.float64, device="cuda")
    for H in (4096, 32768):
        for B in (1, 8, 64, 256):
            logits = (torch.randn((B, V), device="cuda", generator=gen) * 3).to(torch.bfloat16)
            pos = H + 1
            nblk = (pos + bs - 1) // bs
            bt = torch.arange(B * nblk, dtype=torch.int32, device="cuda").view(B, nblk)
            out = torch.rand((B, nblk * bs), device="cuda", generator=gen) < 0.5
            hists = {"zipf": torch.multinomial(zipf, B * nblk * bs, replacement=True, generator=gen).view(B, nblk * bs),
                     "one_token": torch.full((B, nblk * bs), 13, dtype=torch.int64, device="cuda")}
            f32 = lambda v: torch.full((B,), v, dtype=torch.float32, device="cuda")        # noqa: E731
            r, f, p = f32(1.1), f32(0.5), f32(0.3)
            ngram = dict(no_repeat_ngram_size=torch.full((B,), 3, dtype=torch.int32, device="cuda"),
                         dry_allowed_length=torch.full((B,), 2, dtype=torch.int32, device="cuda"), dry_multiplier=f32(0.8),
                         dry_base=f32(1.75), dry_breakers=torch.full((B, 16), -1, dtype=torch.int32, device="cuda"))
            ngram["dry_breakers"][:, :4] = torch.tensor([198, 25, 1, 9], dtype=torch.int32)
            posv = torch.full((B,), pos, dtype=torch.int32, device="cuda")
            sids = torch.arange(B, dtype=torch.int32, device="cuda")
            last = torch.arange(B, dtype=torch.int32, device="cuda")
            empty = torch.empty((0,), dtype=torch.int32, device="cuda")
            work = logits.clone()
            copy_us = 1e3 * time_ms(lambda: work.copy_(logits), iters)
            row = {"what": "ngram_kernel", "B": B, "V": V, "history": H, "dtype": "bf16", "gpu": info}
            for name, ids in (("zipf", hists["zipf"]), ("one_token", hists["one_token"])):
                pages = _pages(ids, out).view(B * nblk, bs).contiguous()
                new = ids[:, H].to(torch.int32).contiguous()
                for arm, kw in (("penalties", {}), ("ngram", ngram)):

                    def kernel():
                        work.copy_(logits)
                        apply_penalties(work, r, f, p, posv, sids, new, last, empty, 0, bt, pages, **kw)

                    kernel()
                    row[f"{arm}_{name}_us"] = 1e3 * time_ms(kernel, iters) - copy_us
            for name in ("zipf", "one_token"):
                row[f"{name}_ngram_over_penalties"] = row[f"ngram_{name}_us"] / row[f"penalties_{name}_us"]
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
        # a recorded history of S - 1 tokens per sequence from a small vocabulary, so n-grams repeat
        m.token_cache.copy_(torch.randint(0, 64, tuple(m.token_cache.shape), generator=g, device="cuda", dtype=torch.int32))
    sids = list(range(B))
    lens = [S] * B
    ids = [[i % 64] for i in range(B)]
    arms = {"greedy": None,
            "penalties": [swiftllm_b200.SamplingParams(repetition_penalty=1.1, frequency_penalty=0.5) for _ in range(B)],
            "penalties_dry_ban": [swiftllm_b200.SamplingParams(repetition_penalty=1.1, frequency_penalty=0.5, dry_multiplier=0.8,
                                                               no_repeat_ngram_size=3, dry_sequence_breakers=(1, 9))
                                  for _ in range(B)]}

    def run(sp, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            m.forward(ids, sids, lens, sampling_params_list=sp)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    for sp in arms.values():
        run(sp, 3)
    times = {k: [] for k in arms}
    for _ in range(4):
        for k, sp in arms.items():
            times[k].append(run(sp, steps))
    best = {k: min(v) for k, v in times.items()}
    print(json.dumps({"what": "decode_step", "B": B, "seqlen": S, "graph": True, "gpu": info,
                      **{f"{k}_ms": v for k, v in times.items()},
                      **{f"spread_{k}_ms": max(v) - best[k] for k, v in times.items()},
                      "ngram_over_penalties_ms_best": best["penalties_dry_ban"] - best["penalties"],
                      "ngram_over_greedy_pct_best": 100 * (best["penalties_dry_ban"] - best["greedy"]) / best["greedy"]}),
          flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--skip-model", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "ngram_bench.py measures on the GPU; there is nothing to measure without one"
    info = gpu_info()
    with torch.inference_mode():
        kernel_bench(args.iters, info)
    if not args.skip_model:
        model_bench(args.steps, info)


if __name__ == "__main__":
    main()
