#!/usr/bin/env python
"""Cost of repetition / frequency / presence penalties (csrc/penalties.cu) on the GPU.

1. Kernel time (CUDA events, mean over --iters launches) at B in {1, 8, 64, 256}, V = 128256 bf16, history 4096 and 32768 tokens
   in the token pages (decode rows, every row penalised), next to a torch version of the same semantics (scatter_add counts +
   where in fp32) on the same inputs; the outputs are asserted equal.
2. The bench.py decode step (Llama-3-8B shapes, batch 64 x 4096 tokens, CUDA-graph replay, greedy): forward() against the same
   step with repetition_penalty=1.1, frequency_penalty=0.5 on every row, alternating blocks of --steps steps.

    python scripts/penalties_bench.py [--iters 100] [--steps 30] [--skip-model]

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


def torch_penalties(logits, r, f, p, hist_ids, hist_out):
    """The same semantics in torch: hist_ids int64 [B, H], hist_out bool [B, H]."""
    B, V = logits.shape
    cnt = torch.zeros((B, V), dtype=torch.int32, device=logits.device).scatter_add_(1, hist_ids, hist_out.int())
    seen = torch.zeros((B, V), dtype=torch.bool, device=logits.device).scatter_(1, hist_ids, True)
    l = logits.float()
    l2 = torch.where(l > 0, l / r[:, None], l * r[:, None])
    t = f[:, None] * cnt.float()
    t = torch.where(cnt > 0, t + p[:, None], t)
    return torch.where(seen, (l2 - t).to(logits.dtype), logits)


def kernel_bench(iters, info):
    from swiftllm_b200.worker.kernels.penalties import apply_penalties
    V, bs = 128256, 16
    gen = torch.Generator(device="cuda").manual_seed(0)
    for H in (4096, 32768):
        for B in (1, 8, 64, 256):
            logits = (torch.randn((B, V), device="cuda", generator=gen) * 3).to(torch.bfloat16)
            pos = H + 1
            nblk = (pos + bs - 1) // bs
            bt = torch.arange(B * nblk, dtype=torch.int32, device="cuda").view(B, nblk)
            ids = torch.randint(0, V, (B, nblk * bs), device="cuda", generator=gen)
            out = torch.rand((B, nblk * bs), device="cuda", generator=gen) < 0.5
            pages = (ids | (out.long() << 31)).to(torch.int64).remainder(1 << 32)
            pages = torch.where(pages >= (1 << 31), pages - (1 << 32), pages).to(torch.int32).view(B * nblk, bs).contiguous()
            new = ids[:, H].to(torch.int32).contiguous()
            r = torch.full((B,), 1.1, device="cuda"); f = torch.full((B,), 0.5, device="cuda"); p = torch.full((B,), 0.3, device="cuda")
            posv = torch.full((B,), pos, dtype=torch.int32, device="cuda")
            sids = torch.arange(B, dtype=torch.int32, device="cuda")
            last = torch.arange(B, dtype=torch.int32, device="cuda")
            empty = torch.empty((0,), dtype=torch.int32, device="cuda")
            hist_ids = torch.cat([ids[:, :H], new[:, None].long()], dim=1)
            hist_out = torch.cat([out[:, :H], torch.ones((B, 1), dtype=torch.bool, device="cuda")], dim=1)
            work = logits.clone()

            def kernel():
                work.copy_(logits)
                apply_penalties(work, r, f, p, posv, sids, new, last, empty, 0, bt, pages)

            kernel()
            ref = torch_penalties(logits, r, f, p, hist_ids, hist_out)
            assert torch.equal(work.view(torch.int16), ref.view(torch.int16)), "kernel and torch disagree"
            copy_us = 1e3 * time_ms(lambda: work.copy_(logits), iters)
            row = {"what": "penalties_kernel", "B": B, "V": V, "history": H, "dtype": "bf16", "gpu": info,
                   "kernel_us": 1e3 * time_ms(kernel, iters) - copy_us,
                   "torch_us": 1e3 * time_ms(lambda: torch_penalties(logits, r, f, p, hist_ids, hist_out), iters),
                   "history_bytes": B * 4 * (H + 1)}
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
        # a recorded history of S - 1 tokens per sequence (the pages are what a penalised prefill + decodes would leave)
        m.token_cache.copy_(torch.randint(0, mc.vocab_size, tuple(m.token_cache.shape), generator=g, device="cuda",
                                          dtype=torch.int32))
    sids = list(range(B))
    lens = [S] * B
    ids = [[i % 1000] for i in range(B)]
    sp = [swiftllm_b200.SamplingParams(repetition_penalty=1.1, frequency_penalty=0.5) for _ in range(B)]

    def run(pen, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            m.forward(ids, sids, lens, sampling_params_list=sp if pen else None)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    run(False, 3); run(True, 3)
    plain, pen = [], []
    for _ in range(4):
        plain.append(run(False, steps))
        pen.append(run(True, steps))
    pm, qm = min(plain), min(pen)
    print(json.dumps({"what": "decode_step", "B": B, "seqlen": S, "graph": True, "gpu": info, "greedy_ms": plain,
                      "greedy_penalties_ms": pen, "spread_greedy_ms": max(plain) - pm, "spread_penalties_ms": max(pen) - qm,
                      "overhead_ms_best": qm - pm, "overhead_pct_best": 100 * (qm - pm) / pm}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--skip-model", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "penalties_bench.py measures on the GPU; there is nothing to measure without one"
    info = gpu_info()
    with torch.inference_mode():
        kernel_bench(args.iters, info)
    if not args.skip_model:
        model_bench(args.steps, info)


if __name__ == "__main__":
    main()
