#!/usr/bin/env python
"""Cost of speculative verification (LlamaModel.forward_speculative, csrc/paged_attn_tc.cu paged_attn_verify_kernel) on one GPU.

1. Kernel time (CUDA events, mean over --iters launches), Llama-3-8B attention heads (32 q / 8 kv, head_dim 128, bf16), context
   4096 cached tokens, B in {1, 8, 64} entries of rows in {1, 2, 4, 8}: the verify kernel, sllm_paged_attention (rows = 1 only)
   and sllm_prefill_attention_paged on the same rows.  Algorithmic bytes = every entry's K/V over its visible length
   (sum_i (prefix_i + rows_i) * nkv * 128 * 2 * 2 B) + Q and O of every row (2 * T * nq * 128 * 2 B), as a fraction of the
   H100 SXM data-sheet 3.35 TB/s.
2. Step time on the bench.py workload shapes (Llama-3-8B, synthetic weights, bf16, 4087 cached tokens per sequence, batch 64,
   8 and 1): forward() eager and graph-replayed against forward_speculative with 1 / 2 / 4 / 8 rows (drafts that are rejected, so
   every call repeats the same state), alternating the arms in blocks of --steps steps.  From the best block of each arm: the
   number of accepted drafts per step a speculative step must average to break even with a graph-replayed decode step, and the
   per-draft acceptance rate alpha that gives it when each draft is accepted independently with probability alpha.

    python scripts/speculative_bench.py [--iters 100] [--steps 20] [--skip-model]

Prints one JSON line per measurement, with the GPU name and power limit."""
import argparse
import json
import os
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from sampling_bench import gpu_info, time_ms  # noqa: E402

HBM = 3.35e12
NQ, NKV, D, BS, CTX = 32, 8, 128, 16, 4096


def _i32(x):
    return torch.tensor(list(x), dtype=torch.int32, device="cuda")


def kernel_bench(iters, info):
    from swiftllm_b200.worker.kernels.paged_attn import paged_attention
    from swiftllm_b200.worker.kernels.prefill_attn import paged_attention_verify, prefill_attention_paged
    dt = torch.bfloat16
    bps = (CTX + 8 + BS - 1) // BS
    gen = torch.Generator(device="cuda").manual_seed(0)
    Bmax = 64
    kc = torch.randn((Bmax * bps, 1, NKV, BS, D), device="cuda", generator=gen).to(dt)
    vc = torch.randn_like(kc)
    bt = torch.randperm(Bmax * bps, device="cuda", generator=gen).to(torch.int32).view(Bmax, bps).contiguous()
    for B in (1, 8, 64):
        for r in (1, 2, 4, 8):
            T = B * r
            q = torch.randn((T, NQ, D), device="cuda", generator=gen).to(dt)
            o_v, o_p = torch.empty_like(q), torch.empty_like(q)
            st = SimpleNamespace(seq_ids=_i32(range(B)), prefill_prefix_lens=_i32([CTX] * B), num_prefill_seqs=B,
                                 max_prefill_kv_len=CTX + r, prefill_seq_start_locs=_i32(range(0, T, r)),
                                 prefill_seq_lens=_i32([r] * B), max_prefill_len=r, softmax_scale=D ** -0.5)
            verify = lambda: paged_attention_verify(q, kc, vc, bt, o_v, None, None, st, 0)      # noqa: E731
            prefill = lambda: prefill_attention_paged(q, kc, vc, bt, o_p, None, None, st, 0)     # noqa: E731
            verify(); prefill()
            torch.cuda.synchronize()
            diff = float((o_v.float() - o_p.float()).abs().max())
            nbytes = B * (CTX + r) * NKV * D * 2 * 2 + 2 * T * NQ * D * 2
            row = {"what": "verify_kernel", "B": B, "rows": r, "context": CTX, "dtype": "bf16", "gpu": info,
                   "verify_us": 1e3 * time_ms(verify, iters), "prefill_paged_us": 1e3 * time_ms(prefill, iters),
                   "bytes": nbytes, "max_abs_diff_verify_vs_prefill": diff}
            if r == 1:
                dst = SimpleNamespace(paged_attn_seq_block_size=0, seq_ids=_i32(range(B)), num_prefill_seqs=0,
                                      decoding_seq_lens=_i32([CTX + 1] * B), max_decoding_len=CTX + 1, softmax_scale=D ** -0.5)
                o_d = torch.empty((B, NQ * D), dtype=dt, device="cuda")
                row["paged_decode_us"] = 1e3 * time_ms(
                    lambda: paged_attention(q, kc, vc, bt, None, SimpleNamespace(block_size=BS), dst, 0, o_d), iters)
            for k in ("verify_us", "prefill_paged_us", "paged_decode_us"):
                if k in row:
                    row[k.replace("_us", "_hbm_frac")] = nbytes / (row[k] * 1e-6) / HBM
            print(json.dumps(row), flush=True)


def _alpha_for(tokens_per_step, k):
    """Per-draft acceptance rate alpha with E[tokens] = (1 - alpha^(k+1)) / (1 - alpha) = tokens_per_step (None if > k + 1)."""
    if tokens_per_step > k + 1:
        return None
    lo, hi = 0.0, 1.0
    for _ in range(60):
        a = (lo + hi) / 2
        e = sum(a ** i for i in range(k + 1))
        lo, hi = (a, hi) if e < tokens_per_step else (lo, a)
    return (lo + hi) / 2


def model_bench(steps, info):
    import swiftllm_b200
    from bench import model_dict
    from swiftllm_b200.worker.weight import synthetic_getter
    # S - 1 + 8 rows stay inside the 256 pages of a 4096-token sequence: an accepted draft never leaves a sequence with more
    # blocks than the plain arm's step expects
    Bmax, S = 64, CTX - 8
    mc = swiftllm_b200.LlamaModelConfig(model_dict("llama3-8b"))
    bps = (S + 8 + BS - 1) // BS
    ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=BS, gpu_mem_utilization=0.97, num_cpu_blocks=0,
                                    max_seqs_in_block_table=Bmax, max_blocks_per_seq=bps + 8, max_batch_size=Bmax,
                                    max_tokens_in_batch=16384, dtype="bfloat16", use_cuda_graph=True)
    m = swiftllm_b200.LlamaModel(ec, mc)
    m.load_weights(synthetic_getter(seed=0, std=0.02, device="cuda"))
    nb = Bmax * bps + 64
    m.init_kvcache_and_swap(nb)
    g = torch.Generator(device="cuda").manual_seed(1234)
    with torch.inference_mode():
        for s in range(0, nb, max(1, nb // 64)):
            m.k_cache[s:s + nb // 64].normal_(generator=g)
            m.v_cache[s:s + nb // 64].normal_(generator=g)
    # every sequence holds S - 1 cached tokens; a plain step feeds token S
    m.gpu_block_manager.allocate_blocks_for_seqs(_i32(range(Bmax)), _i32([S - 1] * Bmax), seq_ids_list=list(range(Bmax)),
                                                 target_lens_list=[S - 1] * Bmax, want_new_blocks=False)
    for B in (64, 8, 1):
        sids = list(range(B))
        ids = [[1000 + i] for i in range(B)]

        def plain(graph, n):
            m.engine_config.use_cuda_graph = graph
            for _ in range(n):
                m.forward(ids, sids, [S] * B)

        def spec(r, n):
            # drafts no model would produce for these synthetic weights: rejected, so each call leaves the same state
            e = [[1000 + i] + [(7 * i + j) % 50 for j in range(r - 1)] for i in range(B)]
            for _ in range(n):
                m.forward_speculative(e, sids, [S - 1] * B)

        arms = {"graph": lambda n: plain(True, n), "eager": lambda n: plain(False, n)}
        for r in (1, 2, 4, 8):
            arms[f"spec{r}"] = (lambda rr: lambda n: spec(rr, n))(r)
        res = {k: [] for k in arms}
        for fn in arms.values():
            fn(3)
        for _ in range(4):
            for k, fn in arms.items():
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn(steps)
                e1.record()
                torch.cuda.synchronize()
                res[k].append(e0.elapsed_time(e1) / steps)
        best = {k: min(v) for k, v in res.items()}
        row = {"what": "step", "B": B, "seqlen": S, "gpu": info, "ms": res, "best_ms": best,
               "spread_ms": {k: max(v) - min(v) for k, v in res.items()}}
        for r in (2, 4, 8):
            t = best[f"spec{r}"] / best["graph"]
            row[f"spec{r}_break_even_accepted_drafts"] = t - 1
            row[f"spec{r}_break_even_alpha"] = _alpha_for(t, r - 1)
        print(json.dumps(row), flush=True)
    m.engine_config.use_cuda_graph = True


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--skip-model", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "speculative_bench.py measures on the GPU; there is nothing to measure without one"
    info = gpu_info()
    print(json.dumps({"gpu": info}), flush=True)
    with torch.inference_mode():
        kernel_bench(args.iters, info)
    if not args.skip_model:
        model_bench(args.steps, info)


if __name__ == "__main__":
    main()
