#!/usr/bin/env python
"""Cost and benefit of FP8 weights (worker/fp8.py, csrc/fp8.cu) on the GPU, at Llama-3-8B shapes (32 layers, H 4096, 32 q / 8 kv
heads of 128, F 14336), synthetic weights, bf16 activations.

1. GEMMs: each projection's torch._scaled_mm (row-wise scales) against the bf16 cuBLAS GEMM at decode M = 1, 8, 32, 64 and a
   prefill M = 4096 (CUDA events around a CUDA graph of --iters launches), with the weight bytes per second against the H100
   SXM data sheet's 3.35 TB/s.
2. The quantizing kernels' time and algorithmic bytes per second at T = 64 and 4096 rows.
3. The engine, the bf16 and FP8 arms alternated (bf16, fp8, bf16, fp8; one model resident at a time): decode step time (CUDA
   graphs, greedy) at batch 1, 8, 32, 64 x context 512, 4096; prefill tokens per second for 4 x 4096; and the KV blocks
   profile_num_blocks finds at gpu_mem_utilization 0.9.

    python scripts/fp8_bench.py [--iters 50] [--steps 20] [--rounds 2] [--skip-model]

Prints one JSON line per measurement, with the GPU name and power limit."""
import argparse
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from lora_bench import graph_time_ms  # noqa: E402
from sampling_bench import gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet
H, NQ, NKV, D, F = 4096, 32, 8, 128, 14336
GEMMS = {"qkv": (H, (NQ + 2 * NKV) * D), "o": (NQ * D, H), "up_gate": (H, 2 * F), "down": (F, H)}     # (K, N)


def emit(info, **kw):
    print(json.dumps(dict(kw, gpu=info)), flush=True)


def gemm_bench(iters, info):
    from swiftllm_b200.worker.kernels.fp8 import quant_fp8_rows
    from swiftllm_b200.worker.kernels.linear import linear, linear_fp8
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, (K, N) in GEMMS.items():
        w = torch.randn(N, K, generator=g, device="cuda", dtype=torch.bfloat16) * 0.02
        wq, ws = quant_fp8_rows(w)
        ws = ws.view(-1)
        for M in (1, 8, 32, 64, 4096):
            x = torch.randn(M, K, generator=g, device="cuda", dtype=torch.bfloat16)
            xq, xs = quant_fp8_rows(x)
            t16 = graph_time_ms(lambda: linear(x, w), iters)
            t8 = graph_time_ms(lambda: linear_fp8(xq, xs, wq, ws, torch.bfloat16), iters)
            emit(info, what="gemm", proj=name, M=M, K=K, N=N, bf16_us=round(t16 * 1e3, 2), fp8_us=round(t8 * 1e3, 2),
                 bf16_weight_share_of_hbm=round(2 * N * K / (t16 * 1e-3) / HBM_BYTES_PER_S, 3),
                 fp8_weight_share_of_hbm=round(N * K / (t8 * 1e-3) / HBM_BYTES_PER_S, 3), fp8_faster=t8 < t16)
        del w, wq


def quant_bench(iters, info):
    from swiftllm_b200.worker.kernels.fp8 import fused_add_rmsnorm_quant_fp8, quant_fp8_rows, silu_and_mul_quant_fp8
    g = torch.Generator(device="cuda").manual_seed(1)
    for T in (64, 4096):
        x = torch.randn(T, H, generator=g, device="cuda", dtype=torch.bfloat16)
        r = torch.randn(T, H, generator=g, device="cuda", dtype=torch.bfloat16)
        nw = torch.ones(H, device="cuda", dtype=torch.bfloat16)
        ug = torch.randn(T, 2 * F, generator=g, device="cuda", dtype=torch.bfloat16)
        for name, fn, nbytes in (
                ("add_rmsnorm_quant", lambda: fused_add_rmsnorm_quant_fp8(x, r, nw, 1e-5), 3 * T * H * 2 + T * H + 4 * T + 2 * H),
                ("silu_and_mul_quant", lambda: silu_and_mul_quant_fp8(ug), 2 * T * F * 2 + T * F + 4 * T),
                ("quant_rows", lambda: quant_fp8_rows(x), T * H * 2 + T * H + 4 * T)):
            t = graph_time_ms(fn, iters)
            emit(info, what="quant_kernel", kernel=name, T=T, us=round(t * 1e3, 2),
                 bytes_per_s=round(nbytes / (t * 1e-3) / 1e9, 1), unit="GB/s",
                 share_of_hbm=round(nbytes / (t * 1e-3) / HBM_BYTES_PER_S, 3))


def engine(quantization, max_tokens):
    import swiftllm_b200
    from swiftllm_b200.model_config import LLAMA3_8B
    from swiftllm_b200.worker.weight import synthetic_getter
    ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=0,
                                    max_seqs_in_block_table=64, max_blocks_per_seq=320, max_batch_size=64,
                                    max_tokens_in_batch=max_tokens, dtype="bfloat16", use_cuda_graph=True,
                                    quantization=quantization)
    m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(LLAMA3_8B))
    m.load_weights(synthetic_getter(seed=0))
    return m


def model_arm(quantization, steps, info, rnd):
    m = engine(quantization, 16384)
    blocks = m.profile_num_blocks()
    emit(info, what="kv_blocks", quantization=quantization, round=rnd, blocks=blocks, tokens=blocks * 16)
    m.init_kvcache_and_swap(min(blocks, 64 * 4200 // 16 + 64))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    prompts = [[(7 * i + j) % 128000 for j in range(4096)] for i in range(4)]
    m.forward(prompts, [0, 1, 2, 3], [])            # warm-up
    m.free_seqs_resources([0, 1, 2, 3])
    torch.cuda.synchronize()
    e0.record()
    m.forward_async(prompts, [0, 1, 2, 3], [])
    e1.record()
    torch.cuda.synchronize()
    m.free_seqs_resources([0, 1, 2, 3])
    emit(info, what="prefill", quantization=quantization, round=rnd, tokens=4 * 4096,
         tok_per_s=round(4 * 4096 / (e0.elapsed_time(e1) * 1e-3)))
    for B in (1, 8, 32, 64):
        for ctx in (512, 4096):
            sids = list(range(B))
            for i in range(3):
                m.forward_async([[1]] * B, sids, [ctx + i] * B)
            torch.cuda.synchronize()
            e0.record()
            for i in range(steps):
                m.forward_async([[1]] * B, sids, [ctx + 3 + i] * B)
            e1.record()
            torch.cuda.synchronize()
            m.free_seqs_resources(sids)
            emit(info, what="decode_step", quantization=quantization, round=rnd, batch=B, context=ctx,
                 ms=round(e0.elapsed_time(e1) / steps, 3))
    del m
    gc.collect()
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--skip-model", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "fp8_bench.py measures on the GPU"
    info = gpu_info()
    with torch.inference_mode():
        gemm_bench(args.iters, info)
        quant_bench(args.iters, info)
        if not args.skip_model:
            for rnd in range(args.rounds):
                for q in (None, "fp8"):
                    model_arm(q, args.steps, info, rnd)


if __name__ == "__main__":
    main()
