#!/usr/bin/env python
"""Cost of multi-LoRA serving (csrc/lora.cu) on the GPU, at Llama-3-8B shapes (H 4096, 32 q / 8 kv heads of 128, F 14336).

1. Kernel time (CUDA events around the replay of a CUDA graph of --iters launches, so the host's launch cost is not timed) of the
   shrink and the expand at each of the four sites (qkv, o,
   up_gate, down), for T = 1, 8, 64, 256 decode rows with 1, 4 and T distinct slots, and a 4 x 4096 prefill with one slot, at
   R = 16 and 64.  Algorithmic bytes and FLOPs come from the shapes (shrink: x, the tiles' A, u; expand: y read and written, the
   tiles' B, u) and are reported against the H100 SXM data sheet (3.35 TB/s HBM3, 989 TFLOP/s dense fp16 / bf16) as the share of
   whichever bound is larger.  Repeated launches read their operands from L2 where they fit, so small shapes can exceed the
   HBM "bound".
2. The bench.py decode step (synthetic weights, batch 64 x 4096 tokens, CUDA-graph replay, greedy, bf16) with 0, 1 and 8 rank-64
   adapters (every row adapted; 8: row i on slot i % 8), alternating blocks of --steps steps.
3. A 4 x 4096-token prefill with and without one rank-64 adapter on every prompt.

    python scripts/lora_bench.py [--iters 100] [--steps 20] [--skip-model]

Prints one JSON line per measurement, with the GPU name and power limit."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from sampling_bench import gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet
TC_FLOPS = 989e12                   # dense fp16 / bf16 tensor-core rate, data sheet
H, NQ, NKV, D, F = 4096, 32, 8, 128, 14336
# site -> (K, N, slice ends, slices)
SITES = {"qkv": (H, (NQ + 2 * NKV) * D, (NQ * D, (NQ + NKV) * D), 3), "o": (NQ * D, H, (H, H), 1),
         "up_gate": (H, 2 * F, (F, 2 * F), 2), "down": (F, H, (H, H), 1)}


def graph_time_ms(fn, iters):
    """Mean time of one fn() launch: `iters` launches captured in one CUDA graph, replayed 5 times after a warm-up."""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (5 * iters)


def kernel_bench(iters, info):
    from swiftllm_b200.worker.kernels.lora import lora_expand, lora_shrink
    from swiftllm_b200.worker.lora import lora_tiles
    dt = torch.bfloat16
    cases = [(f"decode T={T} slots={n}", [i * n // T for i in range(T)], [1] * T) for T in (1, 8, 64, 256)
             for n in sorted({1, min(4, T), T})]
    cases.append(("prefill 4x4096 slots=1", [0] * 4, [4096] * 4))
    for R in (16, 64):
        for site, (K, N, ends, S) in SITES.items():
            nslots = 256
            A = torch.randn((nslots, S * R, K), dtype=dt, device="cuda") * 0.02
            B = torch.randn((nslots, N, R), dtype=dt, device="cuda") * 0.02
            scales = torch.ones((nslots,), dtype=torch.float32, device="cuda")
            mask = torch.full((nslots,), (1 << S) - 1, dtype=torch.int32, device="cuda")
            for name, slots, rows in cases:
                words = lora_tiles(slots, rows)
                tiles = torch.tensor(words, dtype=torch.int32, device="cuda").view(-1, 3)
                T = sum(rows)
                x = torch.randn((T, K), dtype=dt, device="cuda")
                y = torch.randn((T, N), dtype=dt, device="cuda")
                u = torch.empty((T, 3 * R), dtype=dt, device="cuda")
                n_tiles = tiles.shape[0]
                t_s = graph_time_ms(lambda: lora_shrink(x, u, A, tiles, mask), iters)
                t_e = graph_time_ms(lambda: lora_expand(y, u, B, ends, tiles, mask, scales), iters)
                by_s = 2 * (T * K + n_tiles * S * R * K + T * S * R)
                by_e = 2 * (2 * T * N + n_tiles * N * R + T * S * R)
                fl_s, fl_e = 2 * T * K * S * R, 2 * T * N * R
                out = {"what": "kernels", "site": site, "R": R, "case": name, "tiles": n_tiles, "gpu": info}
                for k, t, by, fl in (("shrink", t_s, by_s, fl_s), ("expand", t_e, by_e, fl_e)):
                    bound = max(by / HBM_BYTES_PER_S, fl / TC_FLOPS)
                    out[k] = {"us": round(1e3 * t, 2), "bytes": by, "flops": fl, "GB_s": round(by / t / 1e6, 1),
                              "bound": "hbm" if by / HBM_BYTES_PER_S >= fl / TC_FLOPS else "tensor",
                              "share_of_bound": round(bound / (t * 1e-3), 3)}
                print(json.dumps(out), flush=True)
            del A, B


def _adapter(mc, r, seed):
    """A rank-r adapter on every module of every layer, made on the device."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    shapes = {"q_proj": (NQ * D, H), "k_proj": (NKV * D, H), "v_proj": (NKV * D, H), "o_proj": (H, NQ * D),
              "up_proj": (F, H), "gate_proj": (F, H), "down_proj": (H, F)}
    tensors = {}
    for i in range(mc.num_layers):
        for m, (o, k) in shapes.items():
            blk = "self_attn" if m in ("q_proj", "k_proj", "v_proj", "o_proj") else "mlp"
            p = f"base_model.model.model.layers.{i}.{blk}.{m}."
            tensors[p + "lora_A.weight"] = torch.randn((r, k), generator=g, device="cuda", dtype=torch.bfloat16) * 0.01
            tensors[p + "lora_B.weight"] = torch.randn((o, r), generator=g, device="cuda", dtype=torch.bfloat16) * 0.01
    return dict(r=r, lora_alpha=2 * r, target_modules=list(shapes)), tensors


def model_bench(steps, info):
    import swiftllm_b200
    from bench import model_dict
    from swiftllm_b200.worker.weight import synthetic_getter
    B, S, bs, P = 64, 4096, 16, 4
    mc = swiftllm_b200.LlamaModelConfig(model_dict("llama3-8b"))
    bps = (S + bs - 1) // bs
    ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=bs, gpu_mem_utilization=0.97, num_cpu_blocks=0,
                                    max_seqs_in_block_table=B + P, max_blocks_per_seq=bps + 8, max_batch_size=B,
                                    max_tokens_in_batch=P * S, dtype="bfloat16", use_cuda_graph=True, max_loras=8,
                                    max_lora_rank=64)
    m = swiftllm_b200.LlamaModel(ec, mc)
    m.load_weights(synthetic_getter(seed=0, std=0.02, device="cuda"))
    for s in range(8):
        m.load_lora(s, _adapter(mc, 64, 100 + s))
    torch.cuda.empty_cache()
    nb = (B + P) * bps + 64
    m.init_kvcache_and_swap(nb)
    g = torch.Generator(device="cuda").manual_seed(1234)
    with torch.inference_mode():
        for s in range(0, nb, max(1, nb // 64)):
            m.k_cache[s:s + nb // 64].normal_(generator=g)
            m.v_cache[s:s + nb // 64].normal_(generator=g)
    sids, lens, ids = list(range(B)), [S] * B, [[i % 1000] for i in range(B)]
    mixes = {"0": None, "1": [0] * B, "8": [i % 8 for i in range(B)]}

    def run(mix, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            m.forward(ids, sids, lens, lora_ids_list=mixes[mix])
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    for k in mixes:
        run(k, 3)
    res = {k: [] for k in mixes}
    for _ in range(4):
        for k in mixes:
            res[k].append(run(k, steps))
    best = {k: min(v) for k, v in res.items()}
    print(json.dumps({"what": "decode_step", "B": B, "seqlen": S, "graph": True, "R": 64, "gpu": info, "ms": res,
                      "spread_ms": {k: max(v) - min(v) for k, v in res.items()},
                      "overhead_ms_best": {k: best[k] - best["0"] for k in ("1", "8")},
                      "overhead_pct_best": {k: 100 * (best[k] - best["0"]) / best["0"] for k in ("1", "8")},
                      "graphs": [list(map(str, key)) for key in m._graphs]}), flush=True)

    # prefill: 4 prompts of 4096 tokens on fresh sequences, with and without an adapter, alternating
    psids = list(range(B, B + P))
    prompts = [[(i * 7 + j) % 1000 for j in range(S)] for i in range(P)]

    def prefill(lora):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        m.forward(prompts, psids, [], lora_ids_list=[0] * P if lora else None)
        e1.record()
        torch.cuda.synchronize()
        m.free_seqs_resources(psids)
        return e0.elapsed_time(e1)

    prefill(False); prefill(True)
    pre = {"base": [], "lora": []}
    for _ in range(4):
        pre["base"].append(prefill(False))
        pre["lora"].append(prefill(True))
    b0, b1 = min(pre["base"]), min(pre["lora"])
    print(json.dumps({"what": "prefill", "prompts": P, "tokens": S, "R": 64, "gpu": info, "ms": pre,
                      "overhead_ms_best": b1 - b0, "overhead_pct_best": 100 * (b1 - b0) / b0}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--skip-model", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "lora_bench.py measures on the GPU; there is nothing to measure without one"
    info = gpu_info()
    with torch.inference_mode():
        kernel_bench(args.iters, info)
    if not args.skip_model:
        model_bench(args.steps, info)


if __name__ == "__main__":
    main()
