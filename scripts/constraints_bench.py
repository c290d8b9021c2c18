#!/usr/bin/env python
"""Cost of constrained decoding (allowed-token masks and logit bias, csrc/constraints.cu) on the GPU.

1. Kernel time (CUDA events, mean over --iters launches) at V = 128256 bf16, B in {1, 8, 64, 256}, every row masked with one
   allowed id, 1 % or 50 % of the ids allowed, and 0 or 300 bias entries per row; achieved bytes/s from the algorithmic bytes
   (4 * W mask words + 2 * disallowed ids written + 12 * bias entries per row) and their share of the 3.35 TB/s data-sheet HBM3
   bandwidth of the H100 SXM.  Masking is idempotent and the bias add's cost does not depend on the values, so the launches run
   back to back on the same buffer; the first launch's output is checked against tests/constraints_oracle.py.
2. The bench.py decode step (Llama-3-8B shapes, synthetic weights, batch 64 x 4096 tokens, CUDA-graph replay, greedy):
   forward() against the same step with a fresh 50 % mask on every row each step (about 1 MB more in the step's one staged
   copy), alternating blocks of --steps steps.

    python scripts/constraints_bench.py [--iters 200] [--steps 30] [--skip-model]

Prints one JSON line per measurement, with the GPU name and power limit."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from sampling_bench import gpu_info, time_ms  # noqa: E402

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet


def _region(B, V, allowed, n_bias, rng, graph=False):
    from swiftllm_b200 import SamplingParams, token_mask
    from swiftllm_b200.sampling_params import constraint_words
    masks, disallowed = [], 0
    for _ in range(B):
        ids = [int(rng.integers(0, V))] if allowed == "one" else np.flatnonzero(rng.random(V) < allowed)
        masks.append(token_mask(V, ids))
        disallowed += V - len(ids)
    sp = [SamplingParams(logit_bias={int(v): 1.0 for v in rng.choice(V, n_bias, replace=False)} or None) for _ in range(B)]
    return constraint_words(masks, sp, B, V, graph=graph), masks, sp, disallowed


def kernel_bench(iters, info):
    import constraints_oracle as CO
    from swiftllm_b200.worker.infer_state import ConstraintState
    from swiftllm_b200.worker.kernels.constraints import constrain_logits
    V = 128256
    W = (V + 31) // 32
    rng = np.random.default_rng(0)
    gen = torch.Generator(device="cuda").manual_seed(0)
    for B in (1, 8, 64, 256):
        logits = (torch.randn((B, V), device="cuda", generator=gen) * 3).to(torch.bfloat16)
        for allowed in ("one", 0.01, 0.5):
            for n_bias in (0, 300):
                cw, masks, sp, disallowed = _region(B, V, allowed, n_bias, rng)
                st = ConstraintState.from_staged(torch.from_numpy(cw.words).cuda(), *cw[1:])
                work = logits.clone()
                args = (st.mask_index, st.masks, st.bias_index, st.bias_starts, st.bias_ids, st.bias_values)
                constrain_logits(work, *args)
                if B <= 8:
                    want = CO.constrain(logits.cpu(), masks, [s.logit_bias for s in sp])
                    assert torch.equal(work.cpu().view(torch.int16), want.view(torch.int16)), "kernel and restatement disagree"
                us = 1e3 * time_ms(lambda: constrain_logits(work, *args), iters)
                nbytes = B * 4 * W + 2 * disallowed + 12 * B * n_bias
                print(json.dumps({"what": "constrain_kernel", "B": B, "V": V, "dtype": "bf16", "allowed": allowed,
                                  "bias_entries": n_bias, "gpu": info, "kernel_us": us, "algorithmic_bytes": nbytes,
                                  "achieved_GBps": nbytes / us / 1e3, "share_of_3.35TBps": nbytes / (us * 1e-6) / HBM_BYTES_PER_S}),
                      flush=True)


def model_bench(steps, info):
    import swiftllm_b200
    from bench import model_dict
    from swiftllm_b200.worker.weight import synthetic_getter
    B, S, bs = 64, 4096, 16
    mc = swiftllm_b200.LlamaModelConfig(model_dict("llama3-8b"))
    V = mc.vocab_size
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
    rng = np.random.default_rng(5)
    # 16 mask sets made ahead (making a 50 % mask is host work of the caller's grammar engine, not of this step); each step
    # takes the next one, so consecutive steps never pass the same masks
    pool = [[swiftllm_b200.token_mask(V, np.flatnonzero(rng.random(V) < 0.5)) for _ in range(B)] for _ in range(16)]
    k = [0]

    def run(con, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            masks = None
            if con:
                masks = pool[k[0] % len(pool)]
                k[0] += 1
            m.forward(ids, sids, lens, token_masks_list=masks)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / n

    run(False, 3); run(True, 3)
    plain, con = [], []
    for _ in range(4):
        plain.append(run(False, steps))
        con.append(run(True, steps))
    pm, qm = min(plain), min(con)
    print(json.dumps({"what": "decode_step", "B": B, "seqlen": S, "graph": True, "gpu": info, "greedy_ms": plain,
                      "greedy_constrained_ms": con, "spread_greedy_ms": max(plain) - pm, "spread_constrained_ms": max(con) - qm,
                      "overhead_ms_best": qm - pm, "overhead_pct_best": 100 * (qm - pm) / pm,
                      "graphs": [list(map(str, key)) for key in m._graphs]}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--skip-model", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "constraints_bench.py measures on the GPU; there is nothing to measure without one"
    info = gpu_info()
    with torch.inference_mode():
        kernel_bench(args.iters, info)
    if not args.skip_model:
        model_bench(args.steps, info)


if __name__ == "__main__":
    main()
