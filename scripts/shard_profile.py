#!/usr/bin/env python
"""Per-kernel launch list of ONE tensor-parallel shard's decode step on a single GPU (development tool).

    python scripts/shard_profile.py --tp 8 [--batch 256] [--seqlen 4096] [--fuse-rotary-store]

Runs rank 0's shard of a TP=<tp> model (q/kv heads, FFN columns and KV cache divided by <tp>) in a world-size-1 process
group: every kernel has exactly the shapes it has on an 8-GPU box, only the exchange is missing (the all-reduce of a
1-rank group moves nothing).  What it is for: the multi-GPU box is charged per GPU, and ncu cannot attach to a multi-rank
job - this gives the GEMM / attention / elementwise split of the TP step, and a place to A/B single-GPU changes at TP
shapes, for one GPU-minute.  Its step time is NOT a TP number (no exchange) and is never reported as one."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tp", type=int, default=8)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seqlen", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--model", default="llama3-8b", choices=["llama3-8b", "llama3-70b"])
    ap.add_argument("--fuse-rotary-store", action="store_true")
    ap.add_argument("--tag", default="")
    args = ap.parse_args()
    import torch.distributed as dist
    import swiftllm_b200
    from swiftllm_b200.model_config import LLAMA3_8B, LLAMA3_70B
    from swiftllm_b200.worker.weight import synthetic_getter
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1"); os.environ.setdefault("MASTER_PORT", "29431")
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=dev)
    mc = swiftllm_b200.LlamaModelConfig(dict(LLAMA3_8B if args.model == "llama3-8b" else LLAMA3_70B))
    B, S, bs = args.batch, args.seqlen, 16
    bps = (S + bs - 1) // bs
    nblk = B * bps + 64
    with torch.inference_mode():
        ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=bs, gpu_mem_utilization=0.97, num_cpu_blocks=0,
                                        max_seqs_in_block_table=B, max_blocks_per_seq=bps + 8, max_batch_size=B, max_tokens_in_batch=max(B, 4096),
                                        dtype="bfloat16", tp_size=args.tp, tp_rank=0, use_cuda_graph=True, fused_allreduce=False,
                                        fuse_rotary_store=args.fuse_rotary_store)
        m = swiftllm_b200.LlamaModel(ec, mc)
        m.load_weights(synthetic_getter(seed=0, std=0.02, device=dev))
        m.init_kvcache_and_swap(nblk)
        g = torch.Generator(device=dev); g.manual_seed(1)
        ch = max(1, nblk // 16)
        for s in range(0, nblk, ch):
            m.k_cache[s:s + ch].normal_(generator=g); m.v_cache[s:s + ch].normal_(generator=g)
        gen = torch.Generator().manual_seed(7)
        ids = [[int(t)] for t in torch.randint(0, mc.vocab_size, (B,), generator=gen)]
        sids, lens = list(range(B)), [S] * B
        for _ in range(3):
            ids = [[t] for t in m.forward(ids, sids, lens)]
        graph = next(iter(m._graphs.values()))

        def step():
            graph["meta"][:B].copy_(graph["tokens"].to(torch.int32))
            graph["graph"].replay()
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            step()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.steps
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                step()
            torch.cuda.synchronize()
    rows = {ev.key: [ev.count, float(ev.device_time_total)] for ev in prof.key_averages()
            if ev.device_type == DeviceType.CUDA and ev.device_time_total > 0}
    tot = sum(r[1] for r in rows.values())
    os.makedirs(os.path.join(ROOT, "profile_out"), exist_ok=True)
    path = os.path.join(ROOT, "profile_out", f"shard_launches_tp{args.tp}_b{B}_s{S}{args.tag}.csv")
    with open(path, "w") as f:
        f.write("kernel,launches_per_step,us_per_step,us_per_launch,share\n")
        for k, (c, us) in sorted(rows.items(), key=lambda kv: -kv[1][1]):
            f.write(f"\"{k[:200]}\",{c / 3:.1f},{us / 3:.1f},{us / c:.2f},{us / tot:.4f}\n")
    print(json.dumps({"what": f"one TP={args.tp} shard on one GPU, exchange absent (NOT a TP number)", "model": args.model, "batch": B, "seq_len": S,
                      "graph_replay_ms_per_step": ms, "kernel_busy_us_per_step": tot / 3, "launch_list": os.path.relpath(path, ROOT),
                      "fuse_rotary_store": args.fuse_rotary_store}))
    m._graphs.clear(); torch.cuda.synchronize()
    os._exit(0)


if __name__ == "__main__":
    main()
