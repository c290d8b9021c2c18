#!/usr/bin/env python
"""Tensor-parallel A/B sweep in ONE process group (multi-GPU box time is charged per GPU, so every variant shares one torchrun
start-up and one NCCL init):

    torchrun --nproc-per-node N scripts/tp_sweep.py --gpus N [--batch 256] [--seqlen 4096] [--variants a,b,...] [--profile best]

For every variant (exchange kernel x lm_head sharding x rotary/store fusion) it builds the model shard, fills the KV cache,
warms up, and times K CUDA-graph replays of the decode step (device-resident token feedback, barrier + synchronize on both
sides, max over ranks) and K steps through the public API (host lists in / ints out).  One JSON line per variant on stdout
(rank 0).  `--profile NAME` additionally records a per-kernel launch list of that variant on rank 0 with the torch profiler
(CUPTI; ncu cannot be used on a multi-rank command) and writes it to profile_out/tp_sweep_launches_n<N>_<NAME>.csv.
This is a development tool: the contract numbers come from bench.py."""
import argparse
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

VARIANTS = {
    # name: (fused_allreduce, shard_lm_head, fuse_rotary_store)
    "nccl": (False, False, False),
    "one_shot": (True, False, False),
    "two_shot": ("two_shot", False, False),
    "nvls": ("two_shot_nvls", False, False),
    "ll": ("ll", False, False),
    "ll_nvls": ("ll_nvls", False, False),
    "nccl+lmhead+rs": (False, True, True),
    "one_shot+lmhead+rs": (True, True, True),
    "two_shot+lmhead+rs": ("two_shot", True, True),
    "nvls+lmhead+rs": ("two_shot_nvls", True, True),
    "ll+lmhead+rs": ("ll", True, True),
    "ll_nvls+lmhead+rs": ("ll_nvls", True, True),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, required=True)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seqlen", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--model", default="llama3-8b", choices=["llama3-8b", "llama3-70b"])
    ap.add_argument("--variants", default=",".join(VARIANTS))
    ap.add_argument("--profile", default="", help="variant name(s), comma separated, to record a kernel launch list for (rank 0)")
    args = ap.parse_args()

    import torch.distributed as dist
    import swiftllm_b200
    from swiftllm_b200.model_config import LLAMA3_8B, LLAMA3_70B
    from swiftllm_b200.worker.weight import synthetic_getter

    n = args.gpus
    rank, local = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
    assert int(os.environ.get("WORLD_SIZE", "1")) == n
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl", device_id=dev)
    mc = swiftllm_b200.LlamaModelConfig(dict(LLAMA3_8B if args.model == "llama3-8b" else LLAMA3_70B))
    B, S, bs = args.batch, args.seqlen, 16
    bps = (S + bs - 1) // bs
    num_blocks = B * bps + 64
    gen = torch.Generator().manual_seed(7)
    ids0 = [[int(t)] for t in torch.randint(0, mc.vocab_size, (B,), generator=gen)]
    sids, lens = list(range(B)), [S] * B
    os.makedirs(os.path.join(ROOT, "profile_out"), exist_ok=True)

    def barrier():
        dist.barrier(); torch.cuda.synchronize()

    def timed(fn, steps):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        barrier()
        t = torch.tensor([e0.elapsed_time(e1)], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item()) / steps

    for name in [v for v in args.variants.split(",") if v]:
        fused, shard, frs = VARIANTS[name]
        line = {"variant": name, "n_gpus": n, "batch": B, "seq_len": S, "model": args.model}
        try:
            with torch.inference_mode():
                ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=bs, gpu_mem_utilization=0.97, num_cpu_blocks=0,
                                                max_seqs_in_block_table=B, max_blocks_per_seq=bps + 8, max_batch_size=B,
                                                max_tokens_in_batch=max(B, 4096), dtype="bfloat16", tp_size=n, tp_rank=rank,
                                                use_cuda_graph=True, fused_allreduce=fused, shard_lm_head=shard, fuse_rotary_store=frs)
                model = swiftllm_b200.LlamaModel(ec, mc)
                model.load_weights(synthetic_getter(seed=0, std=0.02, device=dev))
                model.init_kvcache_and_swap(num_blocks)
                g = torch.Generator(device=dev); g.manual_seed(1234 + rank)
                chunk = max(1, num_blocks // 16)
                for s in range(0, num_blocks, chunk):
                    model.k_cache[s:s + chunk].normal_(generator=g); model.v_cache[s:s + chunk].normal_(generator=g)
                state = {"ids": ids0}

                def step_e2e():
                    state["ids"] = [[t] for t in model.forward(state["ids"], sids, lens)]
                for _ in range(args.warmup):
                    step_e2e()
                ms_e2e = timed(step_e2e, args.steps)
                graph = next(iter(model._graphs.values()))

                def step_resident():
                    graph["meta"][:B].copy_(graph["tokens"].to(torch.int32))
                    graph["graph"].replay()
                for _ in range(args.warmup):
                    step_resident()
                ms = timed(step_resident, args.steps)
                line.update({"ms_per_step": ms, "tokens_per_s": B / (ms * 1e-3), "e2e_ms_per_step": ms_e2e,
                             "e2e_tokens_per_s": B / (ms_e2e * 1e-3),
                             "exchange": "nccl" if model.comm is None else (("ll_nvls" if model.comm.nvls else "ll") if model.comm.ll else "nvls" if model.comm.nvls
                                                                            else "two_shot" if model.comm.two_shot else "one_shot"),
                             "lm_head_sharded": bool(shard), "fuse_rotary_store": bool(frs)})
                if name in args.profile.split(","):
                    # every rank must replay (the exchange is collective); only rank 0 records
                    from torch.profiler import ProfilerActivity, profile
                    barrier()
                    if rank == 0:
                        with profile(activities=[ProfilerActivity.CUDA]) as prof:
                            for _ in range(3):
                                step_resident()
                            torch.cuda.synchronize()
                        from torch.autograd import DeviceType
                        rows = {}
                        for ev in prof.key_averages():
                            if ev.device_type == DeviceType.CUDA and ev.device_time_total > 0:
                                rows[ev.key] = [ev.count, float(ev.device_time_total)]
                        tot = sum(r[1] for r in rows.values())
                        path = os.path.join(ROOT, "profile_out", f"tp_sweep_launches_n{n}_{name.replace('+', '_')}_b{B}.csv")
                        with open(path, "w") as f:
                            f.write("kernel,launches_per_step,us_per_step,share\n")
                            for k, (c, us) in sorted(rows.items(), key=lambda kv: -kv[1][1]):
                                f.write(f"\"{k[:160]}\",{c / 3:.1f},{us / 3:.1f},{us / tot:.4f}\n")
                        line["launch_list"] = os.path.relpath(path, ROOT)
                        line["profiled_gpu_us_per_step"] = tot / 3
                    else:
                        for _ in range(3):
                            step_resident()
                        torch.cuda.synchronize()
                    barrier()
                model._graphs.clear()
                torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
                del graph, model
        except Exception as e:  # noqa: BLE001
            line["error"] = f"{type(e).__name__}: {str(e)[:300]}"
        gc.collect(); torch.cuda.empty_cache()
        ok = torch.tensor([0 if "error" in line else 1], device=dev)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN)
        if int(ok.item()) == 0 and "error" not in line:
            line["error"] = "failed on another rank"
        if rank == 0:
            print(json.dumps(line), flush=True)
    torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
    sys.stdout.flush(); sys.stderr.flush()
    os._exit(0)


if __name__ == "__main__":
    main()
