"""Kernel-level prefill attention throughput (TFLOP/s) of both generations, Llama-3-8B head geometry, bf16, next to what the
REFERENCE runs at this call site (transformer_layer.py:86-96: third-party flash_attn_varlen_func; here the installed flash_attn
wheel, library code, timed on the same tensors as a baseline - never on the product path).
FLOPs = 4 * nq * D * sum_i L_i (L_i + 1) / 2 (causal).  Prints one JSON line per (implementation, shape)."""
import json, os, sys, types
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import torch
from swiftllm_b200.worker.kernels.prefill_attn import prefill_attention

def run(gen, Bp, L, nq=32, nkv=8, D=128, iters=10):
    os.environ["SLLM_PREFILL_ATTN_GEN"] = gen
    T = Bp * L
    g = torch.Generator(device="cuda"); g.manual_seed(0)
    q = torch.randn(T, nq, D, device="cuda", dtype=torch.bfloat16, generator=g)
    k = torch.randn(T, nkv, D, device="cuda", dtype=torch.bfloat16, generator=g)
    v = torch.randn(T, nkv, D, device="cuda", dtype=torch.bfloat16, generator=g)
    o = torch.empty_like(q)
    st = types.SimpleNamespace(num_prefill_seqs=Bp, prefill_seq_start_locs=torch.arange(Bp, device="cuda", dtype=torch.int32) * L,
                               prefill_seq_lens=torch.full((Bp,), L, device="cuda", dtype=torch.int32), max_prefill_len=L,
                               softmax_scale=D ** -0.5)
    for _ in range(3):
        prefill_attention(q, k, v, o, None, None, st)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        prefill_attention(q, k, v, o, None, None, st)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    flops = 4 * nq * D * Bp * L * (L + 1) / 2
    return {"gen": "gen1-mma.sync" if gen == "1" else "gen2-wgmma", "Bp": Bp, "L": L, "ms": ms, "tflops": flops / (ms * 1e-3) / 1e12}, o

def run_fa2(Bp, L, nq=32, nkv=8, D=128, iters=10):
    """flash_attn_varlen_func exactly as the reference calls it (causal, same cu_seqlens for q and k)."""
    try:
        from flash_attn import flash_attn_varlen_func
        import flash_attn
    except Exception as e:  # noqa: BLE001
        return {"gen": "reference-call-site flash_attn", "error": str(e)[:200]}, None
    T = Bp * L
    g = torch.Generator(device="cuda"); g.manual_seed(0)
    q = torch.randn(T, nq, D, device="cuda", dtype=torch.bfloat16, generator=g)
    k = torch.randn(T, nkv, D, device="cuda", dtype=torch.bfloat16, generator=g)
    v = torch.randn(T, nkv, D, device="cuda", dtype=torch.bfloat16, generator=g)
    cu = torch.arange(Bp + 1, device="cuda", dtype=torch.int32) * L
    f = lambda: flash_attn_varlen_func(q, k, v, cu, cu, L, L, softmax_scale=D ** -0.5, causal=True)
    try:
        for _ in range(3):
            o = f()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            o = f()
        e1.record(); torch.cuda.synchronize()
    except Exception as e:  # noqa: BLE001
        return {"gen": "reference-call-site flash_attn", "error": str(e)[:200]}, None
    ms = e0.elapsed_time(e1) / iters
    flops = 4 * nq * D * Bp * L * (L + 1) / 2
    return {"gen": f"reference-call-site flash_attn {flash_attn.__version__} (library)", "Bp": Bp, "L": L, "ms": ms,
            "tflops": flops / (ms * 1e-3) / 1e12}, o


peak = 1673.7
try:
    peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["bf16_tflops"])
except Exception:  # noqa: BLE001
    pass
for Bp, L in ((8, 4096), (2, 16384), (32, 1024)):
    r1, o1 = run("1", Bp, L)
    r2, o2 = run("0", Bp, L)
    r2["max_abs_diff_vs_gen1"] = float((o1.float() - o2.float()).abs().max())
    r3, o3 = run_fa2(Bp, L)
    if o3 is not None:
        r3["max_abs_diff_vs_gen2"] = float((o3.float() - o2.float()).abs().max())
        r2["speedup_over_reference_flash_attn"] = r3["ms"] / r2["ms"]
    for r in (r1, r2, r3):
        if "tflops" in r:
            r["frac_of_measured_bf16_peak"] = r["tflops"] / peak
        print(json.dumps(r), flush=True)
