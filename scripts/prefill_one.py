"""A few launches of the wgmma prefill attention kernel at 8 x 4096 tokens (Llama-3-8B heads, bf16) for an ncu capture:
    ncu --set full --import-source on -k regex:prefill_attn_tc_kernel --launch-skip 2 --launch-count 1 -o profile_out/prefill_tc python scripts/prefill_one.py"""
import os, sys, types
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import torch
from swiftllm_b200.worker.kernels.prefill_attn import prefill_attention
os.environ["SLLM_PREFILL_ATTN_GEN"] = "0"
Bp, L, nq, nkv, D = int(os.environ.get("PF_B", 8)), int(os.environ.get("PF_L", 4096)), 32, 8, 128
T = Bp * L
g = torch.Generator(device="cuda"); g.manual_seed(0)
q = torch.randn(T, nq, D, device="cuda", dtype=torch.bfloat16, generator=g)
k = torch.randn(T, nkv, D, device="cuda", dtype=torch.bfloat16, generator=g)
v = torch.randn(T, nkv, D, device="cuda", dtype=torch.bfloat16, generator=g)
o = torch.empty_like(q)
st = types.SimpleNamespace(num_prefill_seqs=Bp, prefill_seq_start_locs=torch.arange(Bp, device="cuda", dtype=torch.int32) * L,
                           prefill_seq_lens=torch.full((Bp,), L, device="cuda", dtype=torch.int32), max_prefill_len=L, softmax_scale=D ** -0.5)
for _ in range(4):
    prefill_attention(q, k, v, o, None, None, st)
torch.cuda.synchronize()
print("ok", float(o.float().abs().mean()))
