"""Restatement of the FP8 numerics (DESIGN.md §8o, csrc/fp8.cu) in torch-CPU.  TEST INFRASTRUCTURE ONLY.

For a row y of the storage dtype:
  1. y is the row the unquantized kernel stores (oracle.kernels' fused_add_rmsnorm / silu_and_mul restate those rows);
  2. s = max(amax(|y|) / 448, 2^-126), fp32 with IEEE division;
  3. q_j = e4m3_rn_satfinite(y_j / s): fp32 IEEE division, round to nearest even, saturation at +-448.  torch's CPU
     `.to(float8_e4m3fn)` rounds to nearest even but does not saturate (464 -> 448, 480 -> NaN), so the values are clamped first;
  4. weights quantized at load use the same formula with rows = output channels;
  5. the GEMM: out[m, n] = round_T(sum_k qa[m, k] qw[n, k] sa[m] sw[n]); here in fp64 (the library accumulates in fp32).
The model restatement (`fp8_model`) runs oracle.model.OracleLlama with every projection an FP8 weight: each projection input is
quantized per row and the GEMM is (5), the rest (norms, rotary, attention, lm_head) exactly as in the 16-bit oracle.
"""
from __future__ import annotations

import contextlib
import copy
import types

import torch

from oracle import kernels as K

E4M3_MAX = 448.0
SCALE_FLOOR = 2.0 ** -126


def quantize_rows(y: torch.Tensor):
    """(q float8_e4m3fn [R, C], s float32 [R]) of the rows of y (16-bit or fp32 values)."""
    y32 = y.to(torch.float32)
    amax = y32.abs().amax(dim=1)
    s = torch.clamp(amax / torch.tensor(E4M3_MAX, dtype=torch.float32), min=SCALE_FLOOR)
    q = (y32 / s[:, None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q, s


def dequantize(q: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """q * s per row, exact in fp64."""
    return q.to(torch.float64) * s.to(torch.float64).reshape(-1, 1)


def add_rmsnorm_quant(x, residual, weight, eps):
    """((q, s) of the fused add+RMSNorm row, the updated residual)."""
    y, r = K.fused_add_rmsnorm(x, residual, weight, eps)
    return quantize_rows(y), r


def silu_and_mul_quant(x):
    F = x.shape[1] // 2
    return quantize_rows(K.silu_and_mul(x)[:, :F])


def linear_fp8_exact(qa, sa, qw, sw, out_dtype):
    """(5) in fp64, one rounding to out_dtype."""
    return (dequantize(qa, sa) @ dequantize(qw, sw).T).to(out_dtype)


class Fp8Weight:
    """An e4m3 projection weight [N, K] with its fp32 per-channel scales."""

    def __init__(self, q, s):
        self.q, self.s = q, s.to(torch.float32).reshape(-1)

    @staticmethod
    def of(w: torch.Tensor) -> "Fp8Weight":
        return Fp8Weight(*quantize_rows(w))

    def rows(self, a, b) -> "Fp8Weight":
        return Fp8Weight(self.q[a:b], self.s[a:b])


PROJECTIONS = ("q_proj", "k_proj", "v_proj", "o_proj", "up_gate_proj", "down_proj")


def fp8_weights(w):
    """A copy of oracle.model.OracleWeights whose projections are quantized per output channel (16-bit -> Fp8Weight)."""
    out = copy.copy(w)
    out.layers = []
    for lw in w.layers:
        nl = copy.copy(lw)
        for n in PROJECTIONS:
            setattr(nl, n, Fp8Weight.of(getattr(lw, n)))
        out.layers.append(nl)
    return out


def _linear(x, w, gemm):
    if isinstance(w, Fp8Weight):
        qa, sa = quantize_rows(x)
        if gemm == "fp64":
            return linear_fp8_exact(qa, sa, w.q, w.s, x.dtype)
        return (dequantize(qa, sa).float() @ dequantize(w.q, w.s).float().T).to(x.dtype)
    return torch.nn.functional.linear(x, w)


@contextlib.contextmanager
def fp8_model(gemm: str = "fp64"):
    """Inside this context oracle.model.OracleLlama evaluates Fp8Weight projections as the FP8 restatement: GEMMs in fp64, or
    with gemm="fp32" on the dequantized operands rounded to fp32 (the CPU tests' stand-in of linear_fp8)."""
    import oracle.model as OM
    saved = OM.F
    OM.F = types.SimpleNamespace(linear=lambda x, w: _linear(x, w, gemm))
    try:
        yield
    finally:
        OM.F = saved


def hf_fp8_tensors(w, F: int, strategy: str = "channel") -> dict:
    """The checkpoint tensors of an FP8 OracleWeights (fp8_weights) in the compressed-tensors layout: `*.weight` e4m3 and
    `*.weight_scale` ([N, 1] per channel, or [1] per tensor when every channel of the projection has the same scale)."""
    d = {"model.embed_tokens.weight": w.wte, "lm_head.weight": w.lm_head, "model.norm.weight": w.final_norm}
    for i, lw in enumerate(w.layers):
        p = f"model.layers.{i}."
        d[p + "input_layernorm.weight"] = lw.attn_norm
        d[p + "post_attention_layernorm.weight"] = lw.ffn_norm
        ug = lw.up_gate_proj
        for key, fw in (("self_attn.q_proj", lw.q_proj), ("self_attn.k_proj", lw.k_proj), ("self_attn.v_proj", lw.v_proj),
                        ("self_attn.o_proj", lw.o_proj), ("mlp.up_proj", ug.rows(0, F)), ("mlp.gate_proj", ug.rows(F, 2 * F)),
                        ("mlp.down_proj", lw.down_proj)):
            d[p + key + ".weight"] = fw.q
            d[p + key + ".weight_scale"] = fw.s[:1].clone() if strategy == "tensor" else fw.s.reshape(-1, 1).clone()
    return d


def compressed_tensors_config(strategy: str = "channel") -> dict:
    """The quantization_config of an llm-compressor FP8-dynamic checkpoint."""
    return {
        "quant_method": "compressed-tensors", "format": "float-quantized", "quantization_status": "compressed",
        "ignore": ["lm_head"], "kv_cache_scheme": None,
        "config_groups": {"group_0": {
            "targets": ["Linear"],
            "weights": {"num_bits": 8, "type": "float", "symmetric": True, "strategy": strategy, "dynamic": False},
            "input_activations": {"num_bits": 8, "type": "float", "symmetric": True, "strategy": "token", "dynamic": True},
            "output_activations": None}},
    }
