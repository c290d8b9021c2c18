"""FP8 (e4m3) weights: which checkpoints are served, and the projections' load-time form (DESIGN.md §8o).

EngineConfig.quantization None follows the checkpoint: a supported FP8 `quantization_config` in config.json turns FP8 on, no
`quantization_config` is the 16-bit engine.  "fp8" also quantizes 16-bit weights (a 16-bit checkpoint, dummy weights, a custom
getter) at load.  FP8 engines run in bfloat16.  Only the qkv, o, up_gate and down projections become e4m3; embeddings, norms, lm_head, activations and the KV
cache stay 16-bit.

Accepted checkpoint formats (anything else raises ValueError naming the field):
  quant_method "compressed-tensors", format "float-quantized": one config group targeting Linear, weights num_bits 8 / type float
      / symmetric / strategy "channel" (weight_scale [N, 1]) or "tensor" (weight_scale [1] or scalar), input activations dynamic
      with strategy "token", `ignore` naming at most lm_head, kv_cache_scheme null;
  quant_method "fp8" (AutoFP8): activation_scheme "dynamic", no weight_block_size, a per-tensor weight_scale.
Static activation scales (`input_scale` tensors) are refused too.

Load-time form of a projection: e4m3 weight [N, K] row-major (the GEMM reads it as w.t(), column-major) and an fp32 scale per
output channel [N] (per-tensor scales are expanded: exact).  Column-parallel slices take weight rows and scales together,
row-parallel slices take weight columns and keep the scales whole.  16-bit weights are quantized one projection at a time on
the device (quant_fp8_rows, rows = output channels, after the tensor-parallel slice), so the device holds at most the FP8 model
and one 16-bit tensor.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

from swiftllm_b200.worker.kernels.fp8 import quant_fp8_rows

QUANTIZATIONS = (None, "fp8")
PROJECTIONS = ("q_proj", "k_proj", "v_proj", "o_proj", "up_proj", "gate_proj", "down_proj")


def _require(cond: bool, msg: str):
    if not cond:
        raise ValueError(f"FP8 checkpoint: {msg}")


def _compressed_tensors(qc: dict) -> str:
    _require(qc.get("format") == "float-quantized",
             f"quantization_config.format {qc.get('format')!r} is not supported (only 'float-quantized')")
    _require(qc.get("kv_cache_scheme") is None, "quantization_config.kv_cache_scheme must be null (the KV cache stays 16-bit)")
    ignore = qc.get("ignore") or []
    _require(all(n == "lm_head" or str(n).endswith(".lm_head") for n in ignore),
             f"quantization_config.ignore may only name lm_head, got {ignore!r}")
    groups = qc.get("config_groups") or {}
    _require(len(groups) == 1, f"quantization_config.config_groups must hold exactly one group, got {len(groups)}")
    (name, g), = groups.items()
    _require(list(g.get("targets") or []) == ["Linear"], f"config_groups.{name}.targets must be ['Linear'], got {g.get('targets')!r}")
    w = g.get("weights") or {}
    for field, want in (("num_bits", 8), ("type", "float"), ("symmetric", True)):
        _require(w.get(field) == want, f"config_groups.{name}.weights.{field} must be {want!r}, got {w.get(field)!r}")
    _require(not w.get("dynamic", False), f"config_groups.{name}.weights.dynamic must be false")
    _require(w.get("block_structure") is None and w.get("group_size") is None,
             f"config_groups.{name}.weights: block-wise and group-wise scales are not supported")
    strategy = w.get("strategy")
    _require(strategy in ("channel", "tensor"),
             f"config_groups.{name}.weights.strategy must be 'channel' or 'tensor', got {strategy!r}")
    a = g.get("input_activations")
    _require(isinstance(a, dict), f"config_groups.{name}.input_activations must be dynamic per-token FP8, got {a!r}")
    for field, want in (("dynamic", True), ("strategy", "token"), ("num_bits", 8), ("type", "float")):
        _require(a.get(field, want) == want, f"config_groups.{name}.input_activations.{field} must be {want!r}, got {a.get(field)!r}")
    _require(g.get("output_activations") is None, f"config_groups.{name}.output_activations must be null")
    return strategy


def _autofp8(qc: dict) -> str:
    _require(qc.get("activation_scheme") == "dynamic",
             f"quantization_config.activation_scheme must be 'dynamic', got {qc.get('activation_scheme')!r}")
    _require(qc.get("weight_block_size") is None,
             f"quantization_config.weight_block_size {qc.get('weight_block_size')!r}: block-wise scales are not supported")
    ignored = qc.get("ignored_layers") or []
    _require(all(n == "lm_head" or str(n).endswith(".lm_head") for n in ignored),
             f"quantization_config.ignored_layers may only name lm_head, got {ignored!r}")
    return "tensor"


def checkpoint_format(raw_config: dict) -> Optional[str]:
    """The weight-scale strategy ("channel" / "tensor") of config.json's FP8 `quantization_config`; None without one.  Raises
    ValueError for any format that is not served."""
    qc = raw_config.get("quantization_config")
    if qc is None:
        return None
    _require(isinstance(qc, dict), "quantization_config must be an object")
    method = qc.get("quant_method")
    if method == "compressed-tensors":
        return _compressed_tensors(qc)
    if method == "fp8":
        return _autofp8(qc)
    raise ValueError(f"quantization_config.quant_method {method!r} is not supported (served: FP8 'compressed-tensors' "
                     f"float-quantized and 'fp8')")


def gemm_shapes(model_config, tp_size: int) -> dict:
    """Per-rank (K, N) of each GEMM."""
    c = model_config
    nq, nkv, D, H, F = c.num_q_heads // tp_size, c.num_kv_heads // tp_size, c.head_dim, c.hidden_size, c.ffn_inter_dim // tp_size
    return {"qkv_proj": (H, (nq + 2 * nkv) * D), "o_proj": (nq * D, H), "up_gate_proj": (H, 2 * F), "down_proj": (F, H)}


def resolve(quantization, model_config, tp_size: int, max_loras: int, dtype: torch.dtype) -> bool:
    """Whether the engine runs FP8 projections.  Raises ValueError for an unknown `quantization`, an unsupported checkpoint
    format, LoRA together with FP8, a float16 engine (torch 2.11's row-wise FP8 GEMM returns wrong float16 outputs on sm_90; its
    bfloat16 outputs are correct), and per-rank GEMM dimensions the FP8 GEMM cannot take (K and N multiples of 16)."""
    if quantization not in QUANTIZATIONS:
        raise ValueError(f"quantization must be one of {QUANTIZATIONS}, got {quantization!r}")
    fp8 = checkpoint_format(getattr(model_config, "raw", {})) is not None or quantization == "fp8"
    if not fp8:
        return False
    if max_loras:
        raise ValueError("LoRA adapters (max_loras > 0) are not supported on an FP8 engine")
    if dtype != torch.bfloat16:
        raise ValueError(f"FP8 weights need dtype bfloat16 (EngineConfig.dtype / --dtype bfloat16), got {dtype}: the library's "
                         f"row-wise FP8 GEMM does not produce correct float16 outputs (scripts/fp8_gemm_dtype_check.py)")
    for name, (K, N) in gemm_shapes(model_config, tp_size).items():
        if K % 16 or N % 16:
            raise ValueError(f"FP8 weights: {name} has per-rank K = {K}, N = {N} at tp_size {tp_size}; both must be multiples of 16")
    return True


def check_no_static_activation_scales(getter: Callable):
    """Refuse static activation scales: the engine quantizes activations per token at run time."""
    keys = getattr(getter, "keys", None)
    bad = sorted(k for k in (keys or ()) if k.endswith(".input_scale"))
    if bad:
        raise ValueError(f"FP8 checkpoint: static activation scales are not supported ({bad[0]} present)")


def channel_scales(scale: torch.Tensor, N: int, key: str) -> torch.Tensor:
    """A checkpoint's weight_scale (per tensor: [1] or scalar; per channel: [N, 1] or [N]) as fp32 [N]; refuses shapes that are
    neither and scales that are not finite and positive."""
    s = scale.to(torch.float32)
    if s.numel() == 1:
        s = s.reshape(1).expand(N)
    elif tuple(s.shape) in ((N, 1), (N,)):
        s = s.reshape(N)
    else:
        raise ValueError(f"FP8 checkpoint: {key}_scale has shape {tuple(scale.shape)}; expected [1], [] or [{N}, 1]")
    bad = ~(torch.isfinite(s) & (s > 0))
    if bool(bad.any()):
        raise ValueError(f"FP8 checkpoint: {key}_scale holds {float(s[bad][0])}; scales must be finite and positive")
    return s.contiguous()


def load_projection(getter: Callable, key: str, shape: tuple, axis: int, tp_rank: int, tp_size: int, dtype: torch.dtype,
                    device):
    """(e4m3 weight [N / tp or N, K or K / tp], fp32 scales [N / tp or N]) of one projection on `device`."""
    from swiftllm_b200.worker.weight import tp_slice
    w = getter(key, shape, dtype)
    assert isinstance(w, torch.Tensor), f"Weight {key} is not a tensor"
    assert tuple(w.shape) == tuple(shape), f"Shape of weight {key} does not match"
    if w.dtype == torch.float8_e4m3fn:
        s = channel_scales(getter(key + "_scale", (shape[0], 1), torch.float32), shape[0], key)
        s = tp_slice(s, 0 if axis == 0 else None, tp_rank, tp_size)
        w = tp_slice(w, axis, tp_rank, tp_size)
        return w.to(device=device).contiguous(), s.to(device=device).contiguous()
    if w.dtype not in (torch.float16, torch.bfloat16, torch.float32):
        raise ValueError(f"FP8 weights: {key} has dtype {w.dtype}; expected float8_e4m3fn or a 16/32-bit float")
    w = tp_slice(w, axis, tp_rank, tp_size).to(device=device, dtype=dtype).contiguous()
    q, s = quant_fp8_rows(w)
    return q, s.view(-1)


def cat_rows(ts) -> torch.Tensor:
    """Row concatenation of e4m3 tensors (through their bytes)."""
    return torch.cat([t.view(torch.uint8) for t in ts], dim=0).view(torch.float8_e4m3fn)

