"""Multi-LoRA serving: the adapter slot pool, PEFT parsing and validation, tensor-parallel slicing, and the per-step tile list.

An adapter adds s·B·A to four GEMM sites per layer, the fused ones of worker/weight.py:

    site      input             slices (in the order of the fused output)     tensor parallelism
    qkv       normed hidden     q_proj | k_proj | v_proj                       column: A whole, B rows sliced like the base rows
    o         attention output  o_proj                                         row: A sliced by input columns, B whole
    up_gate   normed hidden     up_proj | gate_proj  (up first, as weight.py)  column
    down      silu(gate)·up     down_proj                                      row

Row-parallel ranks add their partial (x_r·A_rᵀ)·Bᵀ into their partial output before the exchange sums the ranks; the map is
linear, so the sum of the partials is the whole delta and no collective is added.  Storage: per layer and site one A pool
[max_loras, S·R, K] and one B pool [max_loras, N, R] (R = max_lora_rank rounded up to 16; a smaller adapter is zero-padded),
a slice-mask table int32 [layers, 4, max_loras] (bit s: slice s targeted) and the scales float32 [max_loras].  Modules an adapter
does not target are skipped by the kernels, not applied as zeros: their outputs keep their bits (-0 + 0 would be +0)."""
from __future__ import annotations

import json
import math
import os
import re
from typing import Optional

import torch

from swiftllm_b200.worker.weight import tp_slice

SITES = ("qkv", "o", "up_gate", "down")
# site -> PEFT modules (self_attn / mlp, name) in slice order
SITE_MODULES = {
    "qkv": (("self_attn", "q_proj"), ("self_attn", "k_proj"), ("self_attn", "v_proj")),
    "o": (("self_attn", "o_proj"),),
    "up_gate": (("mlp", "up_proj"), ("mlp", "gate_proj")),
    "down": (("mlp", "down_proj"),),
}
ROW_PARALLEL = ("o_proj", "down_proj")
RANKS = (8, 16, 32, 64)
TILE_ROWS = 64                          # csrc/lora.cu: rows of one tile
SHORT_TILE_ROWS = 16                    # tile rows of runs up to TILE_ROWS long (one m16 fragment)
_KEY = re.compile(r"^base_model\.model\.model\.layers\.(\d+)\.(self_attn|mlp)\.(q|k|v|o|gate|up|down)_proj\.lora_([AB])\.weight$")


def module_shapes(mc) -> dict:
    """PEFT module name -> (out_features, in_features) of the full (unsliced) base weight."""
    H, D, F = mc.hidden_size, mc.head_dim, mc.ffn_inter_dim
    return {"q_proj": (mc.num_q_heads * D, H), "k_proj": (mc.num_kv_heads * D, H), "v_proj": (mc.num_kv_heads * D, H),
            "o_proj": (H, mc.num_q_heads * D), "up_proj": (F, H), "gate_proj": (F, H), "down_proj": (H, F)}


def read_adapter(adapter) -> tuple:
    """(config dict, {PEFT key: tensor}) from a PEFT adapter directory (adapter_config.json + adapter_model.safetensors or
    adapter_model.bin) or from such a pair."""
    if isinstance(adapter, (tuple, list)) and len(adapter) == 2:
        config, tensors = adapter
        if not isinstance(config, dict) or not isinstance(tensors, dict):
            raise ValueError("an in-memory adapter is a (config dict, {PEFT key: tensor}) pair")
        return config, tensors
    if not isinstance(adapter, (str, os.PathLike)) or not os.path.isdir(adapter):
        raise ValueError(f"adapter must be a PEFT adapter directory or a (config, tensors) pair, got {adapter!r}")
    cfg_path = os.path.join(adapter, "adapter_config.json")
    if not os.path.exists(cfg_path):
        raise ValueError(f"{adapter}: no adapter_config.json")
    with open(cfg_path, "r", encoding="utf-8") as f:
        config = json.load(f)
    st, binf = os.path.join(adapter, "adapter_model.safetensors"), os.path.join(adapter, "adapter_model.bin")
    if os.path.exists(st):
        import safetensors.torch
        tensors = safetensors.torch.load_file(st, device="cpu")
    elif os.path.exists(binf):
        tensors = torch.load(binf, map_location="cpu", weights_only=True)
    else:
        raise ValueError(f"{adapter}: neither adapter_model.safetensors nor adapter_model.bin")
    return config, tensors


def parse_adapter(config: dict, tensors: dict, mc, max_rank: int) -> tuple:
    """Validate a PEFT LoRA adapter against the model: (scale, {(layer, module): (A [r, in], B [out, r])}).  Raises ValueError
    for anything this data plane does not apply exactly (see LlamaModel.load_lora)."""
    if str(config.get("peft_type", "LORA")).upper() != "LORA":
        raise ValueError(f"only LoRA adapters are supported, got peft_type {config.get('peft_type')!r}")
    r = config.get("r", 8)
    if isinstance(r, bool) or not isinstance(r, int) or r < 1:
        raise ValueError(f"adapter rank r must be a positive int, got {r!r}")
    if r > max_rank:
        raise ValueError(f"adapter rank {r} exceeds max_lora_rank {max_rank}")
    alpha = config.get("lora_alpha", 8)
    if isinstance(alpha, bool) or not isinstance(alpha, (int, float)) or not math.isfinite(alpha):
        raise ValueError(f"lora_alpha must be a finite number, got {alpha!r}")
    if config.get("fan_in_fan_out", False):
        raise ValueError("fan_in_fan_out adapters (Conv1D layouts) are not supported")
    if config.get("bias", "none") != "none":
        raise ValueError(f"adapters with bias {config.get('bias')!r} are not supported (bias must be 'none')")
    if config.get("use_dora", False):
        raise ValueError("DoRA adapters are not supported")
    for k in ("rank_pattern", "alpha_pattern", "modules_to_save", "layers_to_transform"):
        v = config.get(k)
        if v not in (None, {}, [], ()):
            raise ValueError(f"adapters with a non-empty {k} are not supported")
    tm = config.get("target_modules") or []
    tm = [tm] if isinstance(tm, str) else list(tm)
    if any(("embed_tokens" in str(t)) or ("lm_head" in str(t)) for t in tm):
        raise ValueError("adapters on embed_tokens or lm_head are not supported")
    shapes = module_shapes(mc)
    found = {}
    for key, t in tensors.items():
        if "embed_tokens" in key or "lm_head" in key:
            raise ValueError(f"adapters on embed_tokens or lm_head are not supported ({key})")
        m = _KEY.match(key)
        if m is None:
            raise ValueError(f"unrecognised adapter tensor {key!r}")
        layer, block, name, ab = int(m.group(1)), m.group(2), m.group(3) + "_proj", m.group(4)
        if (block == "self_attn") != (name in ("q_proj", "k_proj", "v_proj", "o_proj")):
            raise ValueError(f"unrecognised adapter tensor {key!r}")
        if layer >= mc.num_layers:
            raise ValueError(f"{key}: layer {layer} outside the model's {mc.num_layers} layers")
        if not isinstance(t, torch.Tensor) or not t.is_floating_point():
            raise ValueError(f"{key} is not a floating-point tensor")
        out_f, in_f = shapes[name]
        want = (r, in_f) if ab == "A" else (out_f, r)
        if tuple(t.shape) != want:
            raise ValueError(f"{key} has shape {tuple(t.shape)}, expected {want}")
        found.setdefault((layer, name), {})[ab] = t
    for (layer, name), d in found.items():
        if set(d) != {"A", "B"}:
            raise ValueError(f"layer {layer} {name}: lora_A and lora_B must both be present")
    scale = float(alpha) / (math.sqrt(r) if config.get("use_rslora", False) else r)
    return scale, {k: (d["A"], d["B"]) for k, d in found.items()}


def lora_tiles(slots: list, rows: list, pad_to: Optional[int] = None) -> list:
    """Flat int32 triples (first row, rows, slot) of a step: runs of consecutive rows with the same slot, in batch order, cut into
    pieces of at most TILE_ROWS rows, or of SHORT_TILE_ROWS rows for a run no longer than TILE_ROWS (decode rows, short prompts):
    a shrink CTA walks the whole K for its tile, so a short run spread over more tiles finishes sooner.  The cut changes no
    value (a row's result does not depend on its tile).  slots[i] (None: base model) and rows[i] are batch entry i's slot and row count.  pad_to:
    append (0, 0, 0) tiles (skipped by the kernels) up to that many tiles."""
    out, start, run = [], 0, None              # run: [first row, rows, slot]
    for s, n in zip(slots, rows):
        if s is not None and n > 0 and run is not None and run[2] == s and run[0] + run[1] == start:
            run[1] += n
        else:
            if run is not None:
                out.append(run)
            run = [start, n, s] if s is not None and n > 0 else None
        start += n
    if run is not None:
        out.append(run)
    words = []
    for first, n, s in out:
        step = TILE_ROWS if n > TILE_ROWS else SHORT_TILE_ROWS
        for o in range(0, n, step):
            words += [first + o, min(step, n - o), s]
    if pad_to is not None:
        assert len(words) // 3 <= pad_to
        words += [0, 0, 0] * (pad_to - len(words) // 3)
    return words


class LoraPool:
    """Adapter slots of one rank: device pools, slice masks and scales, and the shrink output buffer u."""

    def __init__(self, mc, max_loras: int, max_rank: int, dtype: torch.dtype, device, max_tokens: int, tp_rank: int = 0,
                 tp_size: int = 1):
        if isinstance(max_loras, bool) or not isinstance(max_loras, int) or max_loras < 1:
            raise ValueError(f"max_loras must be a positive int, got {max_loras!r}")
        if max_rank not in RANKS:
            raise ValueError(f"max_lora_rank must be one of {RANKS}, got {max_rank!r}")
        self.mc, self.max_loras, self.max_rank, self.dtype, self.device = mc, max_loras, max_rank, dtype, device
        self.tp_rank, self.tp_size = tp_rank, tp_size
        self.rank = (max_rank + 15) // 16 * 16           # storage rank R
        R, D, tp = self.rank, mc.head_dim, tp_size
        nq, nkv, H, F = mc.num_q_heads * D // tp, mc.num_kv_heads * D // tp, mc.hidden_size, mc.ffn_inter_dim // tp
        # site -> (K, N, slice ends (n1, n2), number of slices), on this rank
        self.dims = {"qkv": (H, nq + 2 * nkv, (nq, nq + nkv), 3), "o": (nq, H, (H, H), 1),
                     "up_gate": (H, 2 * F, (F, 2 * F), 2), "down": (F, H, (H, H), 1)}
        for site, (K, N, ends, _) in self.dims.items():
            # csrc/lora.cu's shape rules, checked here so that a model or tensor-parallel split the kernels cannot serve is
            # refused when the pool is made, not in the middle of a forward
            if K % 32 or N % 8 or ends[0] % 8 or ends[1] % 8:
                raise ValueError(f"LoRA site {site} on this rank has in_features {K} (must be a multiple of 32) and out_features "
                                 f"{N} with slice ends {ends} (must be multiples of 8): the LoRA kernels cannot serve this model "
                                 f"at tp_size {tp}")
        self.dims_ends = [self.dims[s][2] for s in SITES]
        self.a, self.b = [], []
        for _ in range(mc.num_layers):
            self.a.append([torch.zeros((max_loras, S * R, K), dtype=dtype, device=device) for K, _, _, S in self.dims.values()])
            self.b.append([torch.zeros((max_loras, N, R), dtype=dtype, device=device) for _, N, _, _ in self.dims.values()])
        self.slice_mask = torch.zeros((mc.num_layers, len(SITES), max_loras), dtype=torch.int32, device=device)
        self.scales = torch.zeros((max_loras,), dtype=torch.float32, device=device)
        self.u = torch.empty((max(1, max_tokens), 3 * R), dtype=dtype, device=device)
        self.loaded = [False] * max_loras

    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for ts in self.a + self.b for t in ts)

    def ensure_rows(self, num_rows: int):
        """Grow u to num_rows rows (never shrunk).  A CUDA graph captured with an adapter holds a reference to the u it was
        captured with (LlamaModel._capture_decode_graph), so a replaced buffer lives exactly as long as the graphs that read it."""
        if num_rows > self.u.shape[0]:
            self.u = torch.empty((num_rows, self.u.shape[1]), dtype=self.dtype, device=self.device)

    def load(self, slot: int, adapter):
        """Validate everything, then copy: an invalid adapter leaves the slot as it was."""
        if isinstance(slot, bool) or not isinstance(slot, int) or not 0 <= slot < self.max_loras:
            raise ValueError(f"LoRA slot {slot!r} outside [0, {self.max_loras})")
        config, tensors = read_adapter(adapter)
        scale, mods = parse_adapter(config, tensors, self.mc, self.max_rank)
        self.unload(slot)
        R, tp, rk = self.rank, self.tp_size, self.tp_rank
        mask = torch.zeros((self.mc.num_layers, len(SITES)), dtype=torch.int32)
        for si, site in enumerate(SITES):
            K, N, ends, S = self.dims[site]
            starts = (0,) + tuple(ends[:S - 1])
            for sl, (_, name) in enumerate(SITE_MODULES[site]):
                for layer in range(self.mc.num_layers):
                    if (layer, name) not in mods:
                        continue
                    A, B = mods[(layer, name)]
                    r = A.shape[0]
                    if name in ROW_PARALLEL:
                        A = tp_slice(A, 1, rk, tp)
                    else:
                        B = tp_slice(B, 0, rk, tp)
                    self.a[layer][si][slot, sl * R:sl * R + r].copy_(A.to(self.dtype))
                    self.b[layer][si][slot, starts[sl]:starts[sl] + B.shape[0], :r].copy_(B.to(self.dtype))
                    mask[layer, si] |= 1 << sl
        self.slice_mask[:, :, slot].copy_(mask)
        self.scales[slot] = scale
        self.loaded[slot] = True

    def unload(self, slot: int):
        if isinstance(slot, bool) or not isinstance(slot, int) or not 0 <= slot < self.max_loras:
            raise ValueError(f"LoRA slot {slot!r} outside [0, {self.max_loras})")
        self.loaded[slot] = False
        self.slice_mask[:, :, slot] = 0
        self.scales[slot] = 0.0
        for ts in self.a + self.b:
            for t in ts:
                t[slot].zero_()
