"""Weights of the data plane.  Attribute names, HF tensor keys and the `up_gate_proj = cat(up, gate)` fusion are
the reference's (swiftllm/worker/weight.py:56-177, :133); loaders cover the same sources (safetensors single /
sharded, pytorch_model.bin, dummy uniform(-1e-3, 1e-3)) plus seeded synthetic weights, and every projection is
sliced for tensor parallelism at load time:

    rank r of N holds   q_proj rows of q heads [r*nq/N, (r+1)*nq/N)        (column-parallel)
                        k_proj / v_proj rows of kv heads [r*nkv/N, ...)     (column-parallel)
                        up / gate rows [r*F/N, (r+1)*F/N), re-fused as [up_r ; gate_r]
                        o_proj / down_proj input columns of the same slices (row-parallel, all-reduced)
    norms and the embedding are replicated; lm_head is replicated, or (shard_lm_head) split by vocabulary rows.
"""
from __future__ import annotations

import json
import os
from typing import Callable, Optional

import torch

from swiftllm_b200.model_config import LlamaModelConfig
from swiftllm_b200.worker import fp8 as fp8_weights

# (attribute, HF key template, shape fn, TP split axis: 0 rows, 1 cols, None replicated)
_LAYER_ITEMS = [
    ("attn_norm", "model.layers.{i}.input_layernorm.weight", lambda c: (c.hidden_size,), None),
    ("q_proj", "model.layers.{i}.self_attn.q_proj.weight", lambda c: (c.hidden_size, c.hidden_size), 0),
    ("k_proj", "model.layers.{i}.self_attn.k_proj.weight", lambda c: (c.num_kv_heads * c.head_dim, c.hidden_size), 0),
    ("v_proj", "model.layers.{i}.self_attn.v_proj.weight", lambda c: (c.num_kv_heads * c.head_dim, c.hidden_size), 0),
    ("o_proj", "model.layers.{i}.self_attn.o_proj.weight", lambda c: (c.hidden_size, c.hidden_size), 1),
    ("ffn_norm", "model.layers.{i}.post_attention_layernorm.weight", lambda c: (c.hidden_size,), None),
    ("up_proj", "model.layers.{i}.mlp.up_proj.weight", lambda c: (c.ffn_inter_dim, c.hidden_size), 0),
    ("gate_proj", "model.layers.{i}.mlp.gate_proj.weight", lambda c: (c.ffn_inter_dim, c.hidden_size), 0),
    ("down_proj", "model.layers.{i}.mlp.down_proj.weight", lambda c: (c.hidden_size, c.ffn_inter_dim), 1),
]


def tp_slice(t: torch.Tensor, axis: Optional[int], tp_rank: int, tp_size: int) -> torch.Tensor:
    if axis is None or tp_size == 1:
        return t
    n = t.shape[axis]
    assert n % tp_size == 0, f"dimension {n} not divisible by tp_size {tp_size}"
    step = n // tp_size
    return t.narrow(axis, tp_rank * step, step)


class LlamaTransformerLayerWeight:
    def __init__(self, layer_id: int, model_config: LlamaModelConfig, dtype: torch.dtype):
        self.layer_id = layer_id
        self.model_config = model_config
        self.dtype = dtype
        self.fp8 = False

    def load_weights(self, getter: Callable, tp_rank: int, tp_size: int, device, fp8: bool = False):
        """fp8: every projection becomes an e4m3 weight plus an fp32 per-output-channel `<name>_scale` (worker/fp8.py)."""
        if fp8:
            return self._load_fp8(getter, tp_rank, tp_size, device)
        for attr, key, shape_fn, axis in _LAYER_ITEMS:
            key = key.format(i=self.layer_id)
            shape = shape_fn(self.model_config)
            w = getter(key, shape, self.dtype)
            if isinstance(w, torch.Tensor) and w.dtype == torch.float8_e4m3fn:
                raise ValueError(f"{key} is float8_e4m3fn: serve FP8 checkpoints with their quantization_config in config.json "
                                 f"or EngineConfig.quantization='fp8'")
            assert isinstance(w, torch.Tensor), f"Weight {key} is not a tensor"
            assert tuple(w.shape) == tuple(shape), f"Shape of weight {key} does not match"
            w = tp_slice(w, axis, tp_rank, tp_size).to(device=device, dtype=self.dtype).contiguous()
            setattr(self, attr, w)
        # up first, gate second (weight.py:133; silu_and_mul reads gate from the second half)
        self.up_gate_proj = torch.cat((self.up_proj, self.gate_proj), dim=0).contiguous()
        del self.up_proj, self.gate_proj
        # q | k | v fused into one GEMM operand (the fusion the reference left commented out, weight.py:131-132);
        # q_proj / k_proj / v_proj stay available as row views of it (no extra memory)
        nq_rows, nkv_rows = self.q_proj.shape[0], self.k_proj.shape[0]
        self.qkv_proj = torch.cat((self.q_proj, self.k_proj, self.v_proj), dim=0).contiguous()
        self.q_proj = self.qkv_proj[:nq_rows]
        self.k_proj = self.qkv_proj[nq_rows:nq_rows + nkv_rows]
        self.v_proj = self.qkv_proj[nq_rows + nkv_rows:]

    def _load_fp8(self, getter: Callable, tp_rank: int, tp_size: int, device):
        self.fp8 = True
        for attr, key, shape_fn, axis in _LAYER_ITEMS:
            key = key.format(i=self.layer_id)
            shape = shape_fn(self.model_config)
            if attr in fp8_weights.PROJECTIONS:
                w, s = fp8_weights.load_projection(getter, key, shape, axis, tp_rank, tp_size, self.dtype, device)
                setattr(self, attr + "_scale", s)
            else:
                w = getter(key, shape, self.dtype)
                assert isinstance(w, torch.Tensor), f"Weight {key} is not a tensor"
                assert tuple(w.shape) == tuple(shape), f"Shape of weight {key} does not match"
                w = tp_slice(w, axis, tp_rank, tp_size).to(device=device, dtype=self.dtype).contiguous()
            setattr(self, attr, w)
        # the 16-bit path's fusions, weights and scales concatenated in the same order
        self.up_gate_proj = fp8_weights.cat_rows((self.up_proj, self.gate_proj))
        self.up_gate_proj_scale = torch.cat((self.up_proj_scale, self.gate_proj_scale))
        self.qkv_proj = fp8_weights.cat_rows((self.q_proj, self.k_proj, self.v_proj))
        self.qkv_proj_scale = torch.cat((self.q_proj_scale, self.k_proj_scale, self.v_proj_scale))
        for n in ("up_proj", "gate_proj", "q_proj", "k_proj", "v_proj"):
            delattr(self, n)
            delattr(self, n + "_scale")


class LlamaWeight:
    def __init__(self, model_config: LlamaModelConfig, dtype: torch.dtype, model_version: str = "llama"):
        self.model_config = model_config
        self.dtype = dtype
        self.model_version = model_version
        self.layers = [LlamaTransformerLayerWeight(i, model_config, dtype) for i in range(model_config.num_layers)]

    def load_weights(self, getter: Callable, tp_rank: int = 0, tp_size: int = 1, device="cuda", shard_lm_head: bool = False,
                     fp8: bool = False):
        c = self.model_config
        if fp8:
            fp8_weights.check_no_static_activation_scales(getter)
        vs = (c.vocab_size, c.hidden_size)
        self.wte = getter("model.embed_tokens.weight", vs, self.dtype).to(device=device, dtype=self.dtype)
        self.lm_head_sharded = bool(shard_lm_head) and tp_size > 1
        if self.lm_head_sharded:
            assert c.vocab_size % tp_size == 0, f"shard_lm_head: vocab_size {c.vocab_size} not divisible by tp_size {tp_size}"
        if self.model_version == "llama3.2":      # tied embeddings (weight.py:157-163); a row slice of wte is a view
            self.lm_head = tp_slice(self.wte, 0, tp_rank, tp_size) if self.lm_head_sharded else self.wte
        else:
            lm_head = getter("lm_head.weight", vs, self.dtype)
            if self.lm_head_sharded:
                lm_head = tp_slice(lm_head, 0, tp_rank, tp_size)
            self.lm_head = lm_head.to(device=device, dtype=self.dtype).contiguous()
        self.final_norm = getter("model.norm.weight", (c.hidden_size,), self.dtype).to(device=device, dtype=self.dtype)
        for layer in self.layers:
            layer.load_weights(getter, tp_rank, tp_size, device, fp8=fp8)


# ---------------------------------------------------------------- getters
def dummy_getter(device="cuda"):
    """weight.py:215-218: uniform(-1e-3, 1e-3), unseeded ("mainly for profiling")."""
    def get(key, shape, dtype):
        return torch.empty(shape, dtype=dtype, device=device).uniform_(-0.001, 0.001)
    return get


def synthetic_getter(seed: int = 0, std: float = 0.02, device="cuda"):
    """Seeded synthetic weights of realistic scale (SURVEY.md §8d): N(0, std) projections, 1 + N(0, std) norms.
    Deterministic per tensor key, so every TP rank generates the same full tensor before slicing."""
    import zlib

    def get(key, shape, dtype):
        g = torch.Generator(device=device)
        g.manual_seed((seed * 1000003 + zlib.crc32(key.encode())) & 0x7FFFFFFF)
        t = torch.randn(shape, generator=g, device=device, dtype=torch.float32) * std
        if key.endswith("norm.weight") or key.endswith("layernorm.weight"):
            t += 1.0
        return t.to(dtype)
    return get


def dict_getter(tensors: dict):
    def get(key, shape, dtype):
        return tensors[key]
    get.keys = tensors.keys()
    return get


def checkpoint_getter(model_path: str, device="cuda"):
    """safetensors (single file or model.safetensors.index.json) or pytorch_model.bin(.index.json), as in
    weight.py:220-268."""
    st_files = [n for n in os.listdir(model_path) if n.endswith(".safetensors")]
    if st_files:
        import safetensors
        index_path = os.path.join(model_path, "model.safetensors.index.json")
        if os.path.exists(index_path):
            with open(index_path, "r", encoding="utf-8") as f:
                index = json.load(f)["weight_map"]
        else:
            assert len(st_files) == 1, "model.safetensors.index.json not found, but there are multiple .safetensors files"
            index = None

        def get(key, shape, dtype):
            fname = index[key] if index is not None else st_files[0]
            with safetensors.safe_open(os.path.join(model_path, fname), framework="pt", device=str(device)) as f:
                return f.get_tensor(key)
        if index is not None:
            get.keys = index.keys()
        else:
            with safetensors.safe_open(os.path.join(model_path, st_files[0]), framework="pt", device="cpu") as f:
                get.keys = list(f.keys())
        return get

    index_path = os.path.join(model_path, "pytorch_model.bin.index.json")
    index = None
    if os.path.exists(index_path):
        with open(index_path, "r", encoding="utf-8") as f:
            index = json.load(f)["weight_map"]
    opened = {}

    def get(key, shape, dtype):
        fname = index[key] if index is not None else "pytorch_model.bin"
        path = os.path.join(model_path, fname)
        if path not in opened:
            opened[path] = torch.load(path, map_location="cpu", mmap=True)
        return opened[path][key]
    return get


def detect_model_version(model_path: Optional[str], model_config: LlamaModelConfig) -> str:
    # weight.py:205-211: "llama3.2" (tied lm_head) iff rope_scaling is a dict
    return "llama3.2" if isinstance(model_config.rope_scaling, dict) else "llama"


def load_weights(model_config: LlamaModelConfig, dtype: torch.dtype, model_path: Optional[str], use_dummy: bool = False,
                 model_version: str = "auto", getter: Optional[Callable] = None, tp_rank: int = 0, tp_size: int = 1,
                 device="cuda", shard_lm_head: bool = False, fp8: bool = False) -> LlamaWeight:
    if model_version == "auto":
        model_version = detect_model_version(model_path, model_config)
    if getter is None:
        getter = dummy_getter(device) if use_dummy else checkpoint_getter(model_path, device)
    weight = LlamaWeight(model_config, dtype, model_version)
    weight.load_weights(getter, tp_rank, tp_size, device, shard_lm_head=shard_lm_head, fp8=fp8)
    return weight
