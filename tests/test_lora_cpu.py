"""CPU: multi-LoRA.  The numerics contract (tests/lora_oracle.py) on hand-made rows, PEFT parsing and the slot pool (with its
tensor-parallel slices), every ValueError, the C ABI's argument checks, and the product's host path with a torch stand-in of the
kernels: adapted logits against a model with merged weights, tile lists, unchanged staging without adapters, graph keys,
speculative rows, and tensor parallelism over gloo."""
import copy
import json
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import lora_oracle as LO

MODS = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")


def _bits(t):
    return t.view(torch.int16)


def make_adapter(cfg, r, seed, modules=MODS, layers=None, alpha=None, std=0.08, **extra):
    """A PEFT LoRA adapter in memory: (config, {key: fp32 tensor}).  B is random too (PEFT initialises it to zero)."""
    H, nq, nkv, F = cfg["hidden_size"], cfg["num_attention_heads"], cfg["num_key_value_heads"], cfg["intermediate_size"]
    D = H // nq
    shapes = {"q_proj": (nq * D, H), "k_proj": (nkv * D, H), "v_proj": (nkv * D, H), "o_proj": (H, nq * D),
              "up_proj": (F, H), "gate_proj": (F, H), "down_proj": (H, F)}
    g = torch.Generator().manual_seed(seed)
    tensors = {}
    for i in range(cfg["num_hidden_layers"]) if layers is None else layers:
        for m in modules:
            blk = "self_attn" if m in ("q_proj", "k_proj", "v_proj", "o_proj") else "mlp"
            out_f, in_f = shapes[m]
            p = f"base_model.model.model.layers.{i}.{blk}.{m}."
            tensors[p + "lora_A.weight"] = torch.randn((r, in_f), generator=g) * std
            tensors[p + "lora_B.weight"] = torch.randn((out_f, r), generator=g) * std
    config = dict(peft_type="LORA", r=r, lora_alpha=alpha if alpha is not None else 2 * r, target_modules=list(modules),
                  bias="none", fan_in_fan_out=False, use_rslora=False, rank_pattern={}, alpha_pattern={}, modules_to_save=None,
                  layers_to_transform=None, **extra)
    return config, tensors


# ---------------------------------------------------------------- the restatement on hand-made rows
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_restatement_slices_scale_and_untouched_elements(dtype):
    R = 16
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(4, 64, generator=g)).to(dtype)
    A = torch.zeros(3 * R, 64, dtype=dtype)
    A[:2] = torch.randn(2, 64, generator=g).to(dtype) * 0.1         # rank 2 in slice 0, slice 1 empty rows, slice 2 rank 1
    A[2 * R] = torch.randn(64, generator=g).to(dtype) * 0.1
    B = torch.zeros(24, R, dtype=dtype)
    B[:8, :2] = torch.randn(8, 2, generator=g).to(dtype)
    B[16:, :1] = torch.randn(8, 1, generator=g).to(dtype)
    y = torch.randn(4, 24, generator=g).to(dtype)
    y[2, 9] = -0.0
    y[2, 0] = -0.0
    out, u = LO.apply(x, y, [0, None, 0, 0], {0: (A, B, 0.5)}, R, ends=(8, 16), site_mask={0: 0b101})
    assert torch.equal(_bits(out[1]), _bits(y[1]))                   # row without a slot
    assert torch.equal(_bits(out[:, 8:16]), _bits(y[:, 8:16]))       # untargeted slice: -0 at (2, 9) kept
    assert _bits(out[2, 9:10]).item() == _bits(torch.tensor([-0.0], dtype=dtype)).item()
    for t in (0, 2, 3):
        for n in list(range(8)) + list(range(16, 24)):
            sl = 0 if n < 8 else 2
            uu = (x[t].double() @ A[sl * R:(sl + 1) * R].double().t()).to(dtype)
            acc = np.float32((uu.double() * B[n].double()).sum().item())
            want = torch.tensor(float(np.float32(np.float32(y[t, n].float().item()) + np.float32(0.5) * acc))).to(dtype)
            assert _bits(out[t, n:n + 1]) == _bits(want.reshape(1)), (t, n)


def test_scale_and_rslora():
    from swiftllm_b200.model_config import LlamaModelConfig
    from swiftllm_b200.worker.lora import parse_adapter
    from test_host_path_cpu import CFG
    mc = LlamaModelConfig(CFG)
    cfg, ten = make_adapter(CFG, 16, 1, alpha=32)
    assert parse_adapter(cfg, ten, mc, 16)[0] == 2.0
    assert parse_adapter(dict(cfg, use_rslora=True), ten, mc, 16)[0] == 8.0
    cfg8, ten8 = make_adapter(CFG, 8, 1, alpha=16)
    assert parse_adapter(cfg8, ten8, mc, 64)[0] == 2.0


def test_expand_of_zero_delta_keeps_negative_zero_only_when_skipped():
    """Why absent modules are skipped: applying a zero delta rounds -0 + 0 to +0."""
    y = torch.tensor([[-0.0, 1.0]], dtype=torch.float16)
    u = torch.zeros((1, 16), dtype=torch.float16)
    B = torch.zeros((2, 16), dtype=torch.float16)
    applied = LO.expand_exact(y, u, B, 1.0, (2, 2), 1, 16)
    assert _bits(applied)[0, 0].item() == 0 and _bits(y)[0, 0].item() != 0
    assert torch.equal(_bits(LO.expand_exact(y, u, B, 1.0, (2, 2), 0, 16)), _bits(y))


# ---------------------------------------------------------------- PEFT parsing, the pool and its TP slices
def _write_dir(tmp_path, config, tensors, fmt="safetensors"):
    d = tmp_path / f"adapter_{fmt}"
    d.mkdir()
    (d / "adapter_config.json").write_text(json.dumps(config))
    if fmt == "safetensors":
        import safetensors.torch
        safetensors.torch.save_file({k: v.contiguous() for k, v in tensors.items()}, str(d / "adapter_model.safetensors"))
    else:
        torch.save(tensors, str(d / "adapter_model.bin"))
    return str(d)


@pytest.mark.parametrize("fmt", ["safetensors", "bin"])
@pytest.mark.parametrize("world", [1, 2, 4])
def test_pool_holds_the_adapter_at_its_offsets_and_tp_slices(tmp_path, fmt, world):
    from swiftllm_b200.model_config import LlamaModelConfig
    from swiftllm_b200.worker.lora import LoraPool, SITES, read_adapter
    from test_host_path_cpu import CFG
    cfg = dict(CFG, num_attention_heads=8, num_key_value_heads=4, hidden_size=128, intermediate_size=256)
    mc = LlamaModelConfig(cfg)
    H, D, F = 128, 16, 256
    config, tensors = make_adapter(cfg, 12, 3, modules=("q_proj", "v_proj", "o_proj", "up_proj", "gate_proj", "down_proj"),
                                   layers=[1], alpha=24)
    path = _write_dir(tmp_path, config, tensors, fmt)
    c2, t2 = read_adapter(path)
    assert c2["r"] == 12 and set(t2) == set(tensors)
    for rank in range(world):
        pool = LoraPool(mc, 3, 16, torch.float16, "cpu", 8, tp_rank=rank, tp_size=world)
        pool.load(2, path)
        R = pool.rank
        assert R == 16 and pool.loaded == [False, False, True] and pool.scales[2].item() == 2.0
        key = lambda m, ab: tensors[f"base_model.model.model.layers.1.{'self_attn' if m[0] in 'qkvo' else 'mlp'}.{m}.lora_{ab}.weight"]
        h = lambda t: t.to(torch.float16)
        nq, nkv, Fl = 8 * D // world, 4 * D // world, F // world
        # layer 0 untouched, every site's mask 0
        assert pool.slice_mask[0, :, 2].tolist() == [0, 0, 0, 0]
        assert pool.slice_mask[1, :, 2].tolist() == [0b101, 1, 0b11, 1]        # k_proj absent: slice 1 of qkv skipped
        a, b = pool.a[1], pool.b[1]
        # qkv: A whole, B rows sliced by heads
        assert torch.equal(a[0][2, :12], h(key("q_proj", "A"))) and not a[0][2, 12:2 * R + 0].any()
        assert torch.equal(a[0][2, 2 * R:2 * R + 12], h(key("v_proj", "A"))) and not a[0][2, 2 * R + 12:].any()
        assert torch.equal(b[0][2, :nq, :12], h(key("q_proj", "B")[rank * nq:(rank + 1) * nq]))
        assert not b[0][2, nq:nq + nkv].any()
        assert torch.equal(b[0][2, nq + nkv:, :12], h(key("v_proj", "B")[rank * nkv:(rank + 1) * nkv]))
        assert not b[0][2, :, 12:].any()
        # o / down: A sliced by input columns, B whole
        assert torch.equal(a[1][2, :12], h(key("o_proj", "A")[:, rank * (H // world):(rank + 1) * (H // world)]))
        assert torch.equal(b[1][2, :, :12], h(key("o_proj", "B")))
        assert torch.equal(a[3][2, :12], h(key("down_proj", "A")[:, rank * Fl:(rank + 1) * Fl]))
        assert torch.equal(b[3][2, :, :12], h(key("down_proj", "B")))
        # up_gate: up first, then gate
        assert torch.equal(a[2][2, :12], h(key("up_proj", "A"))) and torch.equal(a[2][2, R:R + 12], h(key("gate_proj", "A")))
        assert torch.equal(b[2][2, :Fl, :12], h(key("up_proj", "B")[rank * Fl:(rank + 1) * Fl]))
        assert torch.equal(b[2][2, Fl:, :12], h(key("gate_proj", "B")[rank * Fl:(rank + 1) * Fl]))
        assert pool.dims_ends == [(nq, nq + nkv), (H, H), (Fl, 2 * Fl), (H, H)]
        assert not any(t[:2].any() for ts in pool.a + pool.b for t in ts)            # other slots untouched
        pool.unload(2)
        assert pool.loaded[2] is False and not pool.slice_mask.any() and not any(t.any() for ts in pool.a + pool.b for t in ts)
        assert [s for s in SITES] == ["qkv", "o", "up_gate", "down"]


def test_bf16_source_is_rounded_once_to_the_model_dtype():
    from swiftllm_b200.model_config import LlamaModelConfig
    from swiftllm_b200.worker.lora import LoraPool
    from test_host_path_cpu import CFG
    config, tensors = make_adapter(CFG, 8, 4, modules=("o_proj",), layers=[0])
    k = "base_model.model.model.layers.0.self_attn.o_proj.lora_A.weight"
    for dt in (torch.float16, torch.bfloat16):
        pool = LoraPool(LlamaModelConfig(CFG), 1, 8, dt, "cpu", 4)
        pool.load(0, (config, tensors))
        assert torch.equal(pool.a[0][1][0, :8], tensors[k].to(dt))


# ---------------------------------------------------------------- ValueErrors
def _bad_adapters(cfg):
    c, t = make_adapter(cfg, 8, 5)
    k0 = next(iter(t))
    yield "shape", (dict(c, r=4), t)
    big_c, big_t = make_adapter(cfg, 32, 5)
    yield "exceeds max_lora_rank", (big_c, big_t)
    yield "shape", (c, dict(t, **{k0: t[k0][:, :-1]}))
    yield "fan_in_fan_out", (dict(c, fan_in_fan_out=True), t)
    yield "bias", (dict(c, bias="all"), t)
    yield "bias", (dict(c, bias="lora_only"), t)
    for k in ("rank_pattern", "alpha_pattern"):
        yield k, (dict(c, **{k: {"q_proj": 4}}), t)
    yield "modules_to_save", (dict(c, modules_to_save=["lm_head"]), t)
    yield "layers_to_transform", (dict(c, layers_to_transform=[0]), t)
    yield "embed_tokens or lm_head", (dict(c, target_modules=["q_proj", "embed_tokens"]), t)
    yield "embed_tokens or lm_head", (c, dict(t, **{"base_model.model.lm_head.lora_A.weight": torch.zeros(8, 4)}))
    yield "unrecognised", (c, dict(t, **{"base_model.model.model.layers.0.mlp.q_proj.lora_A.weight": torch.zeros(8, 4)}))
    yield "outside the model", (c, dict(t, **{"base_model.model.model.layers.9.mlp.up_proj.lora_A.weight": t[k0]}))
    yield "both be present", (c, {k: v for k, v in t.items() if not k.endswith("q_proj.lora_B.weight")})
    yield "DoRA", (dict(c, use_dora=True), t)


def test_load_lora_value_errors_copy_nothing():
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG, _product
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=2, std=0.08)
    with product_on_cpu():
        m0 = _product(w)
        with pytest.raises(ValueError, match="max_loras"):
            m0.load_lora(0, make_adapter(CFG, 8, 1))
        with pytest.raises(ValueError, match="max_lora_rank"):
            _product(w, max_loras=1, max_lora_rank=12)
        m = _product(w, max_loras=2, max_lora_rank=16)
        good = make_adapter(CFG, 8, 9)
        m.load_lora(1, good)
        before = [t.clone() for ts in m.lora.a + m.lora.b for t in ts] + [m.lora.slice_mask.clone(), m.lora.scales.clone()]
        for slot in (-1, 2, True, 1.0):
            with pytest.raises(ValueError, match="slot"):
                m.load_lora(slot, good)
        for msg, bad in _bad_adapters(CFG):
            with pytest.raises(ValueError, match=msg):
                m.load_lora(1, bad)
        with pytest.raises(ValueError):
            m.load_lora(1, "/nonexistent/adapter/dir")
        after = [t for ts in m.lora.a + m.lora.b for t in ts] + [m.lora.slice_mask, m.lora.scales]
        assert all(torch.equal(a, b) for a, b in zip(before, after)) and m.lora.loaded == [False, True]


def test_forward_value_errors_enqueue_nothing():
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG, _product
    from test_speculative_cpu import SPEC
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=2, std=0.08)
    with product_on_cpu(PATCH + SPEC):
        m = _product(w, max_loras=2, max_lora_rank=16)
        m.load_lora(0, make_adapter(CFG, 8, 9))
        staged = []
        orig = m._stage_metadata
        m._stage_metadata = lambda *parts, **kw: (staged.append(parts), orig(*parts, **kw))[1]
        for ids, kw, msg in (([0], {}, "entries"), ([0, 0, 0], {}, "entries"), ([0, 1], {}, "not loaded"),
                             ([0, 2], {}, "not loaded"), ([0, -1], {}, "not loaded"), ([0, "0"], {}, "slot id"),
                             ([True, None], {}, "slot id"), ([0, None], dict(ignore_kvcache=True), "ignore_kvcache"),
                             ([None, None], dict(ignore_kvcache=True), "ignore_kvcache")):
            with pytest.raises(ValueError, match=msg):
                m.forward([[1, 2], [3]], [0, 1], [], lora_ids_list=ids, **kw)
            with pytest.raises(ValueError, match=msg):
                m.forward_with_logprobs([[1, 2], [3]], [0, 1], [], lora_ids_list=ids, **kw)
        for ids in ([0], [1, None]):
            with pytest.raises(ValueError):
                m.forward_speculative([[1, 2], [3]], [0, 1], [0, 0], lora_ids_list=ids)
        m0 = _product(w)
        with pytest.raises(ValueError, match="not loaded"):
            m0.forward([[1]], [0], [], lora_ids_list=[0])
        assert staged == [] and m.gpu_block_manager.num_free_blocks == m.gpu_block_manager.num_blocks
        with pytest.raises(ValueError, match="slot"):
            m.unload_lora(5)


def test_lora_kernels_reject_invalid_arguments_before_launch():
    from swiftllm_b200 import _lib
    l = _lib.lib()
    sn = (("x", 16), ("ldx", 4096), ("rows", 4), ("K", 4096), ("u", 16), ("ldu", 192), ("a", 16), ("astr", 192 * 4096),
          ("cols", 192), ("tiles", 16), ("nt", 2), ("mask", 16), ("ml", 2), ("dtype", 1), ("stream", None))
    sargs = lambda **kw: [kw.get(n, d) for n, d in sn]
    for kw, msg in (({"dtype": 5}, b"dtype"), ({"rows": -1}, b"num_rows"), ({"K": 48}, b"multiple of 32"), ({"K": 0}, b"in_features"),
                    ({"ldx": 4000}, b"x_row_stride"), ({"ldx": 4100}, b"x_row_stride"), ({"cols": 8}, b"u_cols"),
                    ({"cols": 208}, b"u_cols"), ({"ldu": 100}, b"u_row_stride"), ({"astr": 100}, b"a_slot_stride"),
                    ({"ml": 0}, b"max_loras"), ({"nt": -1}, b"num_tiles"), ({"x": None}, b"null pointer"),
                    ({"tiles": None}, b"null pointer"), ({"mask": None}, b"null pointer"), ({"x": 8}, b"aligned")):
        assert l.sllm_lora_shrink(*sargs(**kw)) != 0, kw
        assert msg in l.sllm_last_error(), (kw, l.sllm_last_error())
    assert l.sllm_lora_shrink(*sargs(nt=0, x=None, u=None, a=None, tiles=None, mask=None)) == 0     # no tiles: nothing to launch
    en = (("y", 16), ("ldy", 6144), ("rows", 4), ("N", 6144), ("u", 16), ("ldu", 192), ("b", 16), ("bstr", 6144 * 64),
          ("R", 64), ("n1", 4096), ("n2", 5120), ("tiles", 16), ("nt", 2), ("mask", 16), ("scales", 16), ("ml", 2), ("dtype", 0),
          ("stream", None))
    eargs = lambda **kw: [kw.get(n, d) for n, d in en]
    for kw, msg in (({"dtype": 5}, b"dtype"), ({"N": 6140}, b"out_features"), ({"ldy": 6000}, b"y_row_stride"),
                    ({"ldy": 6145}, b"y_row_stride"), ({"R": 8}, b"rank"), ({"R": 80}, b"rank"), ({"n1": 4100}, b"slice"),
                    ({"n1": 5200}, b"slice"), ({"n2": 7000}, b"slice"), ({"ldu": 128}, b"u_row_stride"),
                    ({"bstr": 64}, b"b_slot_stride"), ({"ml": 0}, b"max_loras"), ({"nt": 2 ** 31}, b"num_tiles"),
                    ({"scales": None}, b"null pointer"), ({"y": None}, b"null pointer"), ({"u": 4}, b"aligned")):
        assert l.sllm_lora_expand(*eargs(**kw)) != 0, kw
        assert msg in l.sllm_last_error(), (kw, l.sllm_last_error())
    # u columns for one rank suffice for one slice, two ranks for two: those calls pass the stride check and stop at the null
    # pointer check after it; one rank too few does not
    for n1, n2, ldu, msg in ((6144, 6144, 64, b"null pointer"), (4096, 6144, 128, b"null pointer"), (4096, 6144, 64, b"u_row_stride"),
                             (4096, 5120, 128, b"u_row_stride"), (4096, 5120, 192, b"null pointer")):
        assert l.sllm_lora_expand(*eargs(n1=n1, n2=n2, ldu=ldu, y=None)) != 0
        assert msg in l.sllm_last_error(), (n1, n2, ldu, l.sllm_last_error())
    assert l.sllm_lora_expand(*eargs(nt=0, y=None, u=None, b=None, tiles=None, mask=None, scales=None)) == 0


# ---------------------------------------------------------------- tile lists
def test_tile_lists_cut_runs_of_equal_slot():
    from swiftllm_b200.worker.lora import lora_tiles
    t = lambda *a, **kw: np.asarray(lora_tiles(*a, **kw)).reshape(-1, 3).tolist()
    assert t([0, 0, None, 1, 1, 1], [70, 3, 5, 1, 1, 1]) == [[0, 64, 0], [64, 9, 0], [78, 3, 1]]
    assert t([None, None], [3, 1]) == []
    assert t([2], [128]) == [[0, 64, 2], [64, 64, 2]]
    assert t([2], [129]) == [[0, 64, 2], [64, 64, 2], [128, 1, 2]]
    assert t([1, 2, 1, 1], [1, 1, 1, 1], pad_to=4) == [[0, 1, 1], [1, 1, 2], [2, 2, 1], [0, 0, 0]]
    assert t([0, None, 0], [1, 1, 1]) == [[0, 1, 0], [2, 1, 0]]                  # a base row splits the run
    assert t([0, 0], [0, 5]) == [[0, 5, 0]]
    # runs of up to 64 rows: pieces of 16
    assert t([3] * 40, [1] * 40) == [[0, 16, 3], [16, 16, 3], [32, 8, 3]]
    assert t([3, 3], [60, 4]) == [[0, 16, 3], [16, 16, 3], [32, 16, 3], [48, 16, 3]]


# ---------------------------------------------------------------- host path with stand-ins of the kernels
CALLS = []


def _shrink_stand_in(x, u, lora_a, tiles, slice_mask):
    CALLS.append("shrink")
    for r0, n, a in tiles.tolist():
        if n < 1 or int(slice_mask[a]) == 0:
            continue
        u[r0:r0 + n, :lora_a.shape[1]] = LO.shrink(x[r0:r0 + n], lora_a[a])


def _expand_stand_in(y, u, lora_b, ends, tiles, slice_mask, scales):
    CALLS.append("expand")
    R = lora_b.shape[2]
    for r0, n, a in tiles.tolist():
        if n < 1 or int(slice_mask[a]) == 0:
            continue
        y[r0:r0 + n] = LO.expand_exact(y[r0:r0 + n], u[r0:r0 + n], lora_b[a], float(scales[a]), ends, int(slice_mask[a]), R)


PATCH = [("swiftllm_b200.worker.layers.transformer_layer", "lora_shrink", _shrink_stand_in),
         ("swiftllm_b200.worker.layers.transformer_layer", "lora_expand", _expand_stand_in)]


def merged_weights(w, cfg, adapter):
    """OracleWeights with W + s·B·A for every module of the adapter."""
    from swiftllm_b200.model_config import LlamaModelConfig
    from swiftllm_b200.worker.lora import parse_adapter
    config, tensors = adapter
    s, mods = parse_adapter(config, tensors, LlamaModelConfig(cfg), 64)
    F = cfg["intermediate_size"]
    out = copy.deepcopy(w)
    for (i, name), (A, B) in mods.items():
        lw = out.layers[i]
        A, B = A.to(w.wte.dtype), B.to(w.wte.dtype)                  # the pool's one rounding
        if name in ("up_proj", "gate_proj"):
            sl = slice(0, F) if name == "up_proj" else slice(F, 2 * F)
            lw.up_gate_proj = lw.up_gate_proj.clone()
            lw.up_gate_proj[sl] = LO.merged_weight(lw.up_gate_proj[sl], A, B, s)
        else:
            setattr(lw, name, LO.merged_weight(getattr(lw, name), A, B, s))
    return out


def _models(w, cfg=None, **kw):
    from test_host_path_cpu import CFG, _oracle, _product
    return _product(w, max_loras=3, max_lora_rank=16, **kw)


def test_adapted_logits_match_merged_weights_and_base_rows_are_untouched():
    """Mixed batches (prefill + decode, chunked prefill) with two adapters and base rows: adapted rows' logits against an oracle
    model carrying the merged weights W + s·B·A, base rows bit-identical to the same steps run without lora_ids_list.  The
    tolerance: the adapted model rounds u and y + delta where the merged one rounds W + s·B·A; each is half a 16-bit ulp of its
    value, so the difference is a small fraction of what the adapter changes (err_base: the base model against the merged one)."""
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG, _oracle
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=2, std=0.08)
    ad = {0: make_adapter(CFG, 8, 11, std=0.1), 2: make_adapter(CFG, 16, 12, std=0.08, modules=("q_proj", "v_proj", "down_proj"))}
    rng = np.random.default_rng(3)
    with product_on_cpu(PATCH):
        m, base = _models(w), _models(w)
        for s, a in ad.items():
            m.load_lora(s, a)
        oracles = {s: _oracle(merged_weights(w, CFG, a)) for s, a in ad.items()}
        prompts = [rng.integers(0, 300, size=n).tolist() for n in (19, 5, 70)]
        slots = [0, None, 2]
        sids = [0, 1, 2]
        ids, dec = prompts, []
        lens = [19, 5, 70]
        for step in range(3):
            t_m = m.forward(ids, sids, dec, lora_ids_list=slots)
            t_b = base.forward(ids, sids, dec)
            got, ref_b = m.post_layer.last_logits, base.post_layer.last_logits
            for r, s in enumerate(slots):
                if s is None:
                    assert torch.equal(_bits(got[r]), _bits(ref_b[r]))
            for s, o in oracles.items():
                o.forward(ids, sids, dec)
                r = slots.index(s)
                ref = o.last_logits[r].float()
                err = float((got[r].float() - ref).abs().max())
                err_base = float((ref_b[r].float() - ref).abs().max())
                assert err <= 0.1 * err_base and err <= 2e-2 * float(ref.abs().max()), (step, s, err, err_base)
            # the base model and the oracles follow the adapted model's tokens, so every cache holds the same inputs
            lens = [l + 1 for l in lens]
            ids, dec = [[t] for t in t_m], lens


def test_tile_lists_of_mixed_and_speculative_steps_and_unadapted_staging():
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG
    from test_speculative_cpu import SPEC
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=3, std=0.08)
    with product_on_cpu(PATCH + SPEC):
        runs = []
        for variant in range(4):
            m = _models(w) if variant else __import__("test_host_path_cpu")._product(w)
            if variant:
                m.load_lora(1, make_adapter(CFG, 8, 5))
            staged = []
            orig = m._stage_metadata
            m._stage_metadata = lambda *parts, **kw: (staged.append([list(p) for p in parts]), orig(*parts, **kw))[1]
            CALLS.clear()
            kw = [dict(), dict(), dict(lora_ids_list=None), dict(lora_ids_list=[None, None, None])][variant]
            t = m.forward([[1, 2, 3], [4, 5], [6] * 70], [0, 1, 2], [], **kw)
            t += m.forward([[t[0]], [t[1]], [t[2]]], [0, 1, 2], [4, 3, 71], **kw)
            t += m.forward_speculative([[1, 2, 3]], [3], [0], **({} if not kw else dict(lora_ids_list=[None])))[0]
            runs.append((staged, t, list(CALLS)))
            assert CALLS == []
        assert runs[0] == runs[1] == runs[2] == runs[3]
        # adapted: the tiles follow the sampling / constraint words and precede the ids
        m = _models(w)
        m.load_lora(1, make_adapter(CFG, 8, 5))
        m.load_lora(0, make_adapter(CFG, 8, 6))
        staged = []
        orig = m._stage_metadata
        m._stage_metadata = lambda *parts, **kw: (staged.append([list(p) for p in parts]), orig(*parts, **kw))[1]
        m.forward([[1, 2, 3], [4, 5], [6] * 70, [7]], [0, 1, 2, 4], [], lora_ids_list=[1, 1, 1, None])
        assert staged[-1][0] == [0, 64, 1, 64, 11, 1] and len(staged[-1]) == 9
        m.forward([[1], [2], [3], [4]], [0, 1, 2, 4], [4, 3, 71, 2], lora_ids_list=[None, 0, 0, 1])
        assert staged[-1][0] == [1, 2, 0, 3, 1, 1]
        m.forward([[5, 6], [7]], [5, 6], [], lora_ids_list=[0, None])            # mixed: prefill then decode rows
        m.forward([[5, 6, 7], [8]], [7, 5], [3], lora_ids_list=[1, 1])
        assert staged[-1][0] == [0, 4, 1]
        # speculative rows share their entry's slot
        m.forward_speculative([[1, 2, 3], [4, 5]], [0, 1], [4, 4], lora_ids_list=[None, 0])
        assert staged[-1][0] == [3, 2, 0] and len(staged[-1]) == 10


@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "seeded-sampling"])
def test_speculative_with_an_adapter_returns_the_plain_adapted_steps(sampled):
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200 import SamplingParams
    from test_host_path_cpu import CFG
    from test_speculative_cpu import SPEC
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=9, std=0.08)
    rng = np.random.default_rng(7 + sampled)
    sp = SamplingParams(0.9 if sampled else 0.0, seed=21)
    from test_constraints_cpu import PATCH as CON_PATCH          # stand-ins of the sampling kernels
    ad = make_adapter(CFG, 16, 31, std=0.12)
    with product_on_cpu(PATCH + SPEC + CON_PATCH):
        plain, spec = _models(w), _models(w)
        plain.load_lora(2, ad); spec.load_lora(2, ad)
        for sid, (k, wrong) in enumerate(((5, 2), (6, None), (3, 0))):
            prompt = rng.integers(0, 300, size=13 + sid).tolist()
            x = plain.forward([prompt], [sid], [], sampling_params_list=[sp], lora_ids_list=[2])[0]
            assert spec.forward([prompt], [sid], [], sampling_params_list=[sp], lora_ids_list=[2])[0] == x
            L = len(prompt)
            ys, inp = [], x
            for j in range(k + 1):
                ys.append(plain.forward([[inp]], [sid], [L + j + 1], sampling_params_list=[sp], lora_ids_list=[2])[0])
                inp = ys[-1]
            drafts = list(ys[:k])
            if wrong is not None:
                drafts[wrong] = (drafts[wrong] + 1) % 300
            out = spec.forward_speculative([[x] + drafts], [sid], [L], sampling_params_list=[sp], lora_ids_list=[2])[0]
            assert out == ys[:(k if wrong is None else wrong) + 1]


def test_graph_path_keys_and_stages_lora_tiles():
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=5, std=0.08)
    with product_on_cpu(PATCH):
        m = _models(w, use_cuda_graph=True)
        m.load_lora(0, make_adapter(CFG, 8, 5))
        m.load_lora(1, make_adapter(CFG, 8, 6))
        caps, staged = [], []
        orig = m._stage_metadata

        def fake_capture(B, bucket, filtered=None, top_n=None, penalized=False, sampled=True, con=None, **kw):
            caps.append((B, filtered, con, kw))
            nl = 3 * B if kw.get("lora") else 0
            g = type("G", (), {"replay": lambda self: None})()
            return dict(graph=g, meta=torch.zeros((nl + 3 * B,), dtype=torch.int32), tokens=torch.zeros((B,), dtype=torch.int64),
                        logprobs=None)
        m._capture_decode_graph = fake_capture
        m._stage_metadata = lambda *parts, **kw: (staged.append([list(p) for p in parts]), orig(*parts, **kw))[1]
        m.forward([[1, 2, 3], [4, 5], [6]], [0, 1, 2], [])
        m.forward([[1], [2], [3]], [0, 1, 2], [4, 3, 2])
        m.forward([[1], [2], [3]], [0, 1, 2], [5, 4, 3], lora_ids_list=[None, None, None])
        m.forward([[1], [2], [3]], [0, 1, 2], [6, 5, 4], lora_ids_list=[1, None, 1])
        m.forward([[1], [2], [3]], [0, 1, 2], [7, 6, 5], lora_ids_list=[0, 0, 1])
        assert caps == [(3, None, None, {}), (3, None, None, {"lora": True})]
        assert [k[0] for k in m._graphs] == [3, 3] and [k[2:] for k in m._graphs] == [(), ("lora",)]
        assert staged[1][0] == [1, 2, 3] and staged[2][0] == [1, 2, 3]
        assert staged[3][0] == [0, 1, 1, 2, 1, 1, 0, 0, 0] and staged[4][0] == [0, 2, 0, 2, 1, 1, 0, 0, 0]


# ---------------------------------------------------------------- tensor parallelism over gloo
def _tp_worker(rank, world, port, ret, comm):
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import warnings
    import swiftllm_b200
    from cpu_shim import GlooFusedAllReduce, product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200.worker.weight import dict_getter
    from test_host_path_cpu import _hf_tensors
    from test_tp_gloo import CFG
    cfg = dict(CFG, num_hidden_layers=2, vocab_size=96)
    w = OracleWeights.random(cfg, dtype=torch.float16, seed=12, std=0.08)
    ad = make_adapter(cfg, 16, 40, std=0.1)
    extra = [("swiftllm_b200.worker.tp_comm", "FusedAllReduce", GlooFusedAllReduce)] if comm else []
    ok, out = True, []
    with product_on_cpu(PATCH + extra), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        models = []
        for tp in (world, 1):
            ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=2,
                                            max_seqs_in_block_table=8, max_blocks_per_seq=8, max_batch_size=8,
                                            max_tokens_in_batch=128, dtype="float16", tp_size=tp, tp_rank=rank if tp > 1 else 0,
                                            fused_allreduce=(bool(comm) if tp > 1 else False), max_loras=2, max_lora_rank=16)
            m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(cfg))
            m.load_weights(dict_getter(_hf_tensors(w, cfg["intermediate_size"])))
            m.init_kvcache_and_swap(20)
            m.post_layer.keep_logits = True
            m.load_lora(1, ad)
            models.append(m)
        sharded, single = models
        ok &= (sharded.comm is not None) == bool(comm)
        rng = np.random.default_rng(2)
        ids = [rng.integers(0, 96, size=n).tolist() for n in (21, 3)]
        sids, dec, lens = [4, 1], [], [21, 3]
        for step in range(3):
            got = sharded.forward(ids, sids, dec, lora_ids_list=[1, None])
            ref = single.forward(ids, sids, dec, lora_ids_list=[1, None])
            g, r = sharded.post_layer.last_logits.float(), single.post_layer.last_logits.float()
            rel = float((g - r).abs().max() / r.abs().max())
            ok &= rel <= 4e-3
            out.append(rel)
            lens = [l + 1 for l in lens]
            ids, dec = [[x] for x in ref], lens
    gathered = [None] * world
    dist.all_gather_object(gathered, (bool(ok), out))
    if rank == 0:
        ret.put(gathered)
    dist.destroy_process_group()
    ret.close()
    ret.join_thread()
    os._exit(0)


@pytest.mark.parametrize("comm", [False, True], ids=["all-reduce", "fused-exchange"])
def test_tensor_parallel_adapted_logits_equal_the_single_rank_ones(comm):
    """World 2 over gloo: the row-parallel sites add each rank's partial delta before the exchange; the sum equals the single-rank
    delta (within fp16 tolerance) with no added collective."""
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_tp_worker, args=(r, 2, 29970 + int(comm), ret, comm)) for r in range(2)]
    for p in procs:
        p.start()
    out = ret.get(timeout=240)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(ok for ok, _ in out), out


# ---------------------------------------------------------------- examples/offline.py --lora
def test_offline_example_adapter_wrapper_leaves_the_profiling_forward_alone():
    """examples/offline.py --lora wraps the model so that every call runs under the adapter.  The profiling forward
    (profile_num_blocks: ignore_kvcache=True, which takes no adapter) must still run - as the base model - and generation calls,
    speculative ones included, must carry the slot."""
    import importlib.util
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG
    from test_speculative_cpu import SPEC
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("offline_example", os.path.join(root, "examples", "offline.py"))
    ex = importlib.util.module_from_spec(spec); spec.loader.exec_module(ex)
    src = open(os.path.join(root, "examples", "offline.py"), encoding="utf-8").read()
    assert src.index("with_adapter(model, 0)") > src.index("model.init_kvcache_and_swap(num_blocks)")
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=4, std=0.08)
    with product_on_cpu(PATCH + SPEC):
        m, ref = _models(w), _models(w)
        ad = make_adapter(CFG, 8, 3, std=0.1)
        m.load_lora(0, ad); ref.load_lora(0, ad)
        ex.with_adapter(m, 0)
        CALLS.clear()
        m.forward([[1, 2, 3]], [0], [], ignore_kvcache=True)          # what profile_num_blocks runs
        assert CALLS == []
        got = m.forward([[1, 2, 3], [4, 5]], [0, 1], [])
        assert CALLS and got == ref.forward([[1, 2, 3], [4, 5]], [0, 1], [], lora_ids_list=[0, 0])
        assert m.forward_speculative([[got[0], 7]], [0], [3]) == ref.forward_speculative([[got[0], 7]], [0], [3], lora_ids_list=[0])
        assert [r.token for r in m.forward_with_logprobs([[got[1]]], [1], [3])] == \
            ref.forward([[got[1]]], [1], [3], lora_ids_list=[0])


def test_pool_refuses_shapes_the_kernels_cannot_serve():
    from swiftllm_b200.model_config import LlamaModelConfig
    from swiftllm_b200.worker.lora import LoraPool
    from test_host_path_cpu import CFG
    for cfg, tp in ((dict(CFG, intermediate_size=200), 1),             # down in_features 200
                    (dict(CFG, intermediate_size=192), 2),             # down in_features 96 per rank: fine ...
                    (dict(CFG, intermediate_size=192), 4)):            # ... 48 per rank: not a multiple of 32
        mc = LlamaModelConfig(cfg)
        if (mc.ffn_inter_dim // tp) % 32 == 0:
            LoraPool(mc, 1, 8, torch.float16, "cpu", 4, tp_size=tp)
            continue
        with pytest.raises(ValueError, match="multiple of 32"):
            LoraPool(mc, 1, 8, torch.float16, "cpu", 4, tp_size=tp)
    LoraPool(LlamaModelConfig(dict(CFG, num_attention_heads=32, num_key_value_heads=2, hidden_size=128)), 1, 8, torch.float16,
             "cpu", 4)                                              # head_dim 4: k / v slices of 8 columns
    with pytest.raises(ValueError, match="multiples of 8"):
        LoraPool(LlamaModelConfig(dict(CFG, num_attention_heads=32, num_key_value_heads=1, hidden_size=128)), 1, 8, torch.float16,
                 "cpu", 4)                                          # k / v slices of 4 columns


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_ordered_shrink_reference_catches_a_single_dropped_product(dtype):
    """The GPU tests hold the shrink to lora_oracle.shrink_ordered (the kernel's summation order) and its bound.  The correctly
    rounded fp64 result passes that check; u computed with one k element of x dropped does not, at K = 14336 where the worst-case
    bound K * eps32 * sum |x A| (lora_oracle.shrink_bound) lets it through."""
    g = torch.Generator().manual_seed(1)
    K, J = 14336, 48
    x = torch.randn((4, K), generator=g).to(dtype)
    A = (torch.randn((J, K), generator=g) * 0.05).to(dtype)
    ref, E = LO.shrink_ordered(x, A)
    assert bool(LO.shrink_check(LO.shrink(x, A), ref, E).all())
    assert bool(LO.shrink_check(ref.to(dtype), ref, E).all())
    caught = 0
    for k in (0, 5, 777, K - 1):
        xb = x.clone()
        xb[:, k] = 0
        bad = LO.shrink(xb, A)
        assert bool(((bad.double() - LO.shrink(x, A).double()).abs() <= LO.shrink_bound(x, A)).all())     # the loose bound passes it
        caught += int((~LO.shrink_check(bad, ref, E)).any(dim=1).sum())
    assert caught == 4 * 4, caught                                          # every row, every dropped element
