"""CPU: FP8 weights (worker/fp8.py, csrc/fp8.cu's numerics).  The restatement in tests/fp8_oracle.py, checkpoint formats and their
refusals, loading and tensor-parallel slicing, and the product's host path through stand-ins of the FP8 kernels against an fp64
FP8 restatement of the oracle model."""
import json
import os

import numpy as np
import pytest
import torch

import fp8_oracle as FO
from oracle import kernels as K

TL = "swiftllm_b200.worker.layers.transformer_layer"
CALLS = []


def _bits(t):
    return t.view(torch.uint8) if t.dtype == torch.float8_e4m3fn else t.view(torch.int16)


# ---------------------------------------------------------------- the restatement
def test_e4m3_rounding_ties_saturation_and_subnormals():
    # s = 1 exactly: amax 448
    y = torch.tensor([[448.0, 17.0, 19.0, -17.0, 2.0 ** -9, 2.0 ** -10, 3 * 2.0 ** -11, 0.0, -448.0, 240.0, 232.0]],
                     dtype=torch.float32)
    q, s = FO.quantize_rows(y)
    assert float(s[0]) == 1.0
    # ties to even: 17 -> 16, 19 -> 20, 232 (between 224 and 240) -> 224; subnormals: 2^-10 is half the smallest -> 0 (even)
    assert q.float().tolist()[0] == [448.0, 16.0, 20.0, -16.0, 2.0 ** -9, 0.0, 2.0 ** -9, 0.0, -448.0, 240.0, 224.0]
    # the clamp is what makes the cast saturating: torch's cast alone turns 480 into NaN
    assert torch.isnan(torch.tensor([480.0]).to(torch.float8_e4m3fn).float()).all()
    # rows whose amax / 448 rounds down divide to just above 448: saturated, never NaN
    g = torch.Generator().manual_seed(0)
    rows = torch.randn(4096, 64, generator=g, dtype=torch.float32) * torch.rand(4096, 1, generator=g) * 100
    q, s = FO.quantize_rows(rows.to(torch.float16))
    qa = q.float().abs()
    assert not torch.isnan(qa).any() and float(qa.max()) == 448.0
    assert bool(((qa.amax(dim=1) == 448.0) | (rows.abs().amax(dim=1) == 0)).all())


def test_zero_rows_and_the_scale_floor():
    y = torch.zeros(3, 32, dtype=torch.bfloat16)
    y[1, 3] = 2.0 ** -133                     # bf16 subnormal: amax / 448 is below 2^-126
    q, s = FO.quantize_rows(y)
    assert s.tolist() == [2.0 ** -126] * 3
    assert torch.equal(q[0].float(), torch.zeros(32)) and torch.equal(q[2].float(), torch.zeros(32))
    assert float(q[1, 3].float()) == 2.0 ** -7          # 2^-133 / 2^-126, an e4m3 subnormal


def test_per_channel_weight_quantization_and_composition_with_the_row_kernels():
    g = torch.Generator().manual_seed(1)
    w = (torch.randn(48, 64, generator=g) * 0.02).to(torch.float16)
    q, s = FO.quantize_rows(w)
    assert q.shape == w.shape and s.shape == (48,)
    assert bool((q.float().abs().amax(dim=1) == 448.0).all())
    deq = FO.dequantize(q, s)
    assert float(((deq - w.double()).abs() / w.double().abs().amax(dim=1, keepdim=True)).max()) <= 2.0 ** -4
    for dt in (torch.float16, torch.bfloat16):
        x = (torch.randn(5, 64, generator=g) * 3).to(dt)
        r = (torch.randn(5, 64, generator=g)).to(dt)
        nw = (1 + torch.randn(64, generator=g) * 0.1).to(dt)
        (qx, sx), r2 = FO.add_rmsnorm_quant(x, r, nw, 1e-5)
        y, rr = K.fused_add_rmsnorm(x, r, nw, 1e-5)
        assert torch.equal(_bits(r2), _bits(rr))
        q2, s2 = FO.quantize_rows(y)
        assert torch.equal(_bits(qx), _bits(q2)) and torch.equal(sx, s2)
        ug = (torch.randn(5, 128, generator=g) * 2).to(dt)
        qh, sh = FO.silu_and_mul_quant(ug)
        q3, s3 = FO.quantize_rows(K.silu_and_mul(ug)[:, :64])
        assert torch.equal(_bits(qh), _bits(q3)) and torch.equal(sh, s3)


# ---------------------------------------------------------------- checkpoint formats
def _ct(strategy="channel", **edit):
    qc = FO.compressed_tensors_config(strategy)
    g = qc["config_groups"]["group_0"]
    for k, v in edit.items():
        where, _, field = k.partition("__")
        target = {"qc": qc, "w": g["weights"], "a": g["input_activations"], "g": g}[where]
        if v is None and field in target and where != "qc":
            target[field] = None
        else:
            target[field] = v
    return qc


ACCEPTED = [
    ("ct-channel", _ct("channel"), "channel"),
    ("ct-tensor", _ct("tensor"), "tensor"),
    ("ct-no-ignore", _ct("channel", qc__ignore=[]), "channel"),
    ("autofp8", {"quant_method": "fp8", "activation_scheme": "dynamic"}, "tensor"),
    ("autofp8-ignored-lm-head", {"quant_method": "fp8", "activation_scheme": "dynamic", "ignored_layers": ["lm_head"]}, "tensor"),
]

REFUSED = [
    ("awq", {"quant_method": "awq", "bits": 4, "group_size": 128}, "quant_method"),
    ("gptq", {"quant_method": "gptq", "bits": 4}, "quant_method"),
    ("bitsandbytes", {"quant_method": "bitsandbytes", "load_in_8bit": True}, "quant_method"),
    ("fbgemm_fp8", {"quant_method": "fbgemm_fp8", "activation_scale_ub": 1200.0}, "quant_method"),
    ("autofp8-block", {"quant_method": "fp8", "activation_scheme": "dynamic", "weight_block_size": [128, 128]}, "weight_block_size"),
    ("autofp8-static", {"quant_method": "fp8", "activation_scheme": "static"}, "activation_scheme"),
    ("ct-kv-cache", _ct(qc__kv_cache_scheme={"num_bits": 8, "type": "float"}), "kv_cache_scheme"),
    ("ct-ignore-projection", _ct(qc__ignore=["lm_head", "model.layers.0.mlp.down_proj"]), "ignore"),
    ("ct-num-bits", _ct(w__num_bits=4), "num_bits"),
    ("ct-int", _ct(w__type="int"), "type"),
    ("ct-asymmetric", _ct(w__symmetric=False), "symmetric"),
    ("ct-group", _ct(w__strategy="group", w__group_size=128), "group"),
    ("ct-block", _ct(w__strategy="block", w__block_structure=[128, 128]), "block"),
    ("ct-static-activations", _ct(a__dynamic=False), "dynamic"),
    ("ct-tensor-activations", _ct(a__strategy="tensor"), "strategy"),
    ("ct-no-activations", _ct(g__input_activations=None), "input_activations"),
    ("ct-format", _ct(qc__format="pack-quantized"), "format"),
    ("ct-two-groups", dict(_ct(), config_groups={"a": _ct()["config_groups"]["group_0"], "b": _ct()["config_groups"]["group_0"]}),
     "config_groups"),
]


@pytest.mark.parametrize("qc,want", [a[1:] for a in ACCEPTED], ids=[a[0] for a in ACCEPTED])
def test_accepted_checkpoint_formats(qc, want):
    from swiftllm_b200.worker import fp8
    assert fp8.checkpoint_format({"quantization_config": qc}) == want
    assert fp8.checkpoint_format({}) is None


@pytest.mark.parametrize("qc,field", [a[1:] for a in REFUSED], ids=[a[0] for a in REFUSED])
def test_refused_checkpoint_formats_name_the_field(qc, field):
    from swiftllm_b200.worker import fp8
    with pytest.raises(ValueError, match=field):
        fp8.checkpoint_format({"quantization_config": qc})


def _cfg(**kw):
    from test_host_path_cpu import CFG
    return dict(CFG, **kw)


@pytest.mark.parametrize("case", ["unknown", "lora", "float16", "K", "N", "bad-checkpoint"])
def test_engine_refuses_before_allocating(case):
    import swiftllm_b200
    from cpu_shim import product_on_cpu
    cfg = _cfg()
    kw = dict(quantization="fp8")
    if case == "unknown":
        kw = dict(quantization="int4")
    elif case == "lora":
        kw.update(max_loras=1, max_lora_rank=8)
    elif case == "float16":
        pass                                       # the dtype alone
    elif case == "K":
        cfg = _cfg(intermediate_size=200)          # down_proj K = 200
    elif case == "N":
        cfg = _cfg(intermediate_size=196)          # up_gate N = 392, down K = 196
    else:
        kw = {}
        cfg = _cfg(quantization_config={"quant_method": "awq"})
    ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=True, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=2,
                                    max_seqs_in_block_table=8, max_blocks_per_seq=8, max_batch_size=8, max_tokens_in_batch=64,
                                    dtype="float16" if case == "float16" else "bfloat16", **kw)
    with product_on_cpu(), pytest.raises(ValueError, match={"unknown": "quantization", "lora": "LoRA", "float16": "bfloat16",
                                                            "K": "multiples of 16", "N": "multiples of 16",
                                                            "bad-checkpoint": "quant_method"}[case]):
        swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(cfg))


def test_cli_flag():
    import argparse
    import swiftllm_b200
    ap = argparse.ArgumentParser()
    swiftllm_b200.EngineConfig.add_cli_args(ap)
    assert ap.parse_args(["--model-path", "x", "--quantization", "fp8"]).quantization == "fp8"
    assert ap.parse_args(["--model-path", "x"]).quantization is None
    with pytest.raises(SystemExit):
        ap.parse_args(["--model-path", "x", "--quantization", "awq"])


# ---------------------------------------------------------------- stand-ins of the FP8 kernels and of linear_fp8
def _add_rmsnorm_quant(x, residual, weight, eps):
    CALLS.append("add_rmsnorm_quant")
    (q, s), r = FO.add_rmsnorm_quant(x, residual, weight, eps)
    residual.copy_(r)
    return q, s.view(-1, 1)


def _quant_rows(x):
    CALLS.append("quant_rows")
    q, s = FO.quantize_rows(x)
    return q, s.view(-1, 1)


def _silu_and_mul_quant(x):
    CALLS.append("silu_and_mul_quant")
    q, s = FO.silu_and_mul_quant(x)
    return q, s.view(-1, 1)


def _linear_fp8(xq, sx, wq, sw, out_dtype, out=None):
    """Dequantize (exact), then an fp32 GEMM."""
    CALLS.append("linear_fp8" if out is None else "linear_fp8_out")
    y = (FO.dequantize(xq, sx).float() @ FO.dequantize(wq, sw).float().T).to(out_dtype)
    if out is None:
        return y
    out.copy_(y)
    return out


PATCH = [(TL, "fused_add_rmsnorm_quant_fp8", _add_rmsnorm_quant), (TL, "quant_fp8_rows", _quant_rows),
         (TL, "silu_and_mul_quant_fp8", _silu_and_mul_quant), (TL, "linear_fp8", _linear_fp8),
         ("swiftllm_b200.worker.fp8", "quant_fp8_rows", _quant_rows)]


# ---------------------------------------------------------------- loading
def checkpoint_getter(path, device):
    from swiftllm_b200.worker.weight import checkpoint_getter as get
    return get(path, device)


def _write_checkpoint(path, cfg, tensors, qc):
    from safetensors.torch import save_file
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(dict(cfg, quantization_config=qc) if qc is not None else cfg, f)
    save_file({k: v.contiguous() for k, v in tensors.items()}, os.path.join(path, "model.safetensors"))


def _engine(path="", **kw):
    import swiftllm_b200
    from test_host_path_cpu import ENG
    return swiftllm_b200.EngineConfig(model_path=path, use_dummy=False, block_size=ENG["block_size"], gpu_mem_utilization=0.9,
                                      num_cpu_blocks=ENG["num_cpu_blocks"], max_seqs_in_block_table=ENG["max_seqs_in_block_table"],
                                      max_blocks_per_seq=ENG["max_blocks_per_seq"], max_batch_size=8, max_tokens_in_batch=256,
                                      dtype="bfloat16", **kw)


@pytest.mark.parametrize("strategy", ["channel", "tensor"])
def test_checkpoint_loads_to_the_expected_tensors(tmp_path, strategy):
    import swiftllm_b200
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG
    w = OracleWeights.random(CFG, dtype=torch.bfloat16, seed=4, std=0.08)
    fw = FO.fp8_weights(w)
    if strategy == "tensor":                 # one scale per projection: requantize every projection with its largest scale
        for lw in fw.layers:
            for n in FO.PROJECTIONS:
                f = getattr(lw, n)
                s = float(f.s.max())
                setattr(lw, n, FO.Fp8Weight((FO.dequantize(f.q, f.s) / s).float().clamp(-448, 448).to(torch.float8_e4m3fn),
                                            torch.full_like(f.s, s)))
    F = CFG["intermediate_size"]
    tensors = FO.hf_fp8_tensors(fw, F, strategy)
    # safetensors round-trips float8_e4m3fn
    _write_checkpoint(tmp_path, CFG, tensors, FO.compressed_tensors_config(strategy))
    from safetensors.torch import load_file
    back = load_file(os.path.join(tmp_path, "model.safetensors"))
    assert back["model.layers.0.mlp.down_proj.weight"].dtype == torch.float8_e4m3fn
    assert torch.equal(_bits(back["model.layers.0.mlp.down_proj.weight"]), _bits(tensors["model.layers.0.mlp.down_proj.weight"]))
    with product_on_cpu(PATCH):
        m = swiftllm_b200.LlamaModel(_engine(str(tmp_path)))
        assert m.fp8
        m.load_weights(checkpoint_getter(str(tmp_path), device="cpu"))
    for lw, ow in zip(m.weight.layers, fw.layers):
        assert lw.fp8 and lw.qkv_proj.dtype == torch.float8_e4m3fn and lw.qkv_proj_scale.dtype == torch.float32
        want_qkv = FO.Fp8Weight(torch.cat([ow.q_proj.q.view(torch.uint8), ow.k_proj.q.view(torch.uint8),
                                           ow.v_proj.q.view(torch.uint8)]).view(torch.float8_e4m3fn),
                                torch.cat([ow.q_proj.s, ow.k_proj.s, ow.v_proj.s]))
        for got, gs, want in ((lw.qkv_proj, lw.qkv_proj_scale, want_qkv), (lw.o_proj, lw.o_proj_scale, ow.o_proj),
                              (lw.up_gate_proj, lw.up_gate_proj_scale, ow.up_gate_proj),
                              (lw.down_proj, lw.down_proj_scale, ow.down_proj)):
            assert torch.equal(_bits(got), _bits(want.q)) and torch.equal(gs, want.s)
        assert lw.attn_norm.dtype == torch.bfloat16 and torch.equal(lw.attn_norm, ow.attn_norm)
    assert m.weight.lm_head.dtype == torch.bfloat16


@pytest.mark.parametrize("case", ["zero", "negative", "inf", "nan", "shape", "input_scale", "fp8-without-config"])
def test_bad_checkpoints_raise(tmp_path, case):
    import swiftllm_b200
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG
    w = OracleWeights.random(CFG, dtype=torch.bfloat16, seed=4, std=0.08)
    tensors = FO.hf_fp8_tensors(FO.fp8_weights(w), CFG["intermediate_size"])
    key = "model.layers.1.self_attn.o_proj.weight_scale"
    if case in ("zero", "negative", "inf", "nan"):
        tensors[key][3] = {"zero": 0.0, "negative": -1.0, "inf": float("inf"), "nan": float("nan")}[case]
    elif case == "shape":
        tensors[key] = tensors[key][:5]
    elif case == "input_scale":
        tensors["model.layers.0.mlp.up_proj.input_scale"] = torch.tensor([0.1])
    qc = None if case == "fp8-without-config" else FO.compressed_tensors_config()
    _write_checkpoint(tmp_path, CFG, tensors, qc)
    with product_on_cpu(PATCH), pytest.raises(ValueError, match="scale|float8_e4m3fn"):
        m = swiftllm_b200.LlamaModel(_engine(str(tmp_path)))
        m.load_weights(checkpoint_getter(str(tmp_path), device="cpu"))


@pytest.mark.parametrize("world", [2, 4])
def test_tensor_parallel_slices_equal_slices_of_the_dequantized_tensors(world):
    from swiftllm_b200.worker import fp8
    from swiftllm_b200.worker.weight import dict_getter
    g = torch.Generator().manual_seed(7)
    full = FO.Fp8Weight.of((torch.randn(64, 96, generator=g) * 0.05).to(torch.float16))
    for strategy in ("channel", "tensor"):
        s = full.s.reshape(-1, 1) if strategy == "channel" else full.s[:1]
        q = full.q if strategy == "channel" else (FO.dequantize(full.q, full.s) / float(s)).float().clamp(-448, 448).to(
            torch.float8_e4m3fn)
        deq = FO.dequantize(q, s.expand(64, 1).reshape(-1))
        get = dict_getter({"w.weight": q, "w.weight_scale": s})
        for axis in (0, 1):
            parts = [fp8.load_projection(get, "w.weight", (64, 96), axis, r, world, torch.float16, "cpu") for r in range(world)]
            for r, (pq, ps) in enumerate(parts):
                assert pq.dtype == torch.float8_e4m3fn and ps.dtype == torch.float32
                assert ps.shape == ((64 // world,) if axis == 0 else (64,))
                want = deq.chunk(world, dim=axis)[r]
                assert torch.equal(FO.dequantize(pq, ps), want)


# ---------------------------------------------------------------- the host path against the fp64 FP8 restatement
def _fp8_product(w, **kw):
    """test_host_path_cpu._product's engine in bfloat16 (FP8 engines are bfloat16 engines)."""
    import swiftllm_b200
    from swiftllm_b200.worker.weight import dict_getter
    from test_host_path_cpu import CFG, ENG, _hf_tensors
    m = swiftllm_b200.LlamaModel(_engine(**dict(dict(quantization="fp8"), **kw)), swiftllm_b200.LlamaModelConfig(CFG))
    m.load_weights(dict_getter(_hf_tensors(w, CFG["intermediate_size"])))
    m.init_kvcache_and_swap(ENG["num_blocks"])
    m.post_layer.keep_logits = True
    return m


def _bf16_oracle(w):
    from oracle.model import OracleLlama
    from test_host_path_cpu import CFG, ENG
    return OracleLlama(CFG, w, block_size=ENG["block_size"], num_blocks=ENG["num_blocks"], num_cpu_blocks=ENG["num_cpu_blocks"],
                       max_seqs_in_block_table=ENG["max_seqs_in_block_table"], max_blocks_per_seq=ENG["max_blocks_per_seq"],
                       attn="exact", dtype=torch.bfloat16)


def test_host_path_matches_the_fp8_restatement():
    """Prefill, chunked prefill, decode and a mixed batch through the product's host path with the kernel stand-ins (online
    quantization at load) against OracleLlama evaluated as the FP8 restatement in fp64.  Both quantize the same rows; the only
    difference is the GEMM's accumulation (fp32 here, fp64 there) and its rounding."""
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG
    w = OracleWeights.random(CFG, dtype=torch.bfloat16, seed=2, std=0.08)
    rng = np.random.default_rng(5)
    with product_on_cpu(PATCH):
        m = _fp8_product(w)
        assert all(lw.fp8 for lw in m.weight.layers)
        o = _bf16_oracle(FO.fp8_weights(w))
        prompts = [rng.integers(0, 300, size=n).tolist() for n in (19, 5, 40)]
        lens = [19, 5, 40]
        steps = [(prompts[:2], [0, 1], [], None), ([prompts[2][:16]], [2], [], None), ([prompts[2][16:]], [2], [], [16])]
        for ids, sids, dec, prefix in steps:
            CALLS.clear()
            tm = m.forward(ids, sids, dec, prefill_prefix_lens_list=prefix)
            with FO.fp8_model():
                to = o.forward(ids, sids, dec, prefill_prefix_lens_list=prefix)
            assert CALLS.count("linear_fp8") == 4 * CFG["num_hidden_layers"] and "linear_fp8_out" not in CALLS
            _close(m.post_layer.last_logits, o.last_logits, tm, to)
        toks = tm
        for step in range(3):
            lens = [l + 1 for l in lens]
            ids = [[19 + step], [4], [toks[0] if step == 0 else toks[-1]]]
            tm = m.forward(ids, [0, 1, 2], lens)
            with FO.fp8_model():
                to = o.forward(ids, [0, 1, 2], lens)
            _close(m.post_layer.last_logits, o.last_logits, tm, to)
            toks = tm


def _close(got, ref, tm, to):
    """A 16-bit rounding difference of a GEMM output (fp32 against fp64 accumulation) can move a downstream value across an
    e4m3 rounding boundary, a step of 2^-4 relative to that value; so the logits agree within 2^-5 of their largest magnitude, and
    the greedy tokens wherever the restatement's top-2 margin is larger than that."""
    got, ref = got.double(), ref.double()
    tol = 2.0 ** -5 * float(ref.abs().max())
    assert float((got - ref).abs().max()) <= tol
    top2 = ref.topk(2, dim=1).values
    for r, (a, b) in enumerate(zip(tm, to)):
        if float(top2[r, 0] - top2[r, 1]) > 2 * tol:
            assert a == b


def test_unquantized_engine_runs_no_fp8_code():
    """quantization=None (given or by default) without a quantization_config: 16-bit weights, no FP8 stand-in called, and the
    16-bit oracle's logits (test_host_path_cpu's tolerance) and tokens."""
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG, _oracle, _product
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=3, std=0.08)
    with product_on_cpu(PATCH):
        for kw in (dict(), dict(quantization=None)):
            m, o = _product(w, **kw), _oracle(w)
            assert not m.fp8 and all(not lw.fp8 and lw.qkv_proj.dtype == torch.float16 for lw in m.weight.layers)
            CALLS.clear()
            for args in (([[1, 2, 3], [4, 5]], [0, 1], []), None):
                if args is None:
                    args = ([[t[0]], [t[1]]], [0, 1], [4, 3])
                t = m.forward(*args)
                assert t == o.forward(*args)
                ref = o.last_logits.float()
                assert float((m.post_layer.last_logits.float() - ref).abs().max()) <= 1e-5 * float(ref.abs().max())
            assert CALLS == []


def test_graph_key_is_unchanged_by_fp8():
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG
    w = OracleWeights.random(CFG, dtype=torch.bfloat16, seed=5, std=0.08)
    with product_on_cpu(PATCH):
        keys = []
        for q in (None, "fp8"):
            m = _fp8_product(w, use_cuda_graph=True, quantization=q)
            caps = []

            def fake_capture(B, bucket, *a, **kw):
                caps.append(B)
                g = type("G", (), {"replay": lambda self: None})()
                return dict(graph=g, meta=torch.zeros((3 * B,), dtype=torch.int32), tokens=torch.zeros((B,), dtype=torch.int64),
                            logprobs=None)
            m._capture_decode_graph = fake_capture
            m.forward([[1, 2, 3], [4, 5]], [0, 1], [])
            m.forward([[1], [2]], [0, 1], [4, 3])
            keys.append(list(m._graphs))
        assert keys[0] == keys[1] and len(keys[0]) == 1


# ---------------------------------------------------------------- tensor parallelism over gloo
def _tp_worker(rank, world, port, ret, comm):
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import warnings
    import swiftllm_b200
    from cpu_shim import GlooFusedAllReduce, product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200.worker.weight import dict_getter
    from test_host_path_cpu import CFG
    cfg = dict(CFG, quantization_config=FO.compressed_tensors_config())
    w = OracleWeights.random(CFG, dtype=torch.bfloat16, seed=12, std=0.08)
    tensors = FO.hf_fp8_tensors(FO.fp8_weights(w), CFG["intermediate_size"])       # the same e4m3 weights at every world size
    extra = [("swiftllm_b200.worker.tp_comm", "FusedAllReduce", GlooFusedAllReduce)] if comm else []
    fixed = {(TL, "fused_add_rmsnorm_quant_fp8"): _add_rmsnorm_quant_fixed, (TL, "quant_fp8_rows"): _quant_rows_fixed,
             (TL, "silu_and_mul_quant_fp8"): _silu_and_mul_quant_fixed}
    patches = [(m_, a, fixed.get((m_, a), f)) for m_, a, f in PATCH] + extra
    ok, out = True, []
    with product_on_cpu(patches), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        models = []
        for tp in (world, 1):
            ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=2,
                                            max_seqs_in_block_table=8, max_blocks_per_seq=8, max_batch_size=8,
                                            max_tokens_in_batch=128, dtype="bfloat16", tp_size=tp, tp_rank=rank if tp > 1 else 0,
                                            fused_allreduce=(bool(comm) if tp > 1 else False))
            m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(cfg))
            m.load_weights(dict_getter(tensors))
            m.init_kvcache_and_swap(20)
            m.post_layer.keep_logits = True
            models.append(m)
        sharded, single = models
        ok &= (sharded.comm is not None) == bool(comm) and sharded.fp8 and single.fp8
        L = CFG["num_hidden_layers"]
        rng = np.random.default_rng(2)
        ids = [rng.integers(0, 300, size=n).tolist() for n in (21, 3)]
        sids, dec, lens = [4, 1], [], [21, 3]
        for step in range(4):
            CALLS.clear()
            got = sharded.forward(ids, sids, dec)
            # fused exchange: o and down write their partial sums into the exchange buffers, and the exchange's normalised rows
            # (every layer's ffn input, and the attention input of layers after the first) are quantized by the row quantizer;
            # all-reduce: every input but the attention output comes from add+RMSNorm+quantize
            want = ({"linear_fp8_out": 2 * L, "linear_fp8": 2 * L, "quant_rows": 3 * L - 1, "add_rmsnorm_quant": 1} if comm else
                    {"linear_fp8_out": 0, "linear_fp8": 4 * L, "quant_rows": L, "add_rmsnorm_quant": 2 * L})
            ok &= all(CALLS.count(k) == v for k, v in want.items())
            ref = single.forward(ids, sids, dec)
            g, r = sharded.post_layer.last_logits.double(), single.post_layer.last_logits.double()
            rel = float((g - r).abs().max() / r.abs().max())
            out.append((rel, got == ref))
            ok &= rel <= TP_TOL
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


# The kernels scale each row by its own amax, so the row-parallel inputs (attention output, SiLU·mul output) of a rank, quantized
# on its K slice, get other e4m3 values than the single rank's whole rows: two independent quantizations.  That per-row formula
# is the kernels' and is checked bit for bit on the GPU.  This test checks the host path under tensor parallelism, so its
# stand-ins quantize with one fixed power-of-two scale: an element's e4m3 value then does not depend on the slice it is in.
# What remains is the per-rank partial GEMM outputs rounded to bfloat16 before they are summed, which alone moves this small
# random model's logits by about 1 % in a 16-bit engine (measured), and the e4m3 rounding steps (2^-4 of a value) such
# differences cross downstream, which took the FP8 engine's difference to 4.0-5.9 %.  A wiring fault (a scale slice of the
# wrong rank, a partial sum left out) changes the logits by their own order.
TP_TOL = 2.0 ** -3
FIXED_SCALE = 2.0 ** -3         # |y| up to 56 without saturation: the activations of this model stay far below


def _fixed(y):
    s = torch.full((y.shape[0], 1), FIXED_SCALE, dtype=torch.float32)
    return (y.float() / s).clamp(-FO.E4M3_MAX, FO.E4M3_MAX).to(torch.float8_e4m3fn), s


def _add_rmsnorm_quant_fixed(x, residual, weight, eps):
    CALLS.append("add_rmsnorm_quant")
    y, r = K.fused_add_rmsnorm(x, residual, weight, eps)
    residual.copy_(r)
    return _fixed(y)


def _quant_rows_fixed(x):
    CALLS.append("quant_rows")
    return _fixed(x)


def _silu_and_mul_quant_fixed(x):
    CALLS.append("silu_and_mul_quant")
    return _fixed(K.silu_and_mul(x)[:, :x.shape[1] // 2])


@pytest.mark.parametrize("comm", [False, True], ids=["all-reduce", "fused-exchange"])
def test_tensor_parallel_fp8_logits_match_the_single_rank_engine(comm):
    """World 2 over gloo, with the FP8 kernel stand-ins (fixed-scale quantizers, see TP_TOL): the sharded FP8 engine (all-reduce of
    the FP8 GEMMs' partial outputs, or the fused exchange with the GEMM writing into its partial buffers and the exchange's rows
    quantized after it) against the single-rank FP8 engine with the same e4m3 weights: the launches each path makes, and logits
    within TP_TOL of their largest magnitude."""
    import multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_tp_worker, args=(r, 2, 29980 + int(comm), ret, comm)) for r in range(2)]
    for p in procs:
        p.start()
    out = ret.get(timeout=240)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(ok for ok, _ in out), out

