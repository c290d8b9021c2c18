"""Times the UNMODIFIED reference (swiftLLM, placed under baseline/_ref/src by scripts/install_reference.sh; git-ignored) on the GPU:
its own Triton kernels + cuBLAS, BASELINE config 2 (Llama-3-8B shapes, pure decode, batch 256, seq_len 4096) through its
own public API (`LlamaModel.forward`: host lists in, host ints out - the same call bench.py's `e2e` leg makes).
bench.py runs this as a subprocess (N = 1, before it allocates its own model) and reports the result as `reference_triton`;
the contract's `--impl reference` arm stays the CPU port.  Prints one JSON line: decode step time, tokens/s and the time of
its paged_attention (phase 1 + 2, CUDA events on the stream the reference launches it on).

REF_DTYPE=fp16 (default): the tree exactly as shipped (it hard-codes fp16, SURVEY.md "Facts").
REF_DTYPE=bf16: a throw-away COPY of the tree (temp dir, never written back) in which the fp16 literals SURVEY.md lists
(`torch.float16` / `tl.float16` in swiftllm/**.py) are replaced by their bf16 counterparts - the "dtype-patched reference"
BASELINE's bf16 metric needs; nothing else is changed."""
import json, os, re, shutil, statistics, sys, tempfile, types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "baseline", "_ref", "src")
if not os.path.isdir(os.path.join(REF, "swiftllm", "worker")):
    print(json.dumps({"impl": "reference-triton", "unavailable": "baseline/_ref/src missing: run scripts/install_reference.sh"})); sys.exit(0)
DTYPE = os.environ.get("REF_DTYPE", "fp16")
assert DTYPE in ("fp16", "bf16")
SRC = REF
if DTYPE == "bf16":
    SRC = os.path.join(tempfile.mkdtemp(prefix="ref_bf16_"), "src")
    shutil.copytree(os.path.join(REF, "swiftllm"), os.path.join(SRC, "swiftllm"))
    npatched = 0
    for d, _, fs in os.walk(os.path.join(SRC, "swiftllm")):
        for f in fs:
            if f.endswith(".py"):
                p = os.path.join(d, f); t = open(p).read()
                t2 = re.sub(r"\b(torch|tl)\.float16\b", r"\1.bfloat16", t)
                if t2 != t:
                    npatched += t.count(".float16"); open(p, "w").write(t2)
    assert npatched >= 10, npatched
# Triton JIT cache.  The reference's phase-1 kernel unrolls seq_block_size / block_size = 128 pages (tl.static_range,
# paged_attn.py:88) and is specialised three times on cur_layer: ~8 minutes of ptxas on a cold cache.  A cache built
# once may be kept under baseline/_ref/triton_cache/<dtype> (git-ignored): the UNMODIFIED kernels, compiled by the same
# Triton, only not recompiled.  REF_TRITON_CACHE_DIR overrides the location.
cache = os.environ.get("REF_TRITON_CACHE_DIR") or os.path.join(ROOT, "baseline", "_ref", "triton_cache", DTYPE)
packed = os.path.join(ROOT, "baseline", "_ref", f"triton_cache_{DTYPE}.tar.gz")     # how the cache travels (it compresses 8x)
if not os.environ.get("REF_TRITON_CACHE_DIR") and not os.path.isdir(cache) and os.path.exists(packed):
    import tarfile
    os.makedirs(os.path.dirname(cache), exist_ok=True)
    with tarfile.open(packed) as tf:
        tf.extractall(os.path.dirname(cache))
    # Triton's group files list their children by ABSOLUTE path (triton/runtime/cache.py: get_group drops children that do not
    # exist, which turns every lookup into a miss after the cache has moved): point them at where the files are now
    for d, _, fs in os.walk(cache):
        for f in fs:
            if f.startswith("__grp__") and f.endswith(".json"):
                gp = os.path.join(d, f)
                grp = json.load(open(gp))
                grp["child_paths"] = {c: os.path.join(d, os.path.basename(pth)) for c, pth in grp.get("child_paths", {}).items()}
                json.dump(grp, open(gp, "w"))
os.makedirs(cache, exist_ok=True)
os.environ["TRITON_CACHE_DIR"] = cache
sys.path.insert(0, SRC)
sys.path.insert(0, os.path.join(REF, "csrc"))          # swiftllm_c built in place (the reference's `pip install -e csrc`)
import torch
ray = types.ModuleType("ray"); ray.remote = lambda cls: cls; sys.modules["ray"] = ray
try:
    import flash_attn
    sys.modules["vllm_flash_attn"] = flash_attn
except Exception:
    m = types.ModuleType("vllm_flash_attn"); m.flash_attn_varlen_func = None; sys.modules["vllm_flash_attn"] = m
import swiftllm
from swiftllm.worker.layers import transformer_layer as TL

B = int(os.environ.get("REF_BATCH", 256)); S = int(os.environ.get("REF_SEQLEN", 4096)); STEPS = int(os.environ.get("REF_STEPS", 10))
cfg = dict(model_type="llama", num_hidden_layers=32, num_attention_heads=32, num_key_value_heads=8, hidden_size=4096,
           intermediate_size=14336, vocab_size=128256, max_position_embeddings=8192, rope_theta=500000.0, rms_norm_eps=1e-5,
           hidden_act="silu")
tmp = tempfile.mkdtemp(); json.dump(cfg, open(os.path.join(tmp, "config.json"), "w"))
ec = swiftllm.EngineConfig(model_path=tmp, use_dummy=True, block_size=16, gpu_mem_utilization=0.97, num_cpu_blocks=1,
                           max_seqs_in_block_table=B, max_blocks_per_seq=S // 16 + 8, max_batch_size=B, max_tokens_in_batch=8192)
model = swiftllm.LlamaModel(ec)
model.load_weights()
nblk = B * (S // 16) + 64
model.init_kvcache_and_swap(nblk)
with torch.inference_mode():
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    ch = max(1, nblk // 64)
    for s in range(0, nblk, ch):
        model.k_cache[s:s + ch].normal_(generator=g); model.v_cache[s:s + ch].normal_(generator=g)
events = []
orig = TL.paged_attention
def timed_paged(*a, **k):
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record(); orig(*a, **k); e1.record(); events.append((e0, e1))
TL.paged_attention = timed_paged
ids = [[1]] * B; sids = list(range(B)); lens = [S] * B
WARMUP = int(os.environ.get("REF_WARMUP", 3))
import time as _time
_t = _time.perf_counter()
ids = [[t] for t in model.forward(ids, sids, lens)]          # first call: Triton JIT (or cache hits) for every kernel
first_forward_s = round(_time.perf_counter() - _t, 1)
for _ in range(WARMUP):
    ids = [[t] for t in model.forward(ids, sids, lens)]      # sampled tokens fed back, like bench.py's e2e leg
events.clear()
torch.cuda.synchronize()
t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
t0.record()
for _ in range(STEPS):
    ids = [[t] for t in model.forward(ids, sids, lens)]
t1.record(); torch.cuda.synchronize()
ms = t0.elapsed_time(t1) / STEPS
pa = statistics.mean(a.elapsed_time(b) for a, b in events)
alg = B * S * 8 * 128 * 2 * 2 + 2 * B * 32 * 128 * 2
print(json.dumps({"impl": "reference-triton", "dtype": "fp16 (as shipped)" if DTYPE == "fp16" else "bf16 (fp16 literals patched in a temp copy)",
                  "kv_cache_dtype": str(model.k_cache.dtype), "seq_block_size_heuristic": "reference (model.py:305-324)", "metric": "decode_tokens_per_s", "value": B / (ms * 1e-3),
                  "ms_per_step": ms, "paged_attention_ms_per_layer": pa, "paged_attention_GBps_algorithmic": alg / (pa * 1e-3) / 1e9,
                  "triton_cache_dir": os.path.relpath(cache, ROOT), "first_forward_s": first_forward_s,
                  "batch": B, "seq_len": S, "steps": STEPS, "warmup": WARMUP, "triton": __import__("triton").__version__, "torch": torch.__version__}))
