"""CPU: tests/kv_geometry.py against the sources it restates (csrc/kvcache.cu, csrc/swap_gather.cu, csrc/rotary_store.cu,
csrc/allreduce_ll.cu's own row limit, and the one rule every launcher follows for the 48 KB shared-memory default), its static
shared memory against what ptxas reports for the kernels, and the case tables tests/test_kv_block_kernels_gpu.py runs."""
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import kv_geometry as KG

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "swiftllm_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")
# the source of each kernel whose launcher can cross 48 KB of dynamic shared memory
KERNEL_SOURCES = {"allocate_blocks_kernel": "kvcache.cu", "allreduce_add_rmsnorm_kernel": "allreduce_norm.cu",
                  "allreduce_add_rmsnorm_2shot_kernel": "allreduce_norm.cu", "allreduce_add_rmsnorm_ll_kernel": "allreduce_ll.cu",
                  "rmsnorm_kernel": "elementwise.cu", "rmsnorm_kernel<QUANT>": "elementwise.cu",
                  "silu_and_mul_quant_kernel": "fp8.cu"}


def _one(pattern: str, text: str, what: str):
    found = re.findall(pattern, text, re.S)
    assert len(found) == 1, f"{what}: expected one match of {pattern!r}, found {len(found)}"
    return found[0]


def limit_rule_breaches(csrc: str) -> list:
    """The one shared-memory limit rule: the attribute is set only by raise_dynamic_smem (host.cu), which takes the kernel's
    static size from the compiled kernel; no launcher sets it, counts static shared memory or keeps a flag of its own."""
    texts = {f: open(os.path.join(csrc, f)).read() for f in sorted(os.listdir(csrc)) if f.endswith((".cu", ".cuh"))}
    bad = []
    sets = {f: t.count("cudaFuncAttributeMaxDynamicSharedMemorySize") for f, t in texts.items()}
    if {f: n for f, n in sets.items() if n} != {"host.cu": 1}:
        bad.append(("the attribute is set outside raise_dynamic_smem", sets))
    if any("first_use_on_this_device" in t for t in texts.values()):
        bad.append("first_use_on_this_device")
    if re.findall(r"\bsmem\b[^;\n]*[<>]=? 48 \* 1024", "".join(texts.values())):
        bad.append("a launcher's own 48 KB test")
    try:
        _one(r"e = cudaFuncGetAttributes\(&fa, kernel\);\s*limit = 48 \* 1024 - \(int\)fa\.sharedSizeBytes;", texts["host.cu"],
             "static size of the compiled kernel")
    except AssertionError as e:
        bad.append(str(e))
    return bad


def mismatches(csrc: str) -> list:
    read = lambda f: open(os.path.join(csrc, f)).read()
    kv, sw, rs, ll = read("kvcache.cu"), read("swap_gather.cu"), read("rotary_store.cu"), read("allreduce_ll.cu")
    bad = limit_rule_breaches(csrc)
    try:
        # allocator: shared-memory size, refusal, block shape, windows
        _one(r"const size_t smem = \(size_t\)\(2 \* batch \+ 1\) \* sizeof\(int32_t\);", kv, "allocator smem")
        if int(_one(r"SLLM_REQUIRE\(smem <= (\d+) \* 1024, \"allocate_blocks: batch", kv, "allocator cap")) * 1024 != KG.ALLOC_SMEM_MAX:
            bad.append("allocator cap")
        if int(_one(r"allocate_blocks_kernel<<<1, (\d+), smem,", kv, "allocator launch")) != KG.ALLOC_THREADS:
            bad.append("allocator threads")
        if int(_one(r"__launch_bounds__\((\d+)\) allocate_blocks_kernel", kv, "allocator bounds")) != KG.ALLOC_THREADS:
            bad.append("allocator bounds")
        if int(_one(r"const int64_t per_iter = \(int64_t\)blockDim\.x \* (\d+);", kv, "window")) * KG.ALLOC_THREADS != KG.ALLOC_WINDOW:
            bad.append("window")
        flags = dict((int(v), c) for c, v in re.findall(r"if \(([^)]*?)\) atomicOr\(&s_err, (\d)\);", kv))
        flags[1] = _one(r"if \((free_cnt < total) && threadIdx\.x == 0\) s_err \|= 1;", kv, "flag 1")
        flags[8] = _one(r"\(\((new_out != nullptr && total > cap)\) \? 8 : 0\)", kv, "flag 8")
        if flags != {2: "h > tgt", 4: "tgt > mbps", 1: "free_cnt < total", 8: "new_out != nullptr && total > cap"}:
            bad.append(("status flags", flags))
        # tail copy
        t, u = _one(r"constexpr int kTailThreads = (\d+), kTailUnroll = (\d+), kTailChunk = kTailThreads \* kTailUnroll \* 16;",
                    kv, "tail constants")
        if (int(t), int(u)) != (KG.TAIL_THREADS, KG.TAIL_UNROLL):
            bad.append(("tail", t, u))
        _one(r"dim3 grid\(cdiv\(block_bytes, kTailChunk\), batch, 2\);", kv, "tail grid")
        # swap
        if (int(_one(r"constexpr int SW_SPLIT = (\d+);", sw, "SW_SPLIT")), int(_one(r"constexpr int SW_THREADS = (\d+);", sw,
                                                                                     "SW_THREADS"))) != (KG.SW_SPLIT, KG.SW_THREADS):
            bad.append("swap constants")
        _one(r"const int64_t per = \(block_vecs \+ SW_SPLIT - 1\) / SW_SPLIT;", sw, "swap slice")
        _one(r"i < hi; i \+= 2 \* SW_THREADS\) \{\s*const int64_t j = i \+ SW_THREADS;", sw, "swap second access")
        _one(r"dim3 grid\(\(unsigned\)n, SW_SPLIT\);", sw, "swap grid")
        # stores
        _one(r"dim3 grid\(cdiv\(max_prefill_len, block_size\) \+ 1, num_prefill_seqs\);", kv, "chunked grid")
        _one(r"dim3 grid\(cdiv\(max_prefill_len, block_size\), num_prefill_seqs\);", kv, "prefill grid")
        if re.findall(r"store_kv_prefill_kernel<T, (?:true|false)><<<grid, (\d+), 0, stream>>>", kv) != [str(KG.PREFILL_THREADS)] * 2:
            bad.append("prefill threads")
        if int(_one(r"store_kv_decode_kernel<T><<<num_decoding_seqs, (\d+), 0, stream>>>", kv, "decode")) != KG.DECODE_THREADS:
            bad.append("decode threads")
        _one(r"const int64_t total = \(int64_t\)num_decoding_seqs \* \(num_q_heads \+ 2 \* num_kv_heads\) \* \(head_dim / 16\);", rs,
             "rotary_store items")
        if int(_one(r"const int threads = (\d+);", rs, "rotary_store threads")) != KG.ROTARY_STORE_THREADS:
            bad.append("rotary_store threads")
        # the LL kernel's own limit
        ll_max = int(_one(r"SLLM_REQUIRE\(\(size_t\)\(hidden / 8\) \* sizeof\(uint4\) <= (\d+) \* 1024, \"allreduce\(LL\)", ll, "LL"))
        if ll_max * 1024 // 16 * 8 != KG.LL_MAX_HIDDEN:
            bad.append(("LL limit", ll_max))
    except AssertionError as e:          # a statement the patterns no longer find
        return [str(e)]
    return bad


def test_the_mirror_states_the_sources():
    assert mismatches(CSRC) == []


@pytest.mark.parametrize("edit", [
    ("kvcache.cu", "    if (int e = fit_dynamic_smem<allocate_blocks_kernel>(smem, \"allocate_blocks_for_seqs\")) return e;\n",
     "    if (smem + 144 > 48 * 1024) cudaFuncSetAttribute(allocate_blocks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);\n"),
    ("exchange.cuh", "if (int e = dtype == SLLM_F16 ? fit_dynamic_smem<F16>(smem, kernel) : fit_dynamic_smem<BF16>(smem, kernel)) return e;",
     "if (smem + 80 > 48 * 1024) cudaFuncSetAttribute(F16, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);"),
    ("elementwise.cu", "if (int e = fit_dynamic_smem<rmsnorm_kernel<T, FUSED, 0, QUANT>>(smem, what)) return e;",
     "if (smem + 64 > 48 * 1024) return 1;"),
    ("fp8.cu", "if (int e = fit_dynamic_smem<silu_and_mul_quant_kernel<T>>(smem, \"silu_and_mul_quant_fp8\")) return e;",
     "if (smem + 16 * sizeof(float) > 48 * 1024) return 1;"),
    ("prompt_logprobs.cu", "    const int stage_vecs", "    static unsigned long long configured = 0;\n"
     "    if (first_use_on_this_device(configured)) {}\n    const int stage_vecs"),
    ("host.cu", "limit = 48 * 1024 - (int)fa.sharedSizeBytes;", "limit = 48 * 1024 - 64;"),
    ("kvcache.cu", "smem <= 200 * 1024", "smem <= 220 * 1024"),
    ("kvcache.cu", "(int64_t)blockDim.x * 16;", "(int64_t)blockDim.x * 32;"),
    ("kvcache.cu", "if (tgt > mbps) atomicOr(&s_err, 4);", "if (tgt >= mbps) atomicOr(&s_err, 4);"),
    ("kvcache.cu", "kTailUnroll = 8,", "kTailUnroll = 4,"),
    ("swap_gather.cu", "SW_SPLIT = 8;", "SW_SPLIT = 4;"),
    ("swap_gather.cu", "const int64_t j = i + SW_THREADS;", "const int64_t j = i + 2 * SW_THREADS;"),
    ("rotary_store.cu", "const int threads = 256;", "const int threads = 128;"),
    ("allreduce_ll.cu", "sizeof(uint4) <= 48 * 1024", "sizeof(uint4) <= 56 * 1024")],
    ids=["alloc-own-limit", "exchange-own-limit", "rmsnorm-own-limit", "fp8-own-limit", "first-use", "hand-counted-static",
         "alloc-cap", "alloc-window", "alloc-flag4", "tail-unroll", "swap-split", "swap-second", "rotary-threads", "ll-limit"])
def test_a_changed_source_is_noticed(tmp_path, edit):
    f, old, new = edit
    for name in os.listdir(CSRC):
        if name.endswith((".cu", ".cuh")):
            shutil.copy(os.path.join(CSRC, name), tmp_path / name)
    text = (tmp_path / f).read_text()
    assert text.count(old) == 1
    (tmp_path / f).write_text(text.replace(old, new))
    assert mismatches(str(tmp_path)) != []


def _mangled(kernel: str) -> str:
    """Pattern of the mangled names of a KERNEL_SOURCES entry's instances: rmsnorm_kernel's last template argument (QUANT)
    tells its quantizing instances from the others."""
    if kernel.startswith("rmsnorm_kernel"):
        return r"\drmsnorm_kernelI\w*?Lb%dEEEv" % kernel.endswith("<QUANT>")
    return r"\d" + kernel


def static_smem_of_cubins(csrc: str, out_dir) -> dict:
    """kernel name -> set of static shared-memory sizes (SHARED minus the 1 KB system reserve) of its instances, from
    `cuobjdump -res-usage` of each source compiled for sm_90a."""
    files = sorted(set(KERNEL_SOURCES.values()))

    def compile_one(f):
        cubin = os.path.join(str(out_dir), f + ".cubin")
        subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-cubin",
                        "-o", cubin, os.path.join(csrc, f)], check=True, capture_output=True)
        return subprocess.run([CUOBJDUMP, "-res-usage", cubin], check=True, capture_output=True, text=True).stdout

    with ThreadPoolExecutor(max_workers=len(files)) as ex:
        dumps = dict(zip(files, ex.map(compile_one, files)))
    sizes = {}
    for kernel, f in KERNEL_SOURCES.items():
        found = re.findall(r"Function (\S*?" + _mangled(kernel) + r"\S*):\s*\n\s*REG:\d+ STACK:\d+ SHARED:(\d+) ", dumps[f])
        assert found, f"{kernel} not in the cubin of {f}"
        sizes[kernel] = {int(s) - 1024 for _, s in found}
    return sizes


@pytest.mark.skipif(not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)), reason="needs nvcc and cuobjdump")
def test_the_static_shared_memory_is_what_ptxas_reports(tmp_path):
    """STATIC_SMEM puts the GPU tests' edge cases (the allocator's B6126-edge ... B6143, the exchange widths 24544 ... 24576,
    the rows of tests/row_geometry.py) exactly where the launchers start to raise the limit."""
    sizes = static_smem_of_cubins(CSRC, tmp_path)
    assert sizes == {k: {v} for k, v in KG.STATIC_SMEM.items()}, sizes


def test_the_allocator_bands():
    assert [b for b in range(1, 26000) if KG.alloc_needs_raise(b) and KG.alloc_band(b) == "default"] == []
    edge = [b for b in range(1, 26000) if KG.alloc_needs_raise(b) and KG.alloc_smem(b) <= KG.SMEM_DEFAULT]
    assert (edge[0], edge[-1], len(edge)) == (6126, 6143, 18)
    assert KG.MAX_ALLOC_BATCH == 25599 and KG.alloc_band(25600) == "refused"
    from swiftllm_b200.worker.kernels.block_mgmt import MAX_ALLOCATE_BATCH
    assert MAX_ALLOCATE_BATCH == KG.MAX_ALLOC_BATCH


def test_the_exchange_bands():
    """The widths that needed the raised limit but did not get it, per kernel, and the LL limit."""
    band = lambda k: [H for H in range(8, 65537, 8) if KG.exchange_needs_raise(H, k) and (H // 8) * 16 <= KG.SMEM_DEFAULT]
    assert band("allreduce_add_rmsnorm_kernel") == band("allreduce_add_rmsnorm_ll_kernel") == list(range(24552, 24577, 8))
    assert band("allreduce_add_rmsnorm_2shot_kernel") == list(range(24544, 24577, 8))
    assert KG.LL_MAX_HIDDEN == 24576


def test_the_case_tables_cover_every_regime():
    ids = [KG.batch_id(b) for b in KG.ALLOC_BATCHES]
    assert ids[:3] == ["B1-1pass", "B31-1pass", "B32-1pass"] and "B6126-edge" in ids and "B6143-edge" in ids
    assert KG.batch_id(6125) == "B6125-1pass".replace("1pass", f"{KG.scan_passes(6125)}pass") and KG.batch_id(6144) == "B6144-raised"
    assert {KG.scan_passes(b) for b in KG.ALLOC_BATCHES} >= {1, 2, 3}
    assert ids[-1] == "B25599-raised"
    # every batch in the edge band runs before any batch above 12288 (the limit, once raised, stays raised for the process)
    first_big = next(i for i, b in enumerate(KG.ALLOC_BATCHES) if b > 12288)
    assert all(i < first_big for i, b in enumerate(KG.ALLOC_BATCHES) if 6126 <= b <= 6143)
    assert KG.free_map_id((3 * KG.ALLOC_WINDOW + 5, "odd")) == "N49157-odd-W4-window"
    # pages: 32 tail chunks and the second swap access on the 1 MiB page, short last slices on the others
    sizes = {pid: 2 * int(np.prod(shape)) for shape, pid in KG.PAGES}
    assert sizes["P1MiB-32chunks"] == 1 << 20 and KG.tail_chunks(1 << 20) == 32 and KG.swap_second_access(1 << 20)
    assert KG.swap_slices(sizes["P65584B-short-slice"]) == [513] * 7 + [508]
    assert KG.swap_second_access(sizes["P65584B-short-slice"])
    assert KG.swap_slices(sizes["P208B-short-slice"]) == [2] * 6 + [1, 0]
    # a prefill page of 128 tokens x 8 kv heads x 16 vectors: 16384 items on 256 threads
    assert KG.prefill_items(128, 8, 128) == 16384 > KG.PREFILL_THREADS


def test_block_manager_refuses_a_batch_the_allocator_refuses_before_reserving():
    from swiftllm_b200.worker.block_manager import BlockManager
    bm = BlockManager("cpu", 60000, KG.MAX_ALLOC_BATCH + 1, 4, 16, device="cpu")
    sids = list(range(KG.MAX_ALLOC_BATCH + 1))
    with pytest.raises(RuntimeError, match="at most 25599"):
        bm.reserve_blocks_for_seqs(sids, [1] * len(sids))
    assert bm.num_free_blocks == 60000 and not bm._host_nsab.any()
    assert bm.reserve_blocks_for_seqs(sids[:-1], [17] * (len(sids) - 1)) == 2 * KG.MAX_ALLOC_BATCH
