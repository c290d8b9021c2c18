"""CPU: the C-ABI library loads and exports every symbol include/swiftllm_b200.h declares (no compute calls)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "swiftllm_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(sllm_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_expected_surface():
    names = _declared()
    for n in ["sllm_rmsnorm_inplace", "sllm_fused_add_rmsnorm_inplace", "sllm_rotary_embedding_inplace",
              "sllm_silu_and_mul_inplace", "sllm_store_kvcache", "sllm_paged_attention", "sllm_prefill_attention",
              "sllm_set_block_table_and_num_seq_alloc_blocks", "sllm_unset_block_table_and_num_seq_alloc_blocks",
              "sllm_gather_allocated_blocks_and_unset", "sllm_allocate_blocks_for_seqs", "sllm_swap_blocks",
              "sllm_allreduce_add_rmsnorm"]:
        assert n in names


def test_library_exports_every_declared_symbol():
    from swiftllm_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "build with `python -m swiftllm_b200.build`"
    l = ctypes.CDLL(_lib.LIB_PATH)
    for n in _declared():
        assert hasattr(l, n), f"{n} declared in the header but not exported"
    assert set(_declared()) == set(_lib.SIGNATURES), "ctypes signature table out of sync with the header"
    assert _lib.lib().sllm_abi_version() == 1


def _prototypes():
    """name -> (return type, [parameter types]) parsed from the header, reduced to the ctypes classes of _lib.py."""
    src = open(os.path.join(ROOT, "include", "swiftllm_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for ret, name, params in re.findall(r"\b(int64_t|int|const char\*)\s+(sllm_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src):
        kinds = []
        for prm in [x.strip() for x in params.split(",") if x.strip() and x.strip() != "void"]:
            if "*" in prm or prm.startswith("sllm_stream_t"):
                kinds.append("ptr")
            elif prm.startswith("int64_t"):
                kinds.append("i64")
            elif prm.startswith("float"):
                kinds.append("f32")
            elif prm.startswith(("int ", "sllm_dtype_t")):
                kinds.append("i32")
            else:
                raise AssertionError(f"unparsed parameter {prm!r} of {name}")
        out[name] = ({"int": "i32", "int64_t": "i64", "const char*": "str"}[ret], kinds)
    return out


def test_ctypes_signatures_match_the_header_type_by_type():
    """A ctypes table that drifts from the header corrupts arguments silently (an int64 passed as int truncates, a
    missing parameter shifts every later one): compare every prototype with _lib.SIGNATURES."""
    from ctypes import c_char_p, c_float, c_int, c_int64, c_void_p
    from swiftllm_b200 import _lib
    kind = {c_void_p: "ptr", c_int: "i32", c_int64: "i64", c_float: "f32", c_char_p: "str"}
    protos = _prototypes()
    assert set(protos) == set(_lib.SIGNATURES)
    for name, (ret, params) in protos.items():
        res, args = _lib.SIGNATURES[name]
        assert kind[res] == ret, f"{name}: return type {kind[res]} != header {ret}"
        assert [kind[a] for a in args] == params, f"{name}: ctypes argtypes differ from the header"


def test_invalid_arguments_are_rejected_before_launch():
    """Shape validation runs on the host and needs no GPU (the reference raises AssertionError here)."""
    from swiftllm_b200 import _lib
    l = _lib.lib()
    assert l.sllm_rmsnorm_inplace(None, None, 1e-5, 4, 12, 0, None) != 0         # hidden % 8 != 0
    assert b"multiple of 8" in l.sllm_last_error()
    assert l.sllm_paged_attention(1, 1, 1, 1, 1, 1, 1, None, 0, 1.0, 1, 16, 0, 0, 1, 4, 2, 16, 96, 4, 4, 4 * 96, 0, None) != 0
    assert b"head_dim" in l.sllm_last_error()
    assert l.sllm_silu_and_mul_inplace(None, 0, 256, 7, None) == 0              # empty batch is a no-op
    assert l.sllm_prefill_attention_paged(1, 1, 1, 1, 1, 1, 1, 1, 1, 1.0, 1, 8, 8, 0, 1, 4, 2, 16, 96, 4, 4, 4 * 96, 0, None) != 0
    assert b"head_dim" in l.sllm_last_error()
    assert l.sllm_store_kvcache_chunked(1, 1, 1, 1, 1, 1, 1, 1, None, None, 1, 0, 8, 8, 0, 1, 2, 16, 64, 4, 128, 128, 0, None) != 0
    assert b"prefill_prefix_lens" in l.sllm_last_error()
    assert l.sllm_swap_blocks(None, None, 0, 1, None, None, None, None, 16, None) == 0


def test_no_silent_fallback_without_cuda():
    import pytest
    import torch
    from swiftllm_b200.worker.kernels.rmsnorm import rmsnorm_inplace
    if torch.cuda.is_available():
        pytest.skip("CPU-only check")
    x = torch.zeros(2, 64, dtype=torch.float16)
    with pytest.raises(RuntimeError, match="no CPU path"):
        rmsnorm_inplace(x, torch.ones(64, dtype=torch.float16), 1e-5)


def test_validated_kernels_still_have_their_validated_instruction_streams():
    """profiles/validated_kernels.json holds a hash of the (normalised) SASS of every kernel as it last ran `pytest -m gpu`,
    smoke() and bench.py on an H100.  Refactoring a kernel's source without a GPU at hand (templates, shared headers) is only safe
    if the instruction stream it compiles to is unchanged - or the change was reviewed and listed under "equivalent".  A kernel that
    no longer matches must be re-validated on a GPU and the manifest regenerated (scripts/sass_diff.py)."""
    import hashlib
    import importlib.util
    import json
    import shutil
    import subprocess
    import pytest
    if shutil.which("cuobjdump") is None or shutil.which("nvcc") is None:
        pytest.skip("CUDA toolkit not on PATH")
    path = os.path.join(ROOT, "profiles", "validated_kernels.json")
    man = json.load(open(path))
    nvcc = subprocess.run(["nvcc", "--version"], capture_output=True, text=True).stdout
    if man["nvcc"] not in nvcc:
        pytest.skip("different nvcc than the one the manifest was made with")
    spec = importlib.util.spec_from_file_location("sass_diff", os.path.join(ROOT, "scripts", "sass_diff.py"))
    sd = importlib.util.module_from_spec(spec); spec.loader.exec_module(sd)
    have = {hashlib.sha256("\n".join(sd.norm(body)).encode()).hexdigest() for body in sd.kernels().values()}
    assert have, "no objects under swiftllm_b200/csrc/build: run python -m swiftllm_b200.build"
    changed = [name for name, k in man["kernels"].items()
               if k["sha256"] not in have and man["equivalent"].get(name, {}).get("sha256") not in have]
    assert not changed, f"validated kernels whose SASS changed (re-validate on a GPU): {changed}"


def test_product_never_imports_the_oracle_or_reads_the_reference():
    """The oracle is test infrastructure: only tests/, __graft_entry__.smoke() and bench.py's CPU arms may import it; nothing that
    ships may read /root/reference or baseline/_ref (scripts/ref_triton_bench.py and install_reference.sh exist FOR the reference)."""
    offenders = []
    for base in ("swiftllm_b200", "examples"):
        for d, _, files in os.walk(os.path.join(ROOT, base)):
            for f in files:
                if not f.endswith((".py", ".cu", ".cuh", ".h")):
                    continue
                txt = open(os.path.join(d, f), encoding="utf-8").read()
                if re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M) or "/root/reference" in txt or "baseline/_ref" in txt:
                    offenders.append(os.path.relpath(os.path.join(d, f), ROOT))
    assert not offenders, offenders
    # bench.py: the oracle is imported in exactly two places - the CPU arm (cpu_baseline / --impl reference) and the CHECKER that
    # compares sampled attention rows / sequences of the GPU result with it outside every timed region (parity_check)
    import ast
    src = open(os.path.join(ROOT, "bench.py"), encoding="utf-8").read()
    assert "/root/reference" not in src
    where = set()
    for fn in ast.walk(ast.parse(src)):
        if isinstance(fn, ast.FunctionDef):
            for node in ast.walk(fn):
                if isinstance(node, ast.ImportFrom) and (node.module or "").split(".")[0] == "oracle":
                    where.add(fn.name)
                if isinstance(node, ast.Import) and any(a.name.split(".")[0] == "oracle" for a in node.names):
                    where.add(fn.name)
    assert where == {"cpu_decode_sample", "parity_check"}, where
