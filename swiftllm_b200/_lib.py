"""ctypes binding of libswiftllm_b200.so (the C ABI declared in include/swiftllm_b200.h).

There is NO fallback: if the library is missing or the device is not sm_90 every kernel wrapper raises.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# SLLM_LIB_PATH: a development variant of the library (python -m swiftllm_b200.build with SLLM_BUILD_VARIANT); never set by tests / bench
LIB_PATH = os.environ.get("SLLM_LIB_PATH") or os.path.join(_HERE, "libswiftllm_b200.so")

F16, BF16 = 0, 1

_P, _I, _L, _F = c_void_p, c_int, c_int64, c_float

# name -> (restype, argtypes); must list every function of include/swiftllm_b200.h
SIGNATURES = {
    "sllm_abi_version": (_I, []),
    "sllm_last_error": (c_char_p, []),
    "sllm_device_check": (_I, [_I]),
    "sllm_rmsnorm_inplace": (_I, [_P, _P, _F, _L, _I, _I, _P]),
    "sllm_fused_add_rmsnorm_inplace": (_I, [_P, _P, _P, _F, _L, _I, _I, _P]),
    "sllm_rotary_embedding_inplace": (_I, [_P, _P, _P, _P, _L, _I, _I, _I, _L, _L, _I, _P]),
    "sllm_silu_and_mul_inplace": (_I, [_P, _L, _L, _I, _P]),
    "sllm_store_kvcache": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _L, _I, _I, _I, _I, _I, _I, _I, _L, _L, _I, _P]),
    "sllm_rotary_store_kvcache_decode": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _L, _L, _L, _I, _P]),
    "sllm_paged_attention_workspace_bytes": (_L, [_I, _I, _I, _I, _I, _I]),
    "sllm_paged_attention": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _L, _F, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _L, _L, _I, _P]),
    "sllm_prefill_attention": (_I, [_P, _P, _P, _P, _P, _P, _F, _I, _I, _L, _I, _I, _I, _L, _L, _L, _I, _P]),
    "sllm_store_kvcache_chunked": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _L, _I, _I, _I, _I, _I, _I, _I, _L, _L, _I, _P]),
    "sllm_prefill_attention_paged": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _F, _I, _I, _L, _I, _I, _I, _I, _I, _I, _I, _L, _L, _I, _P]),
    "sllm_paged_attention_verify_workspace_bytes": (_L, [_I, _L, _I, _I, _I, _I]),
    "sllm_paged_attention_verify": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _L, _F, _I, _I, _I, _L, _I, _I, _I, _I, _I, _I, _I,
                                         _L, _L, _I, _P]),
    "sllm_paged_attention_kv_map_rank": (_I, []),
    "sllm_set_block_table_and_num_seq_alloc_blocks": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _P]),
    "sllm_truncate_blocks_for_seqs": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "sllm_unset_block_table_and_num_seq_alloc_blocks": (_I, [_P, _P, _P, _P, _I, _I, _P]),
    "sllm_gather_allocated_blocks_and_unset": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _P]),
    "sllm_allocate_blocks_for_seqs": (_I, [_P, _P, _P, _P, _P, _I, _I, _L, _I, _P, _L, _P, _P]),
    "sllm_fork_blocks_for_seqs": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "sllm_copy_block_tails": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _L, _I, _I, _P]),
    "sllm_release_blocks_for_seqs": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _P]),
    "sllm_allreduce_add_rmsnorm": (_I, [_P, _P, _I, _I, _I, _P, _P, _P, _P, _F, _L, _I, _I, _P]),
    "sllm_allreduce_add_rmsnorm_2shot": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _F, _L, _I, _I, _P]),
    "sllm_allreduce_add_rmsnorm_ll": (_I, [_P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _F, _L, _I, _L, _I, _P]),
    "sllm_swap_blocks": (_I, [_P, _P, _L, _I, _P, _P, _P, _P, _L, _P]),
    "sllm_swap_blocks_gathered": (_I, [_P, _P, _L, _I, _P, _P, _P, _P, _L, _P]),
    "sllm_sample_tokens": (_I, [_P, _L, _I, _L, _L, _P, _P, _P, _P, _P, _P, _P, _I, _P]),
    "sllm_sample_tokens_truncated": (_I, [_P, _L, _I, _L, _L, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P]),
    "sllm_token_logprobs": (_I, [_P, _L, _I, _L, _P, _I, _P, _P, _P, _I, _P]),
    "sllm_prompt_logprobs": (_I, [_P, _L, _I, _L, _P, _I, _P, _P, _P, _P, _I, _P]),
    "sllm_apply_penalties": (_I, [_P, _L, _I, _L, _L, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _I, _I, _P, _L, _I, _P]),
    "sllm_apply_penalties_ngram": (_I, [_P, _L, _I, _L, _L, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _I, _I, _P, _L, _P, _P, _P, _P,
                                        _P, _I, _P]),
    "sllm_constrain_logits": (_I, [_P, _L, _I, _L, _L, _P, _P, _L, _I, _P, _P, _L, _P, _P, _L, _I, _P]),
    "sllm_lora_shrink": (_I, [_P, _L, _L, _I, _P, _L, _P, _L, _I, _P, _L, _P, _I, _I, _P]),
    "sllm_lora_expand": (_I, [_P, _L, _L, _I, _P, _L, _P, _L, _I, _I, _I, _P, _L, _P, _P, _I, _I, _P]),
    "sllm_fused_add_rmsnorm_quant_fp8": (_I, [_P, _P, _P, _F, _L, _I, _P, _P, _I, _P]),
    "sllm_silu_and_mul_quant_fp8": (_I, [_P, _L, _L, _L, _P, _P, _I, _P]),
    "sllm_quant_fp8_rows": (_I, [_P, _L, _L, _L, _P, _P, _I, _P]),
}

_lib = None


class NativeLibraryError(RuntimeError):
    pass


def lib() -> ctypes.CDLL:
    """Load (once) and return the native library; raises loudly when it is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeLibraryError(
                f"{LIB_PATH} not found: build it with `python -m swiftllm_b200.build` (nvcc, sm_90a). "
                "swiftllm_b200 has no CPU or PyTorch fallback path.")
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)          # AttributeError if the symbol is missing
            fn.restype = res
            fn.argtypes = args
        if l.sllm_abi_version() != 1:
            raise NativeLibraryError("ABI version mismatch between _lib.py and libswiftllm_b200.so")
        _lib = l
    return _lib


# number of native calls that enqueue device work since import (bench.py reports it as `gpu_launches`)
LAUNCH_CALLS = 0


# SLLM_DEBUG_SYNC=1: synchronise after every native call so that an asynchronous failure (a trapped kernel, an illegal
# address) is reported at the call that caused it instead of at some later sync.  Debugging aid; never set in benchmarks.
DEBUG_SYNC = os.environ.get("SLLM_DEBUG_SYNC", "0") == "1"


def check(rc: int, what: str = ""):
    global LAUNCH_CALLS
    LAUNCH_CALLS += 1
    if rc != 0:
        msg = lib().sllm_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"swiftllm_b200 native call failed{(' in ' + what) if what else ''}: {msg} (code {rc})")
    if DEBUG_SYNC and not torch.cuda.is_current_stream_capturing():
        try:
            torch.cuda.synchronize()
        except RuntimeError as e:
            raise RuntimeError(f"swiftllm_b200: device-side failure detected right after `{what}`: {e}") from e


def dtype_tag(dtype: torch.dtype) -> int:
    if dtype == torch.float16:
        return F16
    if dtype == torch.bfloat16:
        return BF16
    raise TypeError(f"swiftllm_b200 kernels support float16 and bfloat16, got {dtype}")


def stream() -> int:
    """The current torch CUDA stream as a raw cudaStream_t (the reference's convention:
    csrc/src/block_swapping.cpp:15-17, Triton launches)."""
    return torch.cuda.current_stream().cuda_stream


def ptr(t) -> int:
    return 0 if t is None else t.data_ptr()


def row_stride(t: torch.Tensor) -> int:
    """Elements between consecutive token rows of a [T, heads, D] tensor whose heads/D are contiguous within a token
    (a contiguous tensor, as in the reference, or a column slice of a fused QKV GEMM output)."""
    assert t.dim() == 3 and t.stride(2) == 1 and t.stride(1) == t.shape[2], \
        "expected [tokens, heads, head_dim] with heads and head_dim contiguous within a token"
    return t.stride(0) if t.shape[0] > 1 else max(t.stride(0), t.shape[1] * t.shape[2])


_checked_devices = set()


def require_device(t: torch.Tensor):
    """Fail loudly if a tensor is not on an sm_90 (H100) GPU."""
    if not t.is_cuda:
        raise RuntimeError("swiftllm_b200 kernels need CUDA tensors (no CPU path exists)")
    idx = t.device.index if t.device.index is not None else torch.cuda.current_device()
    if idx not in _checked_devices:
        check(lib().sllm_device_check(idx), "device_check")
        _checked_devices.add(idx)
