"""Multi-LoRA: the low-rank shrink (u = x·Aᵀ) and expand (y += s·u·Bᵀ) of per-request adapters, added to a projection's output
next to its GEMM (new: the reference serves one set of weights).  csrc/lora.cu."""
import torch

from swiftllm_b200 import _lib


def _rows(t: torch.Tensor) -> int:
    return t.stride(0) if t.shape[0] > 1 else max(t.stride(0), t.shape[1])


def lora_shrink(
    x: torch.Tensor,                    # [T, K] fp16 / bf16, unit column stride (a row-strided view works)
    u: torch.Tensor,                    # [>= T, >= S * R] same dtype, contiguous rows: columns [0, S * R) of the tiles' rows written
    lora_a: torch.Tensor,               # [max_loras, S * R, K] the slot pool of this site's stacked A slices
    tiles: torch.Tensor,                # [num_tiles, 3] int32 (first row, rows <= 64, slot)
    slice_mask: torch.Tensor,           # [max_loras] int32: bit s set = slice s targeted; 0 = the site is skipped
):
    """u[t] = round(x[t]·Aᵀ) for every row t of a tile whose slot targets the site."""
    assert x.dim() == 2 and x.stride(1) == 1 and u.dim() == 2 and u.stride(1) == 1 and u.dtype == x.dtype
    assert lora_a.dim() == 3 and lora_a.is_contiguous() and lora_a.dtype == x.dtype and lora_a.shape[2] == x.shape[1]
    assert tiles.dtype == torch.int32 and tiles.dim() == 2 and tiles.shape[1] == 3 and tiles.is_contiguous()
    assert slice_mask.dtype == torch.int32 and slice_mask.shape == (lora_a.shape[0],) and slice_mask.is_contiguous()
    assert u.shape[0] >= x.shape[0] and u.shape[1] >= lora_a.shape[1]
    _lib.require_device(x)
    _lib.check(_lib.lib().sllm_lora_shrink(
        x.data_ptr(), _rows(x), x.shape[0], x.shape[1], u.data_ptr(), u.stride(0), lora_a.data_ptr(), lora_a.stride(0),
        lora_a.shape[1], tiles.data_ptr(), tiles.shape[0], slice_mask.data_ptr(), lora_a.shape[0], _lib.dtype_tag(x.dtype),
        _lib.stream()), "lora_shrink")


def lora_expand(
    y: torch.Tensor,                    # [T, N] fp16 / bf16, unit column stride: updated in place
    u: torch.Tensor,                    # the shrink's output buffer
    lora_b: torch.Tensor,               # [max_loras, N, R] the slot pool of this site's B
    slice_ends: tuple,                  # (n1, n2): columns [0, n1), [n1, n2), [n2, N) read u columns [0, R), [R, 2R), [2R, 3R)
    tiles: torch.Tensor,
    slice_mask: torch.Tensor,
    scales: torch.Tensor,               # [max_loras] float32
):
    """y[t, n] = round(float(y[t, n]) + s·(u[t, slice]·B[n])) for every row t of a tile and every targeted slice."""
    assert y.dim() == 2 and y.stride(1) == 1 and u.dtype == y.dtype and u.stride(1) == 1
    assert lora_b.dim() == 3 and lora_b.is_contiguous() and lora_b.dtype == y.dtype and lora_b.shape[1] == y.shape[1]
    assert tiles.dtype == torch.int32 and tiles.dim() == 2 and tiles.shape[1] == 3 and tiles.is_contiguous()
    assert slice_mask.dtype == torch.int32 and slice_mask.shape == (lora_b.shape[0],)
    assert scales.dtype == torch.float32 and scales.shape == (lora_b.shape[0],) and u.shape[0] >= y.shape[0]
    _lib.require_device(y)
    _lib.check(_lib.lib().sllm_lora_expand(
        y.data_ptr(), _rows(y), y.shape[0], y.shape[1], u.data_ptr(), u.stride(0), lora_b.data_ptr(), lora_b.stride(0),
        lora_b.shape[2], int(slice_ends[0]), int(slice_ends[1]), tiles.data_ptr(), tiles.shape[0], slice_mask.data_ptr(),
        scales.data_ptr(), lora_b.shape[0], _lib.dtype_tag(y.dtype), _lib.stream()), "lora_expand")
