"""FP8 weights: per-token e4m3 quantization of the GEMM inputs, fused into the kernels that produce them (new: the reference
serves 16-bit weights).  Each returns (q [rows, cols] float8_e4m3fn, scales [rows, 1] float32), the row-wise operand and scale of
kernels.linear.linear_fp8.  csrc/fp8.cu; numerics in DESIGN.md §8o."""
import torch

from swiftllm_b200 import _lib


def _rows(t: torch.Tensor) -> int:
    return t.stride(0) if t.shape[0] > 1 else max(t.stride(0), t.shape[1])


def _outputs(rows: int, cols: int, device):
    return (torch.empty((rows, cols), dtype=torch.float8_e4m3fn, device=device),
            torch.empty((rows, 1), dtype=torch.float32, device=device))


def fused_add_rmsnorm_quant_fp8(
    x: torch.Tensor,                    # [T, H] fp16 / bf16, contiguous: read, not written
    residual_io: torch.Tensor,          # [T, H] same dtype, contiguous: r = h(x + r)
    weight: torch.Tensor,               # [H]
    eps: float,
):
    """r = x + r (rounded to the storage dtype), then quantize rms_norm(r, w) - the row fused_add_rmsnorm_inplace would store."""
    assert x.is_contiguous() and residual_io.is_contiguous() and weight.is_contiguous()
    assert x.dim() == 2 and residual_io.shape == x.shape and residual_io.dtype == x.dtype and weight.dtype == x.dtype
    _lib.require_device(x)
    T, H = x.shape
    q, s = _outputs(T, H, x.device)
    _lib.check(_lib.lib().sllm_fused_add_rmsnorm_quant_fp8(
        x.data_ptr(), residual_io.data_ptr(), weight.data_ptr(), eps, T, H, q.data_ptr(), s.data_ptr(),
        _lib.dtype_tag(x.dtype), _lib.stream()), "fused_add_rmsnorm_quant_fp8")
    return q, s


def silu_and_mul_quant_fp8(x: torch.Tensor):
    """x [T, 2F] = [up | gate] (unit column stride, row-strided allowed): quantize silu_and_mul_inplace's x[:, :F]; x is not
    written."""
    assert x.dim() == 2 and x.stride(1) == 1 and x.shape[1] % 2 == 0
    _lib.require_device(x)
    T, F = x.shape[0], x.shape[1] // 2
    q, s = _outputs(T, F, x.device)
    _lib.check(_lib.lib().sllm_silu_and_mul_quant_fp8(
        x.data_ptr(), _rows(x), T, F, q.data_ptr(), s.data_ptr(), _lib.dtype_tag(x.dtype), _lib.stream()),
        "silu_and_mul_quant_fp8")
    return q, s


def quant_fp8_rows(x: torch.Tensor):
    """Quantize each row of x [R, C] (unit column stride, row-strided allowed): activations, and weights at load (rows = output
    channels)."""
    assert x.dim() == 2 and x.stride(1) == 1
    _lib.require_device(x)
    R, C = x.shape
    q, s = _outputs(R, C, x.device)
    _lib.check(_lib.lib().sllm_quant_fp8_rows(
        x.data_ptr(), _rows(x), R, C, q.data_ptr(), s.data_ptr(), _lib.dtype_tag(x.dtype), _lib.stream()), "quant_fp8_rows")
    return q, s
