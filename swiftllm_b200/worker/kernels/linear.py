"""Reference: swiftllm/worker/kernels/linear.py:3-12.  A plain library GEMM (cuBLAS through torch), exactly as in
the reference; the hot-path scope (SURVEY.md §8 a9) keeps it a library call."""
import torch


def linear(
    a: torch.Tensor,  # [a, b] (row-strided allowed)
    w: torch.Tensor   # [c, b]
) -> torch.Tensor:    # [a, c]
    return torch.nn.functional.linear(a, w)


def linear_fp8(
    xq: torch.Tensor,           # [M, K] float8_e4m3fn, row-major
    sx: torch.Tensor,           # [M, 1] float32: per-token scales
    wq: torch.Tensor,           # [N, K] float8_e4m3fn, row-major (passed to the GEMM as wq.t(), column-major)
    sw: torch.Tensor,           # [N] float32: per-output-channel scales
    out_dtype: torch.dtype,     # bfloat16 (torch 2.11's float16 outputs of this GEMM are wrong on sm_90)
    out: torch.Tensor = None,   # optional [M, N] out_dtype destination (e.g. the fused exchange's partial buffer)
) -> torch.Tensor:
    """out[m, n] = round(sum_k xq[m, k] * wq[n, k] * sx[m] * sw[n]), fp32 accumulation: the row-wise scaled FP8 GEMM of the library
    (torch._scaled_mm, CUTLASS on sm_90).  Needs K and N multiples of 16."""
    kw = dict(scale_a=sx, scale_b=sw.view(1, -1), out_dtype=out_dtype, use_fast_accum=False)
    if out is None:
        return torch._scaled_mm(xq, wq.t(), **kw)
    return torch._scaled_mm(xq, wq.t(), **kw, out=out)
