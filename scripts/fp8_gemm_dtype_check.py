#!/usr/bin/env python
"""Why FP8 engines run in bfloat16 only: the row-wise scaled FP8 GEMM (torch._scaled_mm with per-row and per-column fp32
scales, what kernels.linear.linear_fp8 calls) against fp64 of the dequantized operands, with bfloat16 and float16 outputs.

On an NVIDIA H100 80GB HBM3 with torch 2.11 the bfloat16 output is within one bfloat16 rounding of fp64 while the float16 output
is wrong (DESIGN.md §8o).  Run this on a later torch to see whether float16 FP8 engines can be served (worker/fp8.py `resolve`
refuses them).

    python scripts/fp8_gemm_dtype_check.py

Prints one JSON line per output dtype, with the GPU name and power limit and the torch version."""
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts"))

import torch  # noqa: E402

from sampling_bench import gpu_info  # noqa: E402


def main():
    assert torch.cuda.is_available(), "fp8_gemm_dtype_check.py runs on the GPU"
    g = torch.Generator(device="cuda").manual_seed(0)
    info = gpu_info()
    for M, K, N in ((8, 4096, 6144), (64, 14336, 4096)):
        a = torch.randn(M, K, generator=g, device="cuda")
        w = torch.randn(N, K, generator=g, device="cuda") * 0.02
        sa = a.abs().amax(1, keepdim=True) / 448
        sw = w.abs().amax(1) / 448
        qa = (a / sa).clamp(-448, 448).to(torch.float8_e4m3fn)
        qw = (w / sw[:, None]).clamp(-448, 448).to(torch.float8_e4m3fn)
        ref = (qa.double() * sa.double()) @ (qw.double() * sw.double()[:, None]).T
        for dt in (torch.bfloat16, torch.float16):
            out = torch._scaled_mm(qa, qw.t(), scale_a=sa, scale_b=sw.view(1, -1), out_dtype=dt, use_fast_accum=False)
            err = (out.double() - ref).abs()
            # one output rounding plus fp32 accumulation: far below 1 % of the largest value for a correct result
            print(json.dumps(dict(M=M, K=K, N=N, out_dtype=str(dt), max_abs_err=float(err.max()), max_abs_ref=float(ref.abs().max()),
                                  correct=bool(float(err.max()) <= 1e-2 * float(ref.abs().max())), torch=torch.__version__,
                                  gpu=info)), flush=True)


if __name__ == "__main__":
    main()
