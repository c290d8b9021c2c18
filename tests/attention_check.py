"""The one comparison every attention test uses: a kernel's output against the fp64 definition (oracle/kernels.py).

Normalisation: each (row, head) is held to its own scale, max_d |o64[row, head, :]|.  A row is a decode sequence or a
prefill token.  Outputs differ in size by an order of magnitude within one batch: a length-1 row returns V itself
(max_d |o| ~ 3.5 for randn V), a length-777 row averages hundreds of values (~ 0.25).  Against the batch's largest
output, a long row could be several percent off and still pass; against its own scale it cannot.  A row whose output is
near zero would make that scale meaningless, so the scale never drops below FLOOR times the batch's largest output.

Tolerance (TOL, per storage dtype, unit roundoff u = 2^-11 for fp16 and 2^-8 for bf16).  Every kernel computes
S = Q K^T with fp32 accumulation and the softmax in fp32 (exp2, running max), rounds P = exp2(s - m) to the storage dtype
as the operand of the P.V MMA (fp32 accumulation), keeps l = sum p in fp32 from the unrounded p, and rounds
o = acc / l once.  So:
  * the output rounding is at most u of the element, hence at most u of the row's scale;
  * the P rounding changes key j's weight by a relative delta_j, |delta_j| <= u, independently across keys.  The error
    of o_d, sum_j delta_j p_j v_jd / l, is a random sum about u / sqrt(3) times the size of o_d itself, whatever the
    length: it is a fixed fraction of the row's own scale, so the normalisation above needs no slack for long rows.
  * fp32 accumulation and exp2.approx are three orders of magnitude below both.
  * The wgmma prefill kernel rescales lazily: its reference point trails the row max by up to 8 (log2 units), so p
    reaches 2^8 and even the largest key's weight is rounded, where the other kernels give it exactly 1.  Rows that a
    few keys dominate (short prefill rows) err more: on an H100 80GB HBM3 (400 W power limit) its worst bf16 ratio in
    the GPU tests was 0.85 of TOL, against 0.77 for the mma.sync kernel at the same shapes.  At the long prompts, sink
    keys and lazy-rescale ramp of tests/test_prefill_regimes_gpu.py (H100 80GB HBM3, 700 W power limit) its worst bf16
    ratio was 0.89 (32 x 1024 packed, and the ramp), against 0.81 for the mma.sync kernel.
On a CPU model of this rounding at the shapes of the GPU tests (tests/test_attention_check_cpu.py), the worst
(row, head) of a batch lands at 1.2-1.6 u with the row max as reference point (up to 7.5e-4 in fp16, 6e-3 in bf16) and
at up to 1.9 u with the lazy one (9e-4, 7.4e-3).  TOL is 3 u for fp16 and 2 u for bf16.
A 2 % weight slip on one split, a dropped tile or page, an off-by-one causal mask, a wrong kv head or a head written to
its neighbour all exceed it at the shapes of the GPU tests (same file).

Set SLLM_ATTN_CHECK_LOG to a file path to append one JSON line per comparison (test id, kernel, dtype, worst
error / tolerance and its row), which is how the worst ratios of a GPU run are collected."""
import json
import os

import torch

TOL = {torch.float16: 1.5e-3, torch.bfloat16: 8e-3}
FLOOR = 1e-3


def _row_desc(r, lens, starts, prefix):
    """Human-readable position of row r: sequence, position in it, kv length."""
    if starts is None:
        return f"sequence {r}" + (f" (length {int(lens[r])})" if lens is not None else "")
    for b, (s0, n) in enumerate(zip(starts, lens)):
        s0, n = int(s0), int(n)
        if s0 <= r < s0 + n:
            pre = int(prefix[b]) if prefix is not None else 0
            pos = pre + r - s0
            return f"sequence {b}, token {r - s0} of {n} (position {pos}, attends to {pos + 1} keys)"
    return f"row {r} (outside every sequence)"


def check_attention(o, o64, nq, lens=None, *, starts=None, prefix=None, tol=None, what="attention"):
    """Assert that `o` (the kernel's output, any shape holding rows x nq heads x D) matches `o64` (fp64, same layout)
    within `tol` (default TOL[o.dtype]) of each (row, head)'s own scale.  Returns the worst error / tolerance.

    Rows are decode sequences when `starts` is None (lens[i] = length of sequence i), else packed prefill tokens of
    the sequences starting at `starts` with lens[i] query rows each (after prefix[i] cached tokens)."""
    if tol is None:
        tol = TOL[o.dtype]
    ref = o64.detach().to("cpu", torch.float64)
    got = o.detach().to("cpu", torch.float64)
    D = ref.shape[-1] if ref.dim() == 3 else ref.shape[-1] // nq
    ref = ref.reshape(-1, nq, D)
    got = got.reshape(-1, nq, D)
    err = (got - ref).abs().amax(-1)
    err = torch.where(torch.isnan(err), torch.full_like(err, float("inf")), err)        # NaN anywhere in a row fails it
    big = float(ref.abs().max())
    scale = ref.abs().amax(-1).clamp_min(max(FLOOR * big, 1e-30))
    ratio = err / scale
    worst = int(torch.argmax(ratio))
    r, h = divmod(worst, nq)
    worst_ratio = float(ratio.reshape(-1)[worst])
    desc = (f"{what}: worst (row, head) is {_row_desc(r, lens, starts, prefix)}, head {h}: "
            f"max|o - o64| = {float(err[r, h]):.3g} = {worst_ratio:.3g} x its scale {float(scale[r, h]):.3g} "
            f"(tolerance {tol:g}, {int((ratio > tol).sum())} of {ratio.numel()} (row, head) pairs over)")
    log = os.environ.get("SLLM_ATTN_CHECK_LOG")
    if log:
        with open(log, "a") as f:
            f.write(json.dumps({"test": os.environ.get("PYTEST_CURRENT_TEST", ""), "kernel": what, "dtype": str(o.dtype),
                                "head_dim": D, "ratio_to_tol": worst_ratio / tol, "detail": desc}) + "\n")
    assert worst_ratio <= tol, desc
    return worst_ratio / tol
