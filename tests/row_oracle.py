"""Restatement of the row kernels' numerics (csrc/elementwise.cu: rmsnorm_kernel, silu_and_mul_kernel; csrc/common.cuh: the
add + RMSNorm row epilogue) in fp64, the bounds a device result must meet, the test data, an fp32 emulation of the kernels'
own summation order and plausible wrong variants of it.  TEST INFRASTRUCTURE ONLY; plain torch on CPU tensors.

With h(.) = round to the storage dtype, u = 2^-24 and eps32 = eps as the fp32 the kernel receives:
  * RMSNorm     ref = x * w / sqrt(mean(x^2) + eps32) in fp64.  The device sums the squares in fp32 in its own order (at most
                H - 1 roundings of a sum of nonnegative terms: relative error <= (H - 1) u), then one division, one add, sqrtf and
                one reciprocal (the square root halves the sum's relative error), and the two fp32 products (x * rstd) * w.  So
                with delta = (H / 2 + 8) u its fp32 result lies within |ref| delta of ref, and the stored value satisfies
                    |out - ref| <= ulp16(|ref| (1 + delta)) / 2 + |ref| delta.
  * fused add   the residual is h(x + r), bit for bit (an fp32 add of two 16-bit values rounded once is the correctly rounded
                16-bit sum); x_out is RMSNorm of that residual.
  * SiLU·mul    out = h(up * h(silu(f(gate)))) with silu = g / (1 + expf(-g)) in fp32.  expf is within 2 fp32 ulps, the add and
                the division are rounded once, so the fp32 silu lies within 8 u |s| (+ a few fp32 subnormal spacings) of the
                fp64 s = g / (1 + exp(-g)): its 16-bit rounding is one of at most two candidates, and the 16-bit product is then
                exact: out == h(up * c) for a candidate c (the product of two 16-bit values is exact in fp64).
                The one exception: where -g > ln(FLT_MAX) (every 16-bit gate <= -88.75) expf(-g) overflows, and the kernel's
                silu is g / inf = -0.  A correctly rounded silu differs from that at the 17 bf16 gates -97, -96.5, ..., -89,
                where it is a nonzero bf16 value (at fp16 gates there it rounds to -0 as well).
                oracle.kernels.silu_and_mul, which restates the reference kernel in fp32, gives -0 there too.  The band is
                pinned to that value: c = -0.
Out of contract: rows whose fp32 sum of squares overflows (bf16 |x| of order 1e19 / sqrt(H) and above).  The test data stays
far inside it (|x| <= 2^15)."""
from __future__ import annotations

import math

import numpy as np
import torch

from lora_oracle import ulp16
from oracle import kernels as K

U32 = 2.0 ** -24                       # unit roundoff of fp32
LN_FLT_MAX = math.log(float(np.finfo(np.float32).max))
KINDS = ("small", "normal", "zeros", "outlier", "big")


def eps32(eps: float) -> float:
    return float(np.float32(eps))


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int16)


def round16(v: torch.Tensor, dtype) -> torch.Tensor:
    """Round fp64 values to the 16-bit dtype once, to nearest even (subnormals and overflow to inf included)."""
    q = ulp16(v, dtype)
    r = torch.round(v / q) * q
    r = torch.where(r.abs() > torch.finfo(dtype).max, torch.copysign(torch.full_like(r, math.inf), r), r)
    return r.to(dtype)                 # exact: r is representable


# ----------------------------------------------------------------------------- RMSNorm
def rmsnorm_ref(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    xd = x.double()
    ms = (xd * xd).mean(dim=-1, keepdim=True)
    return xd * w.double() / torch.sqrt(ms + eps32(eps))


def rmsnorm_bound(ref: torch.Tensor, H: int, dtype) -> torch.Tensor:
    delta = (H / 2 + 8) * U32
    return 0.5 * ulp16(ref.abs() * (1 + delta), dtype) + ref.abs() * delta


def rmsnorm_ok(out: torch.Tensor, x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    """Per element: does the device's x_out meet the bound around the fp64 RMSNorm of x (the post-add row when fused)?"""
    ref = rmsnorm_ref(x, w, eps)
    return (out.double() - ref).abs() <= rmsnorm_bound(ref, x.shape[-1], out.dtype)


def add_residual(x: torch.Tensor, r: torch.Tensor) -> torch.Tensor:
    """h(x + r): the fused kernel's new residual."""
    return (x.float() + r.float()).to(x.dtype)


# ----------------------------------------------------------------------------- SiLU·mul
def silu_candidates(gate: torch.Tensor, pin_band: bool = True):
    """(c0, c1), 16-bit: h(silu) of the device is one of them; in the expf overflow band both are -0 (unless pin_band is
    False: then both come from the fp64 silu there too)."""
    g = gate.double()
    s = g / (1 + torch.exp(-g))
    r = 8 * U32 * s.abs() + 2.0 ** -146
    band = (-g > LN_FLT_MAX) & pin_band
    neg0 = torch.full_like(s, -0.0)
    return (torch.where(band, neg0, round16(s - r, gate.dtype).double()).to(gate.dtype),
            torch.where(band, neg0, round16(s + r, gate.dtype).double()).to(gate.dtype))


def silu_and_mul_ok(out: torch.Tensor, up: torch.Tensor, gate: torch.Tensor, pin_band: bool = True) -> torch.Tensor:
    """Per element: is the device's output h(up * c) for a candidate c, bit for bit?"""
    o = bits(out)
    return torch.stack([bits(round16(up.double() * c.double(), out.dtype)) == o
                        for c in silu_candidates(gate, pin_band)]).any(0)


# ----------------------------------------------------------------------------- test data
def _row(kind: str, H: int, g: torch.Generator, col: int, sign: float) -> torch.Tensor:
    if kind == "zeros":
        return torch.zeros(H, dtype=torch.float64)
    v = torch.randn(H, generator=g, dtype=torch.float64)
    if kind == "small":                # mean square ~1e-6, next to eps: where eps goes is visible
        return v * 1e-3
    if kind == "outlier":              # one large value per row, at a column that moves from row to row
        v[col] = sign * 3.0e4
    elif kind == "big":                # fp16 values near 2^15
        v = torch.sign(v) * (0.5 + 0.499 * torch.rand(H, generator=g, dtype=torch.float64)) * 2.0 ** 15
    return v


def norm_inputs(T: int, H: int, dtype, seed: int, fused: bool):
    """(x, r, w) on the CPU; r is None unless fused.  Row t is of kind KINDS[t % 5]: "small" rows (mean square ~1e-6), random
    rows, zero rows (fused: x = -r, so the sum cancels to zeros), one outlier of 3e4 per row, and values near 2^15.  When fused,
    x and r are half of two rows of the same kind (the outlier in the same column, same sign), so h(x + r) is of that kind and
    stays finite in fp16."""
    g = torch.Generator().manual_seed(seed)
    xs, rs = [], []
    for t in range(T):
        kind = KINDS[t % len(KINDS)]
        col = int(torch.randint(H, (1,), generator=g))
        sign = 1.0 if float(torch.rand(1, generator=g)) < 0.5 else -1.0
        a = _row(kind, H, g, col, sign)
        if not fused:
            xs.append(a)
        elif kind == "zeros":
            b = torch.randn(H, generator=g, dtype=torch.float64)
            xs.append(b); rs.append(-b)
        else:
            xs.append(0.5 * a); rs.append(0.5 * _row(kind, H, g, col, sign))
    w = 1 + 0.1 * torch.randn(H, generator=g, dtype=torch.float64)
    x = torch.stack(xs).to(dtype)
    return x, (torch.stack(rs).to(dtype) if fused else None), w.to(dtype)


def silu_inputs(T: int, F: int, dtype, seed: int) -> torch.Tensor:
    """x [T, 2F] = [up | gate] on the CPU.  Gates: random N(0, 4^2), uniform in [-110, 20], 16-bit subnormals and a list of
    specials (+-0, the smallest subnormals, the whole expf overflow band -97 ... -88.5, +-20); up spans 2^-20 .. 2^6."""
    g = torch.Generator().manual_seed(seed)
    sub = 2.0 ** (-24 if dtype == torch.float16 else -133)
    specials = torch.tensor([0.0, -0.0, sub, -sub, 3 * sub, -5 * sub, 20.0, -20.0, -88.5, -88.75]
                            + [-89.0 - 0.5 * i for i in range(18)], dtype=torch.float64)
    pick = torch.rand(T, F, generator=g, dtype=torch.float64)
    gate = torch.randn(T, F, generator=g, dtype=torch.float64) * 4
    gate = torch.where(pick > 0.45, -110 + 130 * torch.rand(T, F, generator=g, dtype=torch.float64), gate)
    gate = torch.where(pick > 0.75, torch.randn(T, F, generator=g, dtype=torch.float64) * sub * 64, gate)
    gate = torch.where(pick > 0.85, specials[torch.randint(len(specials), (T, F), generator=g)], gate)
    up = torch.randn(T, F, generator=g, dtype=torch.float64) * torch.pow(2.0, torch.randint(-20, 7, (T, F), generator=g))
    return torch.cat([up, gate], dim=1).to(dtype)


# ----------------------------------------------------------------------------- the kernels' order, and wrong variants
def rmsnorm_emulated(x: torch.Tensor, w: torch.Tensor, eps: float, vpt: int, threads: int, *, divisor=None,
                     eps_after_sqrt=False, drop_last_warp=False, neighbour_rstd=False, weight_shift=0) -> torch.Tensor:
    """rmsnorm_kernel's fp32 arithmetic in its own order: thread i adds, per vector i + k * threads it owns, the 4 pairs
    fx^2 + fy^2 (one rounding each) to its partial; warp_sum's xor butterfly; the warps' sums added in warp order; then
    1 / sqrtf(total / H + eps) and h((x * rstd) * w).  The keyword arguments turn it into a wrong variant: another divisor, eps
    added after the square root, the last warp's partial dropped, row t normalised with row t + 1's rstd, the weight read
    `weight_shift` vectors further on."""
    Tn, H = x.shape
    nvec = H // 8
    pairs = x.float().view(Tn, nvec, 4, 2)
    ss = torch.zeros(Tn, threads, dtype=torch.float32)
    for k in range(vpt or -(-nvec // threads)):
        idx = torch.arange(threads) + k * threads
        live = idx < nvec
        p = pairs[:, idx.clamp(max=nvec - 1)]
        for j in range(4):
            q = p[:, :, j, 0] * p[:, :, j, 0] + p[:, :, j, 1] * p[:, :, j, 1]
            ss = torch.where(live, ss + q, ss)
    lanes = torch.arange(threads)
    for o in (16, 8, 4, 2, 1):
        ss = ss + ss[:, lanes ^ o]
    red = ss[:, ::32]
    total = torch.zeros(Tn, dtype=torch.float32)
    for wi in range(red.shape[1] - (1 if drop_last_warp else 0)):
        total = total + red[:, wi]
    mean = total / torch.tensor(float(divisor or H), dtype=torch.float32)
    e = torch.tensor(eps, dtype=torch.float32)
    rstd = 1.0 / (torch.sqrt(mean) + e) if eps_after_sqrt else 1.0 / torch.sqrt(mean + e)
    if neighbour_rstd:
        rstd = rstd.roll(-1)
    wf = w.float().roll(-8 * weight_shift)
    return ((x.float() * rstd[:, None]) * wf).to(x.dtype)


def rmsnorm_numpy_order(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    """oracle.kernels.rmsnorm: the same formula with numpy's pairwise sum of squares."""
    return K.rmsnorm(x, w, eps)


def silu_and_mul_fp32(x: torch.Tensor) -> torch.Tensor:
    """oracle.kernels.silu_and_mul's [T, F] output: the reference kernel's fp32 formula (numpy expf), silu rounded to 16 bits."""
    F = x.shape[1] // 2
    with np.errstate(over="ignore"):
        return K.silu_and_mul(x)[:, :F]


def silu_and_mul_single_rounding(x: torch.Tensor) -> torch.Tensor:
    """Wrong variant: h(up * silu) with the fp32 silu never rounded to 16 bits on its own."""
    F = x.shape[1] // 2
    gate = x[:, F:].float()
    with np.errstate(over="ignore"):
        e = torch.from_numpy(np.exp(-gate.numpy()))
    return (x[:, :F].float() * (gate / (1.0 + e))).to(x.dtype)
