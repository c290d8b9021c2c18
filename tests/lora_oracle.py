"""Restatement of the multi-LoRA numerics contract (csrc/lora.cu, worker/lora.py) in torch fp64, and its error bounds.

At a site with 16-bit input x [T, K] and GEMM output y [T, N], row t with slot a (A [S * R, K], B [N, R], scale s):
  1. u[t, :] = round16(sum_k x[t, k] * A[:, k])                      - the sum in fp32 on the device, exact here;
  2. y[t, n] = round16(float(y[t, n]) + s * sum_j u[t, sl(n) R + j] B[n, j]), the inner sum in fp32 on the device (exact here),
     then one fp32 multiply, one fp32 add and one rounding;
  3. rows without a slot and slices the adapter does not target are not written: bit for bit what they were.
The device's fp32 sums are order-dependent, so a comparison with this restatement uses the bounds below; everything else
(the fp32 multiply and add, the roundings, which elements are written) is exact."""
import torch

EPS32 = 2.0 ** -24                      # unit roundoff of fp32


def ulp16(v: torch.Tensor, dtype) -> torch.Tensor:
    """Spacing of the 16-bit format at |v| (the subnormal spacing below the smallest normal)."""
    mant, emin = (10, -14) if dtype == torch.float16 else (7, -126)
    e = torch.floor(torch.log2(v.abs().double().clamp_min(2.0 ** emin)))
    return torch.pow(2.0, e - mant)


def shrink(x: torch.Tensor, A: torch.Tensor) -> torch.Tensor:
    """u = round16(x·Aᵀ) with the sum exact (fp64): [T, S * R]."""
    return (x.double() @ A.double().t()).to(x.dtype)


def shrink_bound(x: torch.Tensor, A: torch.Tensor) -> torch.Tensor:
    """|device u - shrink(x, A)| bound per element: the fp32 sum's error (K * eps32 * sum |x A|) plus one 16-bit ulp (the two
    results may round to neighbours when the exact sum lies near a rounding boundary)."""
    K = x.shape[1]
    mag = x.double().abs() @ A.double().abs().t()
    exact = x.double() @ A.double().t()
    return 1.01 * K * EPS32 * mag + ulp16(exact.abs() + K * EPS32 * mag, x.dtype)


def shrink_ordered(x: torch.Tensor, A: torch.Tensor, warps: int = 8) -> tuple:
    """The shrink's fp32 sum in the kernel's order (csrc/lora.cu): warp w takes the 32-wide k-chunks w, w + warps, ...; per chunk
    one mma adds the 16 products at k % 8 < 4, then one adds those at k % 8 >= 4; the warps' partials are then added in warp
    order.  Each mma is emulated as one fp32 rounding of (accumulator + exact sum of its 16 products).  Returns (ref [T, J] fp32,
    E [T, J] fp64): E bounds |device fp32 sum - ref|, allowing every mma of the device 4 fp32 roundings of (|accumulator| + sum of
    |products|) where the emulation has one, and every fp32 add of the warp sum one rounding of its result.  The bound grows with
    the running sums, not with K * sum |x A|, so a dropped or mis-paired product (a change of order |u| / sqrt(K)) exceeds it."""
    T, K = x.shape
    xd, Ad = x.double(), A.double()
    pos = torch.arange(32) % 8
    chunks = torch.arange(K).view(K // 32, 32)
    groups = [chunks[:, pos < 4], chunks[:, pos >= 4]]
    err = torch.zeros((T, A.shape[0]), dtype=torch.float64)
    parts = []
    for w in range(warps):
        acc = torch.zeros((T, A.shape[0]), dtype=torch.float32)
        for c in range(w, K // 32, warps):
            for g in groups:
                idx = g[c]
                s = xd[:, idx] @ Ad[:, idx].t()
                mag = xd[:, idx].abs() @ Ad[:, idx].abs().t()
                err += 4 * EPS32 * (acc.double().abs() + mag)
                acc = (acc.double() + s).float()
        parts.append(acc)
    total = parts[0]
    for p in parts[1:]:
        total = (total.double() + p.double()).float()
        err += 2 * EPS32 * (total.double().abs() + p.double().abs())
    return total, 1.01 * err


def shrink_check(u: torch.Tensor, ref: torch.Tensor, E: torch.Tensor) -> torch.Tensor:
    """Per element: is the device's 16-bit u the rounding of an fp32 value within E of ref (|u - ref| <= half a 16-bit ulp of
    |ref| + E, plus E)?"""
    d = (u.double() - ref.double()).abs()
    return d <= 0.5 * ulp16(ref.double().abs() + E, u.dtype) + E


def expand_exact(y: torch.Tensor, u: torch.Tensor, B: torch.Tensor, s: float, ends, mask: int, R: int) -> torch.Tensor:
    """Step 2 for every row of y (all rows adapted), with the inner sum exact then rounded to fp32: the reference the device
    matches within one 16-bit ulp.  ends = (n1, n2) slice ends; mask: bit sl = slice sl targeted."""
    N = y.shape[1]
    out = y.clone()
    bounds = [0, ends[0], ends[1], N]
    for sl in range(3):
        lo, hi = bounds[sl], bounds[sl + 1]
        if lo >= hi or not (mask >> sl) & 1:
            continue
        acc = (u[:, sl * R:(sl + 1) * R].double() @ B[lo:hi].double().t()).float()
        d = torch.tensor(s, dtype=torch.float32) * acc                        # fp32 multiply
        out[:, lo:hi] = (y[:, lo:hi].float() + d).to(y.dtype)                 # fp32 add, one rounding
    return out


def expand_bound(y: torch.Tensor, u: torch.Tensor, B: torch.Tensor, s: float, ref: torch.Tensor, R: int, ends,
                 N: int) -> torch.Tensor:
    """|device y - expand_exact(...)| bound per element: one 16-bit ulp of the result, widened by the device's fp32 inner sum
    (R * eps32 * |s| * sum_j |u_j B_j|) and the fp32 rounding of the multiply and the add."""
    bounds = [0, ends[0], ends[1], N]
    mag = torch.zeros(y.shape, dtype=torch.float64)
    for sl in range(3):
        lo, hi = bounds[sl], bounds[sl + 1]
        if lo < hi:
            mag[:, lo:hi] = u[:, sl * R:(sl + 1) * R].double().abs() @ B[lo:hi].double().abs().t()
    extra = abs(s) * (R + 2) * EPS32 * mag + 2 * EPS32 * y.double().abs()
    return ulp16(ref.double().abs() + extra, y.dtype) + extra


def apply(x, y, slots, adapters, R: int, ends=None, site_mask=None):
    """Steps 1-3 on whole rows: slots[t] is row t's slot or None, adapters[a] = (A, B, s).  site_mask[a]: slice bits of slot a
    at this site (default all).  Returns the new y and u (rows without a slot: u zeros)."""
    N = y.shape[1]
    ends = ends or (N, N)
    out, us = y.clone(), torch.zeros((y.shape[0], max(a[0].shape[0] for a in adapters.values())), dtype=y.dtype)
    for t, a in enumerate(slots):
        if a is None:
            continue
        A, B, s = adapters[a]
        m = 7 if site_mask is None else site_mask[a]
        if m == 0:
            continue
        u = shrink(x[t:t + 1], A)
        us[t, :u.shape[1]] = u[0]
        out[t:t + 1] = expand_exact(y[t:t + 1], u, B, s, ends, m, R)
    return out, us


def merged_weight(W: torch.Tensor, A: torch.Tensor, B: torch.Tensor, s: float) -> torch.Tensor:
    """W + s·B·A in fp64, rounded once: the base weight a merged copy of the adapter would carry."""
    return (W.double() + s * (B.double() @ A.double())).to(W.dtype)
