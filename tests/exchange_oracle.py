"""TEST INFRASTRUCTURE: a plain restatement of the tensor-parallel exchange kernels (csrc/allreduce_norm.cu one-shot and two-shot,
csrc/allreduce_ll.cu LL push), for N ranks that each hold a partial P_r [T, H] of the same activations.

The contract every kernel (and tests/cpu_shim.py: GlooFusedAllReduce) must meet, with h(.) = round to the storage dtype and
f(.) = exact widening to fp32:
  * sum       s = h(sum_r f(P_r))         fp32 accumulation starting from 0, ranks in the fixed order 0, 1, ..., N-1, rounded once
  * residual  R' = h(s + R)               a storage-dtype add, correctly rounded (so R' = h(h(sum) + R): two roundings)
  * x_out     rmsnorm(R') * w             oracle.kernels.rmsnorm
  * ownership row t belongs to rank t % N (two-shot and LL: only the owner reduces, adds and normalises it; the residual is kept
              up to date only on the rows a rank owns)
Tolerance: R' must match bit for bit.  x_out may differ from this restatement by <= 1 ulp, because the kernels sum the squares
in a different fp32 order than numpy's pairwise sum (as in test_rmsnorm_vs_oracle).  Between the three kernels and between
ranks x_out must be bit-identical: they share the thread-count formula and the loop, hence the order of the sum of squares.

LL line format: every 4 payload words (32-bit, i.e. 8 elements) travel as two 16-byte lines {w0, tag, w1, tag}, {w2, tag, w3,
tag}, so one row of H 16-bit elements is H 32-bit words (2H elements) on the wire.  `ll_pack` / `ll_unpack` convert, and
`ll_rs_image` / `ll_ag_image` give what one rank's pushes leave in a peer's receive buffers:
  * rs_recv  [N src][rows_per_rank][H words]: partial row t of rank `src` at [src][t // N] of its owner t % N
  * ag_recv  [max_tokens][H words]:           normalised row t at [t] of every rank but its owner
All helpers are plain torch and work on CPU or CUDA tensors."""
from __future__ import annotations

import torch

from oracle import kernels as K


# ----------------------------------------------------------------------------- arithmetic
def exchange_sum(partials) -> torch.Tensor:
    """h(sum_r f(P_r)): fp32, rank order 0..N-1, accumulator starting from 0, one rounding."""
    acc = torch.zeros(partials[0].shape, dtype=torch.float32, device=partials[0].device)
    for p in partials:
        acc += p.float()
    return acc.to(partials[0].dtype)


def exchange_add(partials, residual) -> torch.Tensor:
    """The new residual h(h(sum) + R)."""
    return exchange_sum(partials) + residual


def exchange_add_norm(partials, residual, weight, eps):
    """(x_out, new residual) of one exchange, every row."""
    r = exchange_add(partials, residual)
    return K.rmsnorm(r.cpu(), weight.cpu(), eps).to(r.device), r


def owned(num_tokens: int, nranks: int, rank: int, device="cpu") -> torch.Tensor:
    """Boolean mask of the rows rank `rank` owns (t % N == rank)."""
    return (torch.arange(num_tokens, device=device) % nranks) == rank


def owned_rows(num_tokens: int, nranks: int, rank: int, device="cpu") -> torch.Tensor:
    """Indices of the rows rank `rank` owns, ascending (none when rank >= T)."""
    return torch.arange(min(rank, num_tokens), num_tokens, nranks, device=device)


# ----------------------------------------------------------------------------- test data
def make_inputs(nranks: int, num_tokens: int, hidden: int, dtype: torch.dtype, seed: int = 0):
    """(partials [N, T, H], residual [T, H], weight [H]) on the CPU; the same arguments give the same data in every test.

    Random partials of a few units sum exactly in fp32, so they cannot tell rank orders apart.  The first min(H, 16) columns
    therefore cancel: in column c ranks a = c % N and b = (c + 1) % N hold +-2^k * u and every other rank a tiny 2^(k-24) * v,
    below half an fp32 ulp of 2^k * u.  Summed in rank order the pair cancels exactly whenever a and b are adjacent and nothing
    comes between them; any other order or grouping rounds some tiny terms away, and the loss (a multiple of 2^(k-23)) is
    several ulps of the residual.  k = 15 keeps fp16 in range; bf16 uses k = 20 so the loss is visible next to a residual
    of order 1.
    The last column witnesses the two roundings: with m fraction bits, P_0 = 2^-(m+1), P_1 = 2^-(2m+2), R = 1 gives
    h(h(sum) + R) = 1 (two ties to even) but h(sum + R) = 1 + 2^-m."""
    g = torch.Generator().manual_seed(seed * 1_000_003 + nranks * 100_003 + num_tokens * 10_007 + hidden * 2
                                      + (dtype == torch.bfloat16))
    P = torch.randn(nranks, num_tokens, hidden, generator=g)
    k, m = (15, 10) if dtype == torch.float16 else (20, 7)
    C = min(hidden - 1, 16)
    u = 1 + 0.99 * torch.rand(num_tokens, C, generator=g)
    v = 0.5 + 0.5 * torch.rand(nranks, num_tokens, C, generator=g)
    tiny = (2.0 ** (k - 24)) * v
    for c in range(C):
        a, b = c % nranks, (c + 1) % nranks
        col = tiny[:, :, c].clone()
        col[a] = (2.0 ** k) * u[:, c]
        col[b] = -(2.0 ** k) * u[:, c]
        P[:, :, c] = col
    P[:, :, -1] = 0
    P[0, :, -1], P[1, :, -1] = 2.0 ** -(m + 1), 2.0 ** -(2 * m + 2)
    residual = torch.randn(num_tokens, hidden, generator=g)
    residual[:, -1] = 1
    weight = 1 + 0.1 * torch.randn(hidden, generator=g)
    return P.to(dtype), residual.to(dtype), weight.to(dtype)


# ----------------------------------------------------------------------------- wrong variants (the data must reject them)
def sum_reversed(partials) -> torch.Tensor:
    return exchange_sum(list(partials)[::-1])


def sum_pairwise(partials) -> torch.Tensor:
    def tree(ps):
        if len(ps) == 1:
            return ps[0].float()
        return tree(ps[: len(ps) // 2]) + tree(ps[len(ps) // 2:])
    return tree(list(partials)).to(partials[0].dtype)


def add_single_rounding(partials, residual) -> torch.Tensor:
    """h(sum + R) with the fp32 sum never rounded to the storage dtype on its own."""
    acc = torch.zeros(partials[0].shape, dtype=torch.float32)
    for p in partials:
        acc += p.float()
    return (acc + residual.float()).to(residual.dtype)


# ----------------------------------------------------------------------------- comparisons
def ulp_distance(a: torch.Tensor, b: torch.Tensor) -> int:
    """Largest distance in representable values of the 16-bit dtype (sign-magnitude aware)."""
    def key(t):
        i = t.contiguous().view(torch.int16).to(torch.int32)
        return torch.where(i < 0, -(i & 0x7FFF), i)
    if a.numel() == 0:
        return 0
    return int((key(a) - key(b)).abs().max())


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int16)


# ----------------------------------------------------------------------------- LL format
def as_i32(x: int) -> int:
    """A uint32 value (an epoch, a tag) as the int32 with the same bits."""
    x &= 0xFFFFFFFF
    return x - (1 << 32) if x >= (1 << 31) else x


def ll_pack(rows: torch.Tensor, tag: int) -> torch.Tensor:
    """[..., H] 16-bit rows -> [..., H] int32 LL words: every payload word followed by the tag."""
    w = rows.contiguous().view(torch.int32)
    return torch.stack((w, torch.full_like(w, as_i32(tag))), dim=-1).reshape(*w.shape[:-1], 2 * w.shape[-1])


def ll_unpack(lines: torch.Tensor, dtype: torch.dtype):
    """[..., H] int32 LL words -> ([..., H] rows of `dtype`, [..., H / 2] int32 tags)."""
    pairs = lines.reshape(*lines.shape[:-1], lines.shape[-1] // 2, 2)
    return pairs[..., 0].contiguous().view(dtype), pairs[..., 1]


def ll_rs_image(partial: torch.Tensor, src: int, dst: int, nranks: int, rows_per_rank: int, tag: int) -> torch.Tensor:
    """What rank `src` pushes into rank `dst`'s rs_recv [N][rows_per_rank][H] (int32, zero where nothing is pushed):
    LL(partial[t]) at [src][t // N] for every row t that `dst` owns (nothing when src == dst)."""
    T, H = partial.shape
    img = torch.zeros(nranks, rows_per_rank, H, dtype=torch.int32, device=partial.device)
    if src != dst:
        rows = owned_rows(T, nranks, dst, partial.device)
        img[src, rows // nranks] = ll_pack(partial[rows], tag)
    return img


def ll_ag_image(x_out: torch.Tensor, src: int, dst: int, nranks: int, max_tokens: int, tag: int) -> torch.Tensor:
    """What rank `src` pushes into rank `dst`'s ag_recv [max_tokens][H] (int32, zero elsewhere): LL(x_out[t]) at [t] for every
    row t that `src` owns (nothing when src == dst: an owner writes its own copy to x_out directly)."""
    T, H = x_out.shape
    img = torch.zeros(max_tokens, H, dtype=torch.int32, device=x_out.device)
    if src != dst:
        rows = owned_rows(T, nranks, src, x_out.device)
        img[rows] = ll_pack(x_out[rows], tag)
    return img
