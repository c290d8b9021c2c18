"""GPU: the row kernels of csrc/elementwise.cu against fp64 (tests/row_oracle.py).  RMSNorm and add + RMSNorm run at every
width of tests/row_geometry.py's table (case ids name the launch instance: VPT4, VPT2, GEN, GEN>48K), in fp16 and bf16, with
rows of every kind in each launch; SiLU·mul runs at model MLP widths, their tensor-parallel shards and odd vector counts.
Every launch writes a [:T] view of a larger buffer, whose rows past T must stay untouched."""
import pytest
import torch

import row_geometry as RG
import row_oracle as RO

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
# (T, eps): every width and dtype runs both eps values
NORM_T = [(1, 1e-6), (7, 1e-5), (64, 1e-6), (300, 1e-5)]


def _fill(T, C, dt, head: torch.Tensor, seed: int) -> torch.Tensor:
    """A [T + 2, C] device buffer: `head` in its first T rows, random rows after."""
    g = torch.Generator().manual_seed(seed)
    return torch.cat([head, torch.randn(2, C, generator=g).to(dt)]).cuda()


def _norm(fused, x, r, w, eps):
    from swiftllm_b200.worker.kernels.rmsnorm import fused_add_rmsnorm_inplace, rmsnorm_inplace
    if fused:
        fused_add_rmsnorm_inplace(x, r, w, eps)
    else:
        rmsnorm_inplace(x, w, eps)


def _report(ok, what):
    bad = (~ok).nonzero()
    return f"{what}: {bad.shape[0]} elements out of bound, first at {bad[:4].tolist()}"


@pytest.mark.parametrize("T,eps", NORM_T, ids=[f"T{t}-eps{e:g}" for t, e in NORM_T])
@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("H", RG.WIDTHS, ids=RG.width_id)
@pytest.mark.parametrize("fused", [False, True], ids=["rmsnorm", "add_rmsnorm"])
def test_rmsnorm_rows_against_fp64(fused, H, dt, T, eps):
    x, r, w = RO.norm_inputs(T, H, dt, seed=H * 11 + T + fused, fused=fused)
    xb = _fill(T, H, dt, x, seed=H + T)
    rb = _fill(T, H, dt, r, seed=H + T + 1) if fused else None
    xb0 = xb.clone(); rb0 = rb.clone() if fused else None
    wd = w.cuda()
    _norm(fused, xb[:T], rb[:T] if fused else None, wd, eps)
    torch.cuda.synchronize()
    # rows past T untouched
    assert torch.equal(RO.bits(xb[T:]), RO.bits(xb0[T:]))
    s = x
    if fused:
        assert torch.equal(RO.bits(rb[T:]), RO.bits(rb0[T:]))
        s = RO.add_residual(x, r)
        assert torch.equal(RO.bits(rb[:T].cpu()), RO.bits(s)), "residual h(x + r)"
    out = xb[:T].cpu()
    ok = RO.rmsnorm_ok(out, s, w, eps)
    assert bool(ok.all()), _report(ok, "x_out")
    # each row alone gives the same bits: a row's result is a function of the row
    xs = [xb0[t:t + 1].clone() for t in range(T)]
    rs = [rb0[t:t + 1].clone() for t in range(T)] if fused else [None] * T
    for t in range(T):
        _norm(fused, xs[t], rs[t], wd, eps)
    assert torch.equal(RO.bits(torch.cat(xs).cpu()), RO.bits(out))
    if fused:
        assert torch.equal(RO.bits(torch.cat(rs).cpu()), RO.bits(s))


# Model MLP widths (Llama-3-8B 14336, Llama-3-70B 28672, Qwen2-7B 18944) and their tensor-parallel shards, then odd vector
# counts with odd T: each thread takes two vectors, so pairs straddle rows and the last thread has one.
SILU_CASES = ([(F, T) for F in (14336, 7168, 3584, 1792, 28672, 18944, 9472, 4736) for T in (1, 64, 257)]
              + [(F, T) for F in (8, 24, 40, 1032) for T in (1, 7, 33, 301)])


@pytest.mark.parametrize("dt", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("F,T", SILU_CASES, ids=[f"F{f}-T{t}" for f, t in SILU_CASES])
def test_silu_and_mul_against_fp64(F, T, dt):
    from swiftllm_b200.worker.kernels.silu_and_mul import silu_and_mul_inplace
    x = RO.silu_inputs(T, F, dt, seed=F * 3 + T)
    xb = _fill(T, 2 * F, dt, x, seed=F + T)
    xb0 = xb.clone()
    silu_and_mul_inplace(xb[:T])
    torch.cuda.synchronize()
    assert torch.equal(RO.bits(xb[T:]), RO.bits(xb0[T:]))
    y = xb[:T].cpu()
    assert torch.equal(RO.bits(y[:, F:]), RO.bits(x[:, F:])), "gate half"
    ok = RO.silu_and_mul_ok(y[:, :F], x[:, :F], x[:, F:])
    assert bool(ok.all()), _report(ok, "h(up * h(silu))")
