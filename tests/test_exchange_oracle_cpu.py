"""CPU: the restatement of the tensor-parallel exchange (tests/exchange_oracle.py) against the gloo stand-in that every CPU
tensor-parallel test runs on (tests/cpu_shim.py: GlooFusedAllReduce), and proof that the data of the GPU exchange tests
(tests/test_exchange_kernels_gpu.py) tells the right summation order and rounding points from plausible wrong ones."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import exchange_oracle as X
import test_exchange_kernels_gpu as G

DTYPES = [torch.float16, torch.bfloat16]
EPS = 1e-5


def _gloo_worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import exchange_oracle as X
    from cpu_shim import GlooFusedAllReduce
    bad = []
    for dtype in DTYPES:
        for T, H in ((world - 1, 8), (world + 1, 1032), (131, 4096)):
            P, R, w = X.make_inputs(world, T, H, dtype)
            x_ref, r_ref = X.exchange_add_norm(list(P), R, w, EPS)
            for two_shot in (False, True):
                comm = GlooFusedAllReduce(T + 2, H, dtype, "cpu", two_shot=two_shot)
                slot = int(two_shot)
                comm.partial_out(slot, T).copy_(P[rank])
                res = R.clone()
                out = comm.reduce_add_norm(slot, T, res, w, EPS)
                rows = X.owned(T, world, rank) if two_shot else torch.ones(T, dtype=torch.bool)
                tag = f"{dtype} T={T} H={H} two_shot={two_shot} rank={rank}"
                if not torch.equal(X.bits(out), X.bits(x_ref)):
                    bad.append(f"x_out {tag}")
                if not torch.equal(X.bits(res[rows]), X.bits(r_ref[rows])):
                    bad.append(f"residual {tag}")
    gathered = [None] * world
    dist.all_gather_object(gathered, bad)
    if rank == 0:
        ret.put(gathered)
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_stand_in_matches_the_restatement_bit_for_bit(world):
    """x_out (every row) and the residual rows a rank maintains (all rows one-shot, its own rows two-shot) of the stand-in are
    the restatement's, bit for bit - so the CPU tensor-parallel tests built on it hold the product to the kernels' contract."""
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, 29840 + world, ret)) for r in range(world)]
    for p in procs:
        p.start()
    bad = ret.get(timeout=240)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert bad == [[]] * world, bad


# every (N, H, T) shape of the GPU tests; T = None there is 2 * SMs + 5, 269 on a 132-SM H100
SHAPES = sorted({(N, H, 269 if T is None else T) for N, H, T in G.FLAG_CASES + G.LL_CASES})


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "N%d-H%d-T%d" % s)
def test_exchange_data_tells_wrong_orders_and_roundings_apart(dtype, shape):
    """Each plausible mistake changes the residual, which the GPU tests compare bit for bit: a reversed or pairwise rank order
    (only meaningful from N = 3 on - two terms added to 0 commute) and a single rounding h(sum + R) instead of h(h(sum) + R).
    A test with ordinary random partials could pass the first two: their fp32 sums are exact."""
    N, H, T = shape
    P, R, w = X.make_inputs(N, T, H, dtype)
    parts = list(P)
    ref = X.exchange_add(parts, R)
    assert not torch.equal(X.bits(X.add_single_rounding(parts, R)), X.bits(ref))
    if N >= 3:
        assert not torch.equal(X.bits(X.sum_reversed(parts) + R), X.bits(ref))
        assert not torch.equal(X.bits(X.sum_pairwise(parts) + R), X.bits(ref))


def test_ll_pack_layout():
    """{w0, tag, w1, tag} lines, a row of H 16-bit values -> H int32 words; the push images put rows where the kernel's
    indexing (csrc/allreduce_ll.cu) puts them."""
    x = torch.arange(1, 17, dtype=torch.int16).view(torch.float16).reshape(2, 8)
    lines = X.ll_pack(x, 0xFFFFFFFE)
    words = x.view(torch.int32)
    assert lines.shape == (2, 8) and lines.dtype == torch.int32
    assert lines[0].tolist() == [int(words[0, 0]), -2, int(words[0, 1]), -2, int(words[0, 2]), -2, int(words[0, 3]), -2]
    payload, tags = X.ll_unpack(lines, torch.float16)
    assert torch.equal(X.bits(payload), X.bits(x)) and bool((tags == -2).all())
    N, T, H, rpr = 3, 7, 8, 4
    P = torch.randn(T, H).to(torch.bfloat16)
    img = X.ll_rs_image(P, src=2, dst=1, nranks=N, rows_per_rank=rpr, tag=5)
    for t in range(T):
        got = img[2, t // N]
        assert torch.equal(got, X.ll_pack(P[t], 5)) == (t % N == 1)
    assert int(img[:2].abs().sum()) == 0 and int(img[2, 3].abs().sum()) == 0
    assert int(X.ll_rs_image(P, 1, 1, N, rpr, 5).abs().sum()) == 0
    # T < N: a rank past the last row owns nothing, pushes nothing and receives nothing
    assert int(X.ll_rs_image(P[:2], 0, 2, N, rpr, 5).abs().sum()) == 0
    assert int(X.ll_ag_image(P[:2], 2, 0, N, 3, 5).abs().sum()) == 0
    ag = X.ll_ag_image(P, src=0, dst=2, nranks=N, max_tokens=T + 1, tag=9)
    for t in range(T + 1):
        assert torch.equal(ag[t], X.ll_pack(P[t], 9)) if t < T and t % N == 0 else int(ag[t].abs().sum()) == 0
