"""GPU: the three tensor-parallel exchange kernels - one-shot and two-shot (csrc/allreduce_norm.cu) and LL push
(csrc/allreduce_ll.cu) - held to the restatement in tests/exchange_oracle.py on ONE GPU.

Each kernel reaches its peers only through the pointer arrays the host passes, so every rank of a world of 2..8 can be given
its own buffers on one device and launched one after the other through the C ABI (as worker/tp_comm.py calls it, without a
process group or symmetric memory).  The kernels wait on two kinds of memory only: flags (one-shot, two-shot) and tagged
receive lines (LL).  Every test writes those BEFORE a launch so that each wait is already satisfied - flags "ahead" of the
epoch, receive lines tagged with it - whatever a kernel's indexing does: no launch can spin, and a wrong index shows up as a
wrong value.  Ranks are never launched concurrently and nothing relies on CTAs being co-resident.  Checked, per rank:
every byte the kernel writes (residual, x_out, the flags it publishes, the lines it pushes into its peers' receive
buffers, its epoch state) and that it writes nothing else.

The NVLS variants (multimem loads / stores through an NVSwitch multicast object) cannot run on one GPU; tests/test_tp_gpu.py
covers them on a multi-GPU machine."""
import ctypes
import functools

import pytest
import torch

import exchange_oracle as X

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.float16, torch.bfloat16]
EPS = 1e-5
E = 0x2345              # epoch of a single exchange under test: the epoch state holds E - 1 before the launch
AHEAD = 1000            # flags pre-filled with epoch + AHEAD: a peer that is "ahead" never makes a rank wait
EXTRA_ROWS = 3          # rows past the T in use in x_out / residual: a kernel must leave them alone

# (N, H, T).  H = 8: 1 vector / 32 threads;  1032: 129 vectors, 160 threads (ragged loop);  4096: 512 threads;  8192: two
# vectors per thread;  24544 / 24552 / 24576: the 48 KB edge, where the row plus the kernel's static shared memory (64 B, two-shot
# 80 B) first needs the raised limit;  28672: 56 KB of dynamic shared memory (the LL kernel refuses it).  The raised limit lasts
# for the process, so the edge cases come before the 28672 ones: after 28672 they would pass without testing the launcher.
# T = N - 1 leaves a rank without a row to own;  T = None stands for 2 * SMs + 5 (LL: CTAs loop over several rows);
# T = 1024 is the largest LL exchange (MAX_LL_TOKENS).
FLAG_CASES = [(2, 8, 1), (8, 4096, 1), (3, 1032, 2), (4, 4096, 5), (8, 8192, 7), (8, 1032, 131), (2, 4096, 131),
              (3, 8192, 131), (2, 24544, 3), (3, 24552, 2), (4, 24576, 5), (3, 28672, 4), (4, 28672, 3), (8, 28672, 9), (4, 8192, 1024), (2, 1032, 1024), (8, 8, 1024)]
LL_CASES = [(2, 8, 1), (8, 4096, 1), (3, 1032, 2), (4, 4096, 5), (8, 8192, 7), (8, 1032, 131), (2, 8, 131), (2, 24544, 3),
            (3, 24552, 2), (4, 24576, 5), (2, 4096, None),
            (4, 1032, None), (8, 8192, None), (4, 8192, 1024), (3, 4096, 1024), (8, 8, 1024)]


def _case_id(c):
    return "N%d-H%d-T%s" % (c[0], c[1], "2sm+5" if c[2] is None else c[2])


@functools.lru_cache(maxsize=1)
def _lib():
    from swiftllm_b200 import _lib
    _lib.require_device(torch.empty(1, device=DEV))
    return _lib


def _resolve_T(T):
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count + 5 if T is None else T


def _ptrs(ts):
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _junk(shape, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = torch.randint(-2 ** 31, 2 ** 31 - 1, shape, dtype=torch.int32, device=DEV, generator=g)
    return w.view(dtype) if dtype != torch.int32 else w


@functools.lru_cache(maxsize=6)
def _reference(N, T, H, dtype, seed=0):
    """Inputs and the restatement's (x_out, residual), on the device."""
    P, R, w = X.make_inputs(N, T, H, dtype, seed)
    x_ref, r_ref = X.exchange_add_norm(list(P), R, w, EPS)
    return P.to(DEV), R.to(DEV), w.to(DEV), x_ref.to(DEV), r_ref.to(DEV)


class Ranks:
    """Per-rank buffers of a world of N on one device: residual and x_out [T + EXTRA_ROWS, H] (junk past T; x_out junk
    everywhere), epoch state uint32[32] (junk outside the slots in use)."""

    def __init__(self, N, T, H, dtype, R):
        self.N, self.T, self.H, self.dtype = N, T, H, dtype
        self.res = torch.cat((R, _junk((EXTRA_ROWS, H // 2), dtype, 1).view(EXTRA_ROWS, H))).repeat(N, 1, 1)
        self.xo = _junk((N, T + EXTRA_ROWS, H // 2), dtype, 2).view(N, T + EXTRA_ROWS, H)
        self.res0, self.xo0 = self.res.clone(), self.xo.clone()
        self.epoch = _junk((N, 32), torch.int32, 3)

    def set_epoch(self, slot, last):
        self.epoch[:, slot] = X.as_i32(last)
        self.epoch[:, 16 + slot] = 0

    def rows(self, rank=None):
        """[T + EXTRA_ROWS] mask of the rows < T (owned by `rank`, if given)."""
        t = torch.arange(self.T + EXTRA_ROWS, device=DEV)
        return (t < self.T) & ((t % self.N == rank) if rank is not None else True)


def _check(rc, what):
    _lib().check(rc, what)
    torch.cuda.synchronize()


def _pads(N, e):
    """Signal pads of every rank, uint32 [16 rows][8 ranks], all "ahead" of epoch e."""
    return torch.full((N, 16 * 8), X.as_i32(e + AHEAD), dtype=torch.int32, device=DEV)


def _expect_epoch(before, r, slot, e):
    exp = before.clone()
    exp[r, slot] = X.as_i32(e)
    exp[r, 16 + slot] = 0
    return exp


# ----------------------------------------------------------------------------- launch every rank in sequence
def run_one_shot(P, w, rk: Ranks, slot, e, with_weight=True):
    """One exchange: ranks 0..N-1 in sequence.  After rank r: rank r's flag for epoch e is in slot row `slot` of every pad and
    nothing else in any pad has changed; r's epoch advanced once, its done counter is back to 0."""
    L, N, T, H = _lib(), rk.N, rk.T, rk.H
    pads = _pads(N, e)
    expect = pads.clone()
    bufs, flags = _ptrs(list(P)), _ptrs(list(pads))
    for r in range(N):
        before = rk.epoch.clone()
        _check(L.lib().sllm_allreduce_add_rmsnorm(
            ctypes.cast(bufs, ctypes.c_void_p), ctypes.cast(flags, ctypes.c_void_p), r, N, slot, rk.epoch[r].data_ptr(),
            rk.xo[r].data_ptr(), rk.res[r].data_ptr(), w.data_ptr() if with_weight else None, EPS, T, H,
            L.dtype_tag(rk.dtype), L.stream()), "allreduce_add_rmsnorm")
        expect[:, slot * 8 + r] = X.as_i32(e)
        assert torch.equal(pads, expect), f"one-shot rank {r}: flags"
        assert torch.equal(rk.epoch, _expect_epoch(before, r, slot, e)), f"one-shot rank {r}: epoch state"


def run_two_shot(P, w, rk: Ranks, slot, e, x_expect=None):
    """One exchange: ranks 0..N-1 in sequence.  After rank r, every rank's x_out holds `x_expect` on the rows owned by ranks
    0..r (when given) and its old content everywhere else; the flags of barriers A (row slot) and B (row 8 + slot) are
    published in every pad - by ranks that own no row too."""
    L, N, T, H = _lib(), rk.N, rk.T, rk.H
    pads = _pads(N, e)
    expect = pads.clone()
    bufs, flags, xouts = _ptrs(list(P)), _ptrs(list(pads)), _ptrs(list(rk.xo))
    t = torch.arange(T + EXTRA_ROWS, device=DEV)
    xo_before = rk.xo.clone()
    for r in range(N):
        before = rk.epoch.clone()
        _check(L.lib().sllm_allreduce_add_rmsnorm_2shot(
            ctypes.cast(bufs, ctypes.c_void_p), ctypes.cast(xouts, ctypes.c_void_p), ctypes.cast(flags, ctypes.c_void_p), None, None,
            r, N, slot, rk.epoch[r].data_ptr(), rk.res[r].data_ptr(), w.data_ptr(), EPS, T, H, L.dtype_tag(rk.dtype),
            L.stream()), "allreduce_add_rmsnorm_2shot")
        expect[:, slot * 8 + r] = X.as_i32(e)
        expect[:, (8 + slot) * 8 + r] = X.as_i32(e)
        assert torch.equal(pads, expect), f"two-shot rank {r}: flags"
        assert torch.equal(rk.epoch, _expect_epoch(before, r, slot, e)), f"two-shot rank {r}: epoch state"
        if x_expect is not None:
            done = ((t < T) & (t % N <= r))[:, None]
            for k in range(N):
                want = torch.where(done, torch.cat((x_expect, xo_before[k, T:])), xo_before[k])
                assert torch.equal(X.bits(rk.xo[k]), X.bits(want)), f"two-shot after rank {r}: x_out of rank {k}"


def run_ll(P, w, rk: Ranks, slot, e, rows_per_rank, max_tokens, seed=0):
    """One exchange: ranks 0..N-1 in sequence.  Before rank r's launch, every line of r's own receive buffers is tagged e:
    rs_recv carries the peers' partial rows where they would have pushed them, ag_recv random rows G[t] for the rows r does not
    own, everything else junk; every peer's receive buffers are zero.  After it: the non-owned rows of r's x_out are G, its
    own buffers are unchanged, and each peer's buffers hold exactly r's pushes (rs_recv: its partial rows that peer owns;
    ag_recv: r's normalised rows) and zeros elsewhere."""
    L, N, T, H, dtype = _lib(), rk.N, rk.T, rk.H, rk.dtype
    rs = torch.zeros(N, N, rows_per_rank, H, dtype=torch.int32, device=DEV)
    ag = torch.zeros(N, max_tokens, H, dtype=torch.int32, device=DEV)
    rs_p, ag_p = _ptrs(list(rs)), _ptrs(list(ag))
    for r in range(N):
        rs.zero_(); ag.zero_()
        rs[r] = _junk((N, rows_per_rank, H), torch.int32, 100 * seed + 2 * r + 10)
        ag[r] = _junk((max_tokens, H), torch.int32, 100 * seed + 2 * r + 11)
        rs[r].view(N, rows_per_rank, H // 2, 2)[..., 1] = X.as_i32(e)
        ag[r].view(max_tokens, H // 2, 2)[..., 1] = X.as_i32(e)
        mine = X.owned_rows(T, N, r, DEV)
        for s in range(N):
            if s != r:
                rs[r, s, mine // N] = X.ll_pack(P[s][mine], e)
        others = torch.nonzero(~X.owned(T, N, r, DEV)).flatten()
        G = _junk((T, H // 2), dtype, 100 * seed + r + 50).view(T, H)
        ag[r, others] = X.ll_pack(G[others], e)
        rs_mine, ag_mine, before = rs[r].clone(), ag[r].clone(), rk.epoch.clone()
        xo_before = rk.xo[r].clone()
        _check(L.lib().sllm_allreduce_add_rmsnorm_ll(
            P[r].data_ptr(), ctypes.cast(rs_p, ctypes.c_void_p), ctypes.cast(ag_p, ctypes.c_void_p), None, r, N, slot,
            rk.epoch[r].data_ptr(), rk.xo[r].data_ptr(), rk.res[r].data_ptr(), w.data_ptr(), EPS, T, H, rows_per_rank,
            L.dtype_tag(dtype), L.stream()), "allreduce_add_rmsnorm_ll")
        assert torch.equal(rk.epoch, _expect_epoch(before, r, slot, e)), f"LL rank {r}: epoch state"
        assert torch.equal(X.bits(rk.xo[r, others]), X.bits(G[others])), f"LL rank {r}: phase-3 rows of x_out"
        assert torch.equal(X.bits(rk.xo[r, T:]), X.bits(xo_before[T:])), f"LL rank {r}: x_out rows >= T"
        assert torch.equal(rs[r], rs_mine) and torch.equal(ag[r], ag_mine), f"LL rank {r}: wrote its own receive buffers"
        for k in range(N):
            if k != r:
                assert torch.equal(rs[k], X.ll_rs_image(P[r], r, k, N, rows_per_rank, e)), f"LL rank {r}: rs_recv of rank {k}"
                assert torch.equal(ag[k], X.ll_ag_image(rk.xo[r, :T], r, k, N, max_tokens, e)), f"LL rank {r}: ag_recv of rank {k}"


# ----------------------------------------------------------------------------- one exchange, every shape
def _diff(got, want):
    """Where two row blocks differ: count and the first few (row, column, got, want)."""
    bad = torch.nonzero(X.bits(got) != X.bits(want))
    return f"{len(bad)} values differ, first: " + ", ".join(
        f"[{int(i)}, {int(j)}] {float(got[i, j])!r} vs {float(want[i, j])!r}" for i, j in bad[:4].tolist())


def _check_rows(rk: Ranks, r, rows, x_ref, r_ref, what, x=True):
    """Rank r against the restatement on `rows` (< T): residual bit for bit, x_out within 1 ulp; the rest of its residual
    keeps its old content."""
    got, want = rk.res[r, rows], r_ref[rows[: rk.T]]
    assert torch.equal(X.bits(got), X.bits(want)), f"{what}: residual of rank {r}: {_diff(got, want)}"
    assert torch.equal(X.bits(rk.res[r, ~rows]), X.bits(rk.res0[r, ~rows])), f"{what}: residual rows of rank {r} it does not own"
    if x:
        got, want = rk.xo[r, rows], x_ref[rows[: rk.T]]
        assert X.ulp_distance(got, want) <= 1, f"{what}: x_out of rank {r}: {_diff(got, want)}"


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", FLAG_CASES, ids=_case_id)
def test_one_shot_vs_restatement(case, dtype):
    N, H, T = case
    P, R, w, x_ref, r_ref = _reference(N, T, H, dtype)
    rk = Ranks(N, T, H, dtype, R)
    rk.set_epoch(0, E - 1)
    run_one_shot(P, w, rk, 0, E)
    for r in range(N):
        _check_rows(rk, r, rk.rows(), x_ref, r_ref, "one-shot")
        assert torch.equal(X.bits(rk.xo[r, :T]), X.bits(rk.xo[0, :T])), f"one-shot: x_out of rank {r} differs from rank 0's"
        assert torch.equal(X.bits(rk.xo[r, T:]), X.bits(rk.xo0[r, T:])), f"one-shot: x_out rows >= T of rank {r}"


@pytest.mark.parametrize("dtype", DTYPES)
def test_one_shot_without_weight_only_updates_the_residual(dtype):
    N, H, T = 3, 1032, 4
    P, R, w, x_ref, r_ref = _reference(N, T, H, dtype)
    rk = Ranks(N, T, H, dtype, R)
    rk.set_epoch(5, E - 1)
    run_one_shot(P, w, rk, 5, E, with_weight=False)
    for r in range(N):
        _check_rows(rk, r, rk.rows(), x_ref, r_ref, "one-shot, weight NULL", x=False)
    assert torch.equal(X.bits(rk.xo), X.bits(rk.xo0)), "one-shot with weight NULL wrote x_out"


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", FLAG_CASES, ids=_case_id)
def test_two_shot_vs_restatement_and_one_shot(case, dtype):
    """x_out is complete on every rank once all have run, bit-identical to the one-shot kernel's; each residual is the
    restatement's on the rows its rank owns and untouched on the others."""
    N, H, T = case
    P, R, w, x_ref, r_ref = _reference(N, T, H, dtype)
    one = Ranks(N, T, H, dtype, R)
    one.set_epoch(0, E - 1)
    run_one_shot(P, w, one, 0, E)
    rk = Ranks(N, T, H, dtype, R)
    rk.set_epoch(3, E - 1)
    run_two_shot(P, w, rk, 3, E, x_expect=one.xo[0, :T])
    for r in range(N):
        _check_rows(rk, r, rk.rows(r), x_ref, r_ref, "two-shot")
        assert torch.equal(X.bits(rk.xo[r, :T]), X.bits(one.xo[0, :T])), f"two-shot: x_out of rank {r} differs from one-shot"


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", LL_CASES, ids=_case_id)
def test_ll_vs_restatement_and_two_shot(case, dtype):
    N, H, T = case
    T = _resolve_T(T)
    P, R, w, x_ref, r_ref = _reference(N, T, H, dtype)
    two = Ranks(N, T, H, dtype, R)
    two.set_epoch(1, E - 1)
    run_two_shot(P, w, two, 1, E)
    rk = Ranks(N, T, H, dtype, R)
    rk.set_epoch(9, E - 1)
    # one spare row per source in rs_recv and two in ag_recv: pushes must land at [src][t // N] / [t], not at a packed index
    run_ll(P, w, rk, 9, E, rows_per_rank=(T + N - 1) // N + 1, max_tokens=T + 2)
    for r in range(N):
        mine = rk.rows(r)
        _check_rows(rk, r, mine, x_ref, r_ref, "LL")
        assert torch.equal(X.bits(rk.xo[r, mine]), X.bits(two.xo[r, mine])), f"LL: owned rows of rank {r} differ from two-shot"


@pytest.mark.parametrize("dtype", DTYPES)
def test_ll_rejects_a_row_too_large_for_shared_memory(dtype):
    """24584 is the first width past the 48 KB row the LL check accepts (LL_CASES runs 24576); 28672 is a model's."""
    L, N, T = _lib(), 2, 2
    for H in (24584, 28672):
        x = torch.zeros(T, H, dtype=dtype, device=DEV)
        st = torch.zeros(32, dtype=torch.int32, device=DEV)
        bufs = _ptrs([x, x])
        rc = L.lib().sllm_allreduce_add_rmsnorm_ll(x.data_ptr(), ctypes.cast(bufs, ctypes.c_void_p), ctypes.cast(bufs, ctypes.c_void_p),
                                                   None, 0, N, 0, st.data_ptr(), x.data_ptr(), x.data_ptr(), x[0].data_ptr(), EPS, T,
                                                   H, 1, L.dtype_tag(dtype), L.stream())
        assert rc != 0 and b"too large" in L.lib().sllm_last_error(), H
        torch.cuda.synchronize()
        assert int(st.abs().sum()) == 0 and int(x.abs().sum()) == 0, H


# ----------------------------------------------------------------------------- epochs
@pytest.mark.parametrize("kernel", ["one_shot", "two_shot", "ll"])
def test_consecutive_exchanges_across_the_epoch_wrap(kernel):
    """Six exchanges alternating slots 0 and 1 with fresh partials, from epoch state 0xFFFFFFFC: the flags the test pre-fills
    (epoch + 1000) wrap past 2^32 and must still read as "ahead", every launch advances its slot's epoch exactly once and leaves
    the other slot's alone, and the residual carries from one exchange to the next."""
    N, H, T, dtype = 3, 1032, 5, torch.float16
    P, R, w, _, _ = _reference(N, T, H, dtype, 1)
    rk = Ranks(N, T, H, dtype, R)
    rk.set_epoch(0, 0xFFFFFFFC); rk.set_epoch(1, 0xFFFFFFFC)
    r_ref = R
    for k in range(6):
        slot, e = k % 2, (0xFFFFFFFC + 1 + k // 2) & 0xFFFFFFFF
        P = X.make_inputs(N, T, H, dtype, seed=10 + k)[0].to(DEV)
        x_ref, r_ref = X.exchange_add_norm(list(P), r_ref, w, EPS)
        if kernel == "one_shot":
            run_one_shot(P, w, rk, slot, e)
        elif kernel == "two_shot":
            run_two_shot(P, w, rk, slot, e)
        else:
            run_ll(P, w, rk, slot, e, rows_per_rank=(T + N - 1) // N, max_tokens=T, seed=k)
        assert rk.epoch[:, slot].tolist() == [X.as_i32(e)] * N
        assert rk.epoch[:, 1 - slot].tolist() == [X.as_i32(0xFFFFFFFC + (k + 1) // 2)] * N
        for r in range(N):
            rows = rk.rows() if kernel == "one_shot" else rk.rows(r)
            assert torch.equal(X.bits(rk.res[r, rows]), X.bits(r_ref[rows[:T]])), f"exchange {k}: residual of rank {r}"
            assert X.ulp_distance(rk.xo[r, rows], x_ref[rows[:T]]) <= 1, f"exchange {k}: x_out of rank {r}"


def test_two_shot_graph_replay_advances_the_epoch():
    """One rank's two-shot launch captured in a CUDA graph and replayed 3 times: the epoch lives in device memory, so each
    replay is a new exchange - epoch and published flags reach e0 + 3, and the residual has taken 3 exchanges."""
    L, N, H, T, dtype, slot, e0 = _lib(), 2, 1032, 3, torch.bfloat16, 1, 0x7FFFFFF0
    P, R, w, _, _ = _reference(N, T, H, dtype)
    rk = Ranks(N, T, H, dtype, R)
    rk.set_epoch(slot, e0)
    pads = torch.full((N, 16 * 8), X.as_i32(e0 + 2 ** 30), dtype=torch.int32, device=DEV)
    bufs, flags, xouts = _ptrs(list(P)), _ptrs(list(pads)), _ptrs(list(rk.xo))
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        rc = L.lib().sllm_allreduce_add_rmsnorm_2shot(
            ctypes.cast(bufs, ctypes.c_void_p), ctypes.cast(xouts, ctypes.c_void_p), ctypes.cast(flags, ctypes.c_void_p), None, None,
            0, N, slot, rk.epoch[0].data_ptr(), rk.res[0].data_ptr(), w.data_ptr(), EPS, T, H, L.dtype_tag(dtype), L.stream())
    assert rc == 0, L.lib().sllm_last_error()
    torch.cuda.synchronize()
    assert int(rk.epoch[0, slot]) == X.as_i32(e0)                  # captured, not run
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    assert int(rk.epoch[0, slot]) == X.as_i32(e0 + 3) and int(rk.epoch[0, 16 + slot]) == 0
    expect = torch.full_like(pads, X.as_i32(e0 + 2 ** 30))
    expect[:, slot * 8] = X.as_i32(e0 + 3)
    expect[:, (8 + slot) * 8] = X.as_i32(e0 + 3)
    assert torch.equal(pads, expect)
    r_ref = R
    for _ in range(3):
        x_ref, r_ref = X.exchange_add_norm(list(P), r_ref, w, EPS)
    rows = rk.rows(0)
    _check_rows(rk, 0, rows, x_ref, r_ref, "graph replay")
    assert torch.equal(X.bits(rk.xo[1, rows]), X.bits(rk.xo[0, rows]))
    assert torch.equal(X.bits(rk.xo[1, ~rows]), X.bits(rk.xo0[1, ~rows]))
