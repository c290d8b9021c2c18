"""GPU: the log-probability kernel (csrc/logprobs.cu) against the numpy restatement and fp64 log_softmax
(tests/logprobs_oracle.py), and LlamaModel.forward_with_logprobs (eager, CUDA graph, chunked and mixed batches, sampled rows)
against log_softmax of the model's own logits."""
import numpy as np
import pytest
import torch

import logprobs_oracle as LO

pytestmark = pytest.mark.gpu


def _run(logits, tokens, n):
    from swiftllm_b200.worker.kernels.logprobs import token_logprobs
    tl, ids, tlp = token_logprobs(logits, torch.as_tensor(tokens, dtype=torch.int64, device=logits.device), n)
    return tl.cpu().numpy(), ids.cpu().numpy(), tlp.cpu().numpy()


def _same(a, b):
    """Bit-identical (NaN == NaN)."""
    return all(np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x, y.view(np.uint32) if y.dtype == np.float32 else y)
               for x, y in zip(a, b))


def _close_to_fp64(got, ref64, what):
    fin = np.isfinite(ref64)
    assert (got[~fin] == ref64[~fin]).all(), what
    err = np.abs(got[fin].astype(np.float64) - ref64[fin]).max(initial=0)
    assert err <= LO.TOL, (what, err)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V", [1000, 32001, 128256, 16032])
@pytest.mark.parametrize("B", [1, 3, 64, 257])
def test_kernel_matches_the_restatement(B, V, dtype):
    g = torch.Generator(device="cuda").manual_seed(B * 3 + V)
    logits = (torch.randn((B, V), generator=g, device="cuda") * 2.5).to(dtype)
    logits[:, ::97] = logits[:, 5:6]                       # repeated values
    if B > 1:
        logits[1, ::40] = logits[1].max()                  # the maximum repeated: ties at every top-N boundary
        logits[1, 3] = -0.0
    rng = np.random.default_rng(B + V)
    tokens = rng.integers(0, V, size=B)
    tokens[0] = int(torch.argmax(logits[0]))
    ref64 = LO.log_softmax64(logits)
    rows = np.arange(B)
    for n in (0, 1, 5, 20):
        got = _run(logits, tokens, n)
        assert _same(got, _run(logits, tokens, n)), "not deterministic run to run"
        tl, ids, tlp = got
        want_tl, want_ids, _ = LO.token_logprobs(logits, tokens, n)
        assert np.array_equal(ids, want_ids), n
        _close_to_fp64(tl, ref64[rows, tokens], ("token", n))
        _close_to_fp64(tlp, np.take_along_axis(ref64, ids.astype(np.int64), axis=1), ("top", n))
        _close_to_fp64(want_tl, ref64[rows, tokens], ("restatement", n))
        hit = ids == tokens[:, None]
        assert np.array_equal(tlp[hit].view(np.uint32), np.repeat(tl, hit.sum(axis=1)).view(np.uint32))
        if n:
            assert ids[0, 0] == tokens[0] and tlp[0, 0] == tl[0]           # the argmax token is top[0]
        for r in range(min(B, 3)):                                           # a row alone == the same row in the batch
            alone = _run(logits[r:r + 1], tokens[r:r + 1], n)
            assert _same(alone, (tl[r:r + 1], ids[r:r + 1], tlp[r:r + 1])), (r, n)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_nan_inf_and_out_of_range_rows(dtype):
    V = 32001
    logits = (torch.randn((7, V), device="cuda") * 3).to(dtype)
    logits[0, 100] = float("nan")
    logits[1, 31999] = float("inf")
    logits[2, :] = -float("inf")
    logits[3, ::2] = -float("inf")
    logits[4, 7] = -float("nan")
    tokens = [100, 5, 0, 0, 3, -1, V]
    tl, ids, tlp = _run(logits, tokens, 20)
    want_tl, want_ids, want_tlp = LO.token_logprobs(logits, tokens, 20)
    assert np.array_equal(ids, want_ids)
    assert np.isnan(tl[[0, 1, 2, 4]]).all() and np.isnan(tlp[[0, 1, 2, 4]]).all()
    assert tl[3] == -np.inf and np.isfinite(tlp[3]).all()
    assert np.isnan(tl[5:]).all() and np.isfinite(tlp[5:]).all()
    _close_to_fp64(tlp[3:4], np.take_along_axis(LO.log_softmax64(logits[3:4]), ids[3:4].astype(np.int64), axis=1), "row 3")
    # fewer entries than top_n: the rest are id -1, NaN
    small = logits[5:7, :7].contiguous()
    tl, ids, tlp = _run(small, [1, 2], 20)
    assert (ids[:, 7:] == -1).all() and np.isnan(tlp[:, 7:]).all()
    assert np.array_equal(ids, LO.token_logprobs(small, [1, 2], 20)[1])


def test_row_strided_logits():
    V = 16032
    big = torch.randn((5, V + 64), device="cuda").to(torch.bfloat16)
    view = big[:, 8:V + 8]
    got = _run(view, [1, 2, 3, 4, 5], 5)
    assert _same(got, _run(view.contiguous(), [1, 2, 3, 4, 5], 5))


# ---------------------------------------------------------------- through LlamaModel
def _models():
    from test_sampling_gpu import _model, _weights
    w = _weights()
    return _model(False, w=w), _model(True, w=w), _model(True, w=w)


def _lp_params(n, shift=0):
    from swiftllm_b200 import SamplingParams
    c = [SamplingParams(0.0, logprobs=5), SamplingParams(0.8, seed=21, logprobs=0), SamplingParams(1.3, top_k=9, seed=22, logprobs=20),
         SamplingParams(0.7, top_p=0.85, seed=23), SamplingParams(1.0, top_k=40, top_p=0.9, seed=24, logprobs=3),
         SamplingParams(0.0, logprobs=1)]
    return [c[(i + shift) % len(c)] for i in range(n)]


def _check(m, res, sp):
    ref = torch.log_softmax(m.post_layer.last_logits.double(), dim=1).cpu().numpy()
    for i, (r, p) in enumerate(zip(res, sp)):
        if p.logprobs is None:
            assert r.logprob is None and r.top is None
            continue
        assert abs(r.logprob - ref[i, r.token]) <= LO.TOL
        assert len(r.top) == p.logprobs
        ids = [t for t, _ in r.top]
        assert ids == sorted(range(ref.shape[1]), key=lambda v: (-ref[i, v], v))[:p.logprobs]
        assert all(abs(lp - ref[i, t]) <= LO.TOL for t, lp in r.top)
        if r.token in ids:
            assert r.top[ids.index(r.token)][1] == r.logprob
        if p.temperature == 0 and r.top:
            assert r.top[0] == (r.token, r.logprob)


def test_model_logprobs_eager_graph_chunked_and_mixed():
    from test_model_gpu import _script
    eager, graph, plain = _models()
    for m in (eager, graph):
        m.post_layer.keep_logits = True
    rng = np.random.default_rng(4)
    prompts = _script(rng); sids = [3, 9, 0]
    sp = _lp_params(3)
    a = eager.forward_with_logprobs(prompts, sids, [], sampling_params_list=sp)
    b = graph.forward_with_logprobs(prompts, sids, [], sampling_params_list=sp)
    c = plain.forward(prompts, sids, [], sampling_params_list=sp)
    assert a == b and [r.token for r in a] == c
    _check(eager, a, sp)
    lens = [len(p) for p in prompts]
    for step in range(8):                                   # decode: graph replay vs eager, and tokens == forward()
        lens = [l + 1 for l in lens]
        sp = _lp_params(3, step)
        ids = [[r.token] for r in a]
        a = eager.forward_with_logprobs(ids, sids, lens, sampling_params_list=sp)
        b = graph.forward_with_logprobs(ids, sids, lens, sampling_params_list=sp)
        c = plain.forward(ids, sids, lens, sampling_params_list=sp)
        assert a == b, step
        assert [r.token for r in a] == c, step
        assert torch.equal(eager.post_layer.last_logits, graph.post_layer.last_logits)
        _check(eager, a, sp)
    assert all(k[-2] == "logprobs" for k in graph._graphs)
    assert {k[-1] for k in graph._graphs} == {20, 5, 3}            # one graph per per-launch N
    assert all("logprobs" not in k for k in plain._graphs)  # forward() keeps its graphs
    # mixed: chunked prefill of a new prompt + the three decodes; then prefill only
    p4 = rng.integers(0, 1000, size=50).tolist()
    eager.forward([p4[:20]], [5], [], prefill_prefix_lens_list=[0])
    lens = [l + 1 for l in lens]
    sp = _lp_params(4, 1)
    t = eager.forward_with_logprobs([p4[20:50]] + [[r.token] for r in a], [5] + sids, lens, prefill_prefix_lens_list=[20],
                                    sampling_params_list=sp)
    _check(eager, t, sp)
    sp = _lp_params(2, 2)
    t = eager.forward_with_logprobs([p4[:7], p4[:30]], [1, 2], [], sampling_params_list=sp)
    _check(eager, t, sp)


def _tp_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    import swiftllm_b200
    from swiftllm_b200.worker.weight import synthetic_getter
    from test_tp_gpu import CFG
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    out = []
    for graph in (False, True):
        ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=2,
                                        max_seqs_in_block_table=8, max_blocks_per_seq=16, max_batch_size=4, max_tokens_in_batch=256,
                                        dtype="bfloat16", tp_size=world, tp_rank=rank, use_cuda_graph=graph, shard_lm_head=True)
        m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(CFG))
        m.load_weights(synthetic_getter(seed=11, std=0.05, device=f"cuda:{rank}"))
        m.init_kvcache_and_swap(40)
        res = m.forward_with_logprobs([[1, 2, 3, 4, 5], [7, 8], [9] * 20], [0, 1, 2], [], sampling_params_list=_lp_params(3, 1))
        seq = [res]
        lens = [5, 2, 20]
        for step in range(4):
            lens = [l + 1 for l in lens]
            ids = [[r.token] for r in res]
            sp = _lp_params(3, step)
            plain = m.forward(ids, [0, 1, 2], lens, sampling_params_list=sp)     # the same step twice: same KV writes
            res = m.forward_with_logprobs(ids, [0, 1, 2], lens, sampling_params_list=sp)
            assert [r.token for r in res] == plain
            seq.append(res)
        out.append(seq)
    got = [None] * world
    dist.all_gather_object(got, out)
    if rank == 0:
        q.put(got)
    dist.destroy_process_group()


def test_tensor_parallel_ranks_return_identical_logprobs():
    """Two GPUs, vocabulary-sharded lm_head: every rank returns the same tokens and log-probabilities (eager and graph), and
    the tokens are forward()'s."""
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_tp_worker, args=(r, 2, 29941, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        got = q.get(timeout=420)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.exitcode is None:
                p.kill()
    assert all(p.exitcode == 0 for p in procs)
    assert got[0] == got[1]
