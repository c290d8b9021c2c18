"""GPU: the sampling kernel (csrc/sampling.cu) against the numpy restatement (tests/sampling_oracle.py), and sampling through
LlamaModel.forward (eager, CUDA graph, chunked prefill) against the restatement applied to the model's own logits."""
import numpy as np
import pytest
import torch

import sampling_oracle as SO

pytestmark = pytest.mark.gpu

KINDS = ["greedy", "temperature", "top_k", "top_p", "both"]


def _params(B, V, rng):
    kind = [KINDS[i % len(KINDS)] for i in range(B)]
    temp = [0.0 if k == "greedy" else float(rng.choice([0.5, 0.8, 1.0, 1.7])) for k in kind]
    top_k = [int(rng.choice([1, 5, 50, V // 3 + 1, V + 7])) if k in ("top_k", "both") else 0 for k in kind]
    top_p = [float(np.float32(rng.choice([1e-4, 0.3, 0.9, 0.95]))) if k in ("top_p", "both") else 1.0 for k in kind]
    seed = [int(x) for x in rng.integers(0, 2 ** 63, size=B)]
    pos = [int(x) for x in rng.integers(1, 5000, size=B)]
    return temp, top_k, top_p, seed, pos


def _run(logits, temp, top_k, top_p, seed, pos, vocab_offset=0, pairs=False):
    from swiftllm_b200.worker.kernels.sampling import sample_tokens
    d = logits.device
    out = torch.empty((logits.shape[0], 2), dtype=torch.float32, device=d) if pairs else None
    tok = sample_tokens(logits, torch.tensor(temp, dtype=torch.float32, device=d), torch.tensor(top_k, dtype=torch.int32, device=d),
                        torch.tensor(top_p, dtype=torch.float32, device=d), torch.tensor(seed, dtype=torch.int64, device=d),
                        torch.tensor(pos, dtype=torch.int32, device=d), vocab_offset=vocab_offset, out_pairs=out)
    return (tok, out) if pairs else tok


def _kept_by_kernel(logits, r, temp, top_k, top_p, pos, n_seeds=64):
    """Tokens the kernel can return for row r: union over seeds (a subset of the kept set; used to check it is inside)."""
    row = logits[r:r + 1].expand(n_seeds, -1).contiguous()
    toks = _run(row, [temp] * n_seeds, [top_k] * n_seeds, [top_p] * n_seeds, list(range(1, n_seeds + 1)), [pos] * n_seeds)
    return set(toks.tolist())


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V", [1000, 32000, 128256, 16032])
@pytest.mark.parametrize("B", [1, 3, 64, 257])
def test_kernel_matches_the_restatement(B, V, dtype):
    if B == 257 and V == 128256 and dtype == torch.float16:
        pytest.skip("covered by bf16 at this size (CPU restatement time)")
    rng = np.random.default_rng(B * 7 + V)
    g = torch.Generator(device="cuda").manual_seed(B + V)
    logits = (torch.randn((B, V), generator=g, device="cuda") * 2.5).to(dtype)
    logits[:, ::97] = logits[:, 5:6]                      # repeated values: ties at the top-k / top-p boundaries
    temp, top_k, top_p, seed, pos = _params(B, V, rng)
    tok = _run(logits, temp, top_k, top_p, seed, pos)
    again = _run(logits, temp, top_k, top_p, seed, pos)
    assert torch.equal(tok, again), "not deterministic run to run"
    greedy = [i for i in range(B) if temp[i] == 0]
    assert torch.equal(tok[greedy], torch.argmax(logits[greedy], dim=1))
    # a row alone == the same row inside the batch
    for r in range(min(B, 5)):
        alone = _run(logits[r:r + 1], temp[r:r + 1], top_k[r:r + 1], top_p[r:r + 1], seed[r:r + 1], pos[r:r + 1])
        assert int(alone) == int(tok[r])
    ref = SO.sample_tokens(logits, temp, top_k, top_p, seed, pos)
    got = tok.tolist()
    exempt = 0
    for r, res in enumerate(ref):
        if res.kept is not None and res.boundary_margin <= 1e-4:
            exempt += 1
            continue
        if got[r] != res.token:
            assert res.gap <= 1e-5 * abs(res.score), (r, got[r], res.token, res.gap, temp[r], top_k[r], top_p[r])
            exempt += 1
        if res.kept is not None:
            assert res.kept[got[r]], (r, "token outside the kept set")
    # kept sets: the tokens a row can produce over many seeds lie inside the restatement's kept set, and a kept set of one
    # token (k = 1, tiny p) is hit exactly
    for r in [i for i in range(min(B, 10)) if ref[i].kept is not None and ref[i].boundary_margin > 1e-4]:
        reach = _kept_by_kernel(logits, r, temp[r], top_k[r], top_p[r], pos[r])
        kept = set(np.nonzero(ref[r].kept)[0].tolist())
        assert reach <= kept, (r, sorted(reach - kept)[:5])
        if len(kept) == 1:
            assert reach == kept
    print(f"B={B} V={V} {dtype}: {exempt} of {B} rows exempt")
    assert exempt <= B // 2 + 2


def test_sharded_pairs_merge_to_the_unsharded_token():
    B, V, N = 16, 128256, 8
    Vs = V // N
    rng = np.random.default_rng(3)
    logits = (torch.randn((B, V), device="cuda") * 2).to(torch.bfloat16)
    temp = [0.0 if i % 4 == 0 else 0.9 for i in range(B)]
    seed = [int(x) for x in rng.integers(0, 2 ** 63, size=B)]
    pos = list(range(100, 100 + B))
    full = _run(logits, temp, [0] * B, [1.0] * B, seed, pos)
    pairs = torch.stack([_run(logits[:, n * Vs:(n + 1) * Vs].contiguous(), temp, [0] * B, [1.0] * B, seed, pos, vocab_offset=n * Vs,
                              pairs=True)[1] for n in range(N)])
    from swiftllm_b200.worker.layers.post_layer import merge_sharded_argmax
    assert torch.equal(merge_sharded_argmax(pairs), full)


def test_distribution_matches_the_filtered_softmax():
    from scipy.stats import chisquare
    V, S = 48, 20000
    logits = (torch.linspace(-2, 2, V, device="cuda") ** 3).to(torch.bfloat16)
    T, k, p = 0.9, 30, 0.9
    rows = logits[None].expand(S, V).contiguous()
    tok = _run(rows, [T] * S, [k] * S, [p] * S, list(range(S)), [17] * S).cpu().numpy()
    res = SO.sample_tokens(logits[None], [T], [k], [p], [0], [17])[0]
    kept = res.kept
    prob = np.where(kept, np.exp((logits.float().cpu().numpy() - logits.float().max().item()) / T), 0)
    prob /= prob.sum()
    assert kept[tok].all()
    cnt = np.bincount(tok, minlength=V)[kept]
    assert chisquare(cnt, prob[kept] * S).pvalue > 1e-3


def test_invalid_launch_arguments_raise():
    from swiftllm_b200 import _lib
    l = _lib.lib()
    assert l.sllm_sample_tokens(1, 2, 2_000_000, 2_000_000, 0, 1, 1, 1, 1, 1, 1, None, 1, None) != 0
    assert b"shared memory" in l.sllm_last_error()


# ---------------------------------------------------------------- through LlamaModel
def _model(graph=False, sampling_seed=0, w=None):
    import swiftllm_b200
    from test_model_gpu import ENG2, TINY2, _make_model
    m = _make_model(TINY2, ENG2, w, dtype="bfloat16", graph=graph)
    m.engine_config.sampling_seed = sampling_seed
    m._sampling_rng = np.random.default_rng(sampling_seed)
    return m


def _weights():
    from oracle.model import OracleWeights
    from test_model_gpu import TINY2
    return OracleWeights.random(TINY2, dtype=torch.bfloat16, seed=5, std=0.05)


def _sp(n, shift=0):
    from swiftllm_b200 import SamplingParams
    c = [SamplingParams(0.0), SamplingParams(0.8, seed=21), SamplingParams(1.3, top_k=9, seed=22),
         SamplingParams(0.7, top_p=0.85, seed=23), SamplingParams(1.0, top_k=40, top_p=0.9, seed=24)]
    return [c[(i + shift) % len(c)] for i in range(n)]


def _check(m, toks, sp, seq_lens, seeds=None):
    seeds = seeds if seeds is not None else [s.seed for s in sp]
    ref = SO.sample_tokens(m.post_layer.last_logits, [s.temperature for s in sp], [s.top_k for s in sp], [s.top_p for s in sp],
                           seeds, seq_lens)
    for t, r in zip(toks, ref):
        assert t == r.token or r.gap <= 1e-5 * abs(r.score) or r.boundary_margin <= 1e-4, (t, r.token, r.gap)


def test_model_sampling_matches_the_restatement_eager_graph_and_chunked():
    from swiftllm_b200 import SamplingParams
    from test_model_gpu import _script
    w = _weights()
    eager, graph = _model(False, w=w), _model(True, w=w)
    rng = np.random.default_rng(2)
    prompts = _script(rng); sids = [3, 9, 0]
    # all-greedy params == no params
    a = eager.forward(prompts, sids, [], sampling_params_list=[SamplingParams()] * 3)
    b = graph.forward(prompts, sids, [])
    assert a == b
    lens = [len(p) for p in prompts]
    sp = _sp(3)
    for step in range(12):                                  # decode: graph replay vs eager, and against the restatement
        lens = [l + 1 for l in lens]
        sp = _sp(3, step)
        a = eager.forward([[t] for t in a], sids, lens, sampling_params_list=sp)
        b = graph.forward([[t] for t in b], sids, lens, sampling_params_list=sp)
        assert a == b
        assert torch.equal(eager.post_layer.last_logits, graph.post_layer.last_logits)
        _check(eager, a, sp, lens)
    assert {k[2:] for k in graph._graphs} == {(True, False)}
    # greedy steps still replay the greedy graph
    lens = [l + 1 for l in lens]
    g_greedy = graph.forward([[t] for t in b], sids, lens)
    assert g_greedy == eager.forward([[t] for t in a], sids, lens)
    # mixed batch: chunked prefill of a new prompt + the three decodes
    p4 = rng.integers(0, 512, size=50).tolist()
    eager.forward([p4[:20]], [5], [], prefill_prefix_lens_list=[0])
    lens = [l + 1 for l in lens]
    sp = _sp(4, 1)
    t = eager.forward([p4[20:50]] + [[x] for x in g_greedy], [5] + sids, lens, prefill_prefix_lens_list=[20], sampling_params_list=sp)
    _check(eager, t, sp, [50] + lens)
    # prefill only
    sp = _sp(2, 3)
    t = eager.forward([p4[:7], p4[:30]], [1, 2], [], sampling_params_list=sp)
    _check(eager, t, sp, [7, 30])


def test_unseeded_rows_are_reproducible_from_sampling_seed():
    from swiftllm_b200 import SamplingParams
    w = _weights()
    runs = []
    for _ in range(2):
        m = _model(False, sampling_seed=1234, w=w)
        toks = m.forward([[1, 2, 3, 4]] * 4, [0, 1, 2, 3], [], sampling_params_list=[SamplingParams(1.0)] * 4)
        toks2 = m.forward([[t] for t in toks], [0, 1, 2, 3], [5] * 4, sampling_params_list=[SamplingParams(1.0)] * 4)
        runs.append((toks, toks2))
    assert runs[0] == runs[1]


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
        toks = m.forward([[1, 2, 3, 4, 5], [7, 8], [9] * 20], [0, 1, 2], [], sampling_params_list=_sp(3, 1))
        seq = [toks]
        lens = [5, 2, 20]
        for step in range(6):                               # even steps filter (gathered rows), odd ones exchange pairs
            lens = [l + 1 for l in lens]
            from swiftllm_b200 import SamplingParams
            sp = _sp(3, step) if step % 2 == 0 else [SamplingParams(0.9, seed=5 + i) for i in range(3)]
            toks = m.forward([[t] for t in toks], [0, 1, 2], lens, sampling_params_list=sp)
            seq.append(toks)
        out.append(seq)
    got = [None] * world
    dist.all_gather_object(got, out)
    if rank == 0:
        q.put(got)
    dist.destroy_process_group()


def test_tensor_parallel_ranks_return_identical_sampled_tokens():
    """Two GPUs, vocabulary-sharded lm_head: every rank returns the same tokens (both sharded branches, eager and graph)."""
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_tp_worker, args=(r, 2, 29931, q)) for r in range(2)]
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
