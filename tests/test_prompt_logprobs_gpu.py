"""GPU: the prompt log-probability kernel (csrc/prompt_logprobs.cu) bit for bit against sllm_token_logprobs on the same rows, its
ids and ranks against the numpy restatement (tests/prompt_logprobs_oracle.py) and its values against fp64; and
LlamaModel.forward_with_logprobs with SamplingParams.prompt_logprobs against the kernel on the model's own prompt-row logits,
those logits against the exact-arithmetic oracle, chunked against whole prompts, and its memory against profile_num_blocks."""
import numpy as np
import pytest
import torch

import logprobs_oracle as LO
import prompt_logprobs_oracle as PO

pytestmark = pytest.mark.gpu


def _prompt(logits, targets, n):
    from swiftllm_b200.worker.kernels.logprobs import prompt_logprobs
    out = prompt_logprobs(logits, torch.as_tensor(np.asarray(targets), dtype=torch.int32, device=logits.device), n)
    return tuple(t.cpu().numpy() for t in out)


def _token(logits, targets, n):
    from swiftllm_b200.worker.kernels.logprobs import token_logprobs
    out = token_logprobs(logits, torch.as_tensor(np.asarray(targets), dtype=torch.int64, device=logits.device), n)
    return tuple(t.cpu().numpy() for t in out)


def _bits(x):
    return x.view(np.uint32) if x.dtype == np.float32 else x


def _same(a, b):
    """Bit-identical (NaN == NaN)."""
    return all(np.array_equal(_bits(x), _bits(y)) for x, y in zip(a, b))


def _close_to_fp64(got, ref64, what):
    nan, fin = np.isnan(ref64), np.isfinite(ref64)
    assert np.isnan(got[nan]).all(), what
    assert (got[~fin & ~nan] == ref64[~fin & ~nan]).all(), what
    err = np.abs(got[fin].astype(np.float64) - ref64[fin]).max(initial=0)
    assert err <= LO.TOL, (what, err)


def _check_against_token_kernel_and_restatement(logits, targets, n, sample_rows):
    got = _prompt(logits, targets, n)
    lp, rank, ids, tlp = got
    assert _same(got, _prompt(logits, targets, n)), "not deterministic run to run"
    t_lp, t_ids, t_tlp = _token(logits, np.asarray(targets) % logits.shape[1], n)
    ok = (np.asarray(targets) >= 0) & (np.asarray(targets) < logits.shape[1])
    assert np.array_equal(_bits(lp[ok]), _bits(t_lp[ok])), n
    assert np.isnan(lp[~ok]).all() and (rank[~ok] == -1).all()
    assert np.array_equal(ids, t_ids) and np.array_equal(_bits(tlp), _bits(t_tlp)), n
    sub = logits[sample_rows]
    tg = np.asarray(targets)[sample_rows]
    w_lp, w_rank, w_ids, _ = PO.prompt_logprobs(sub, tg, n)
    assert np.array_equal(ids[sample_rows], w_ids) and np.array_equal(rank[sample_rows], w_rank), n
    ref64 = LO.log_softmax64(sub)
    okr = ok[sample_rows]
    _close_to_fp64(lp[sample_rows][okr], ref64[np.arange(len(tg))[okr], tg[okr]], ("target", n))
    _close_to_fp64(tlp[sample_rows], np.take_along_axis(ref64, ids[sample_rows].astype(np.int64).clip(0), axis=1), ("top", n))
    return got


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V", [1000, 32001, 128256])
@pytest.mark.parametrize("R", [1, 3, 257, 4097])
def test_kernel_matches_token_logprobs_and_the_restatement(R, V, dtype):
    g = torch.Generator(device="cuda").manual_seed(R * 5 + V)
    logits = (torch.randn((R, V), generator=g, device="cuda") * 2.5).to(dtype)
    logits[:, ::97] = logits[:, 5:6]                        # repeated values
    if R > 1:
        logits[1, ::40] = logits[1].max()                   # the maximum repeated: more candidates than the select buffer holds
        logits[1, 3] = -0.0
    if R > 2:
        logits[2, :] = 0.0; logits[2, 7] = -0.0             # every logit tied: rank 1 for all, ids 0 .. N-1
    rng = np.random.default_rng(R + V)
    targets = rng.integers(0, V, size=R)
    targets[0] = int(torch.argmax(logits[0]))
    if R > 2:
        targets[2] = 7
    sample = sorted(set([0, 1, 2, R // 2, R - 1]) & set(range(R)))
    for n in (0, 1, 5, 20):
        lp, rank, ids, tlp = _check_against_token_kernel_and_restatement(logits, targets, n, sample)
        assert rank[0] == 1                                 # the greedy token
        if n:
            assert ids[0, 0] == targets[0] and tlp[0, 0] == lp[0]
        if R > 2:
            assert rank[2] == 1 and (n == 0 or ids[2].tolist() == list(range(min(n, V))))
    for r in range(min(R, 3)):                              # a row alone == the same row in the batch
        alone = _prompt(logits[r:r + 1], targets[r:r + 1], 5)
        assert _same(alone, tuple(x[r:r + 1] for x in _prompt(logits, targets, 5)))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_edge_rows(dtype):
    V = 32001
    logits = (torch.randn((9, V), device="cuda") * 3).to(dtype)
    logits[0, 100] = float("nan")
    logits[1, 31999] = float("inf")
    logits[2, :] = -float("inf")
    logits[3, ::2] = -float("inf")
    logits[4, 7] = -float("nan")
    logits[6, 11] = -0.0; logits[6, 12] = 0.0; logits[6] = logits[6].clamp(max=0)
    targets = [100, 5, 0, 0, 3, -1, 12, V, 31999]
    got = _check_against_token_kernel_and_restatement(logits, targets, 20, list(range(9)))
    lp, rank, ids, tlp = got
    assert np.isnan(lp[[0, 1, 2, 4]]).all() and np.isnan(tlp[[0, 1, 2, 4]]).all()
    assert rank[0] == 1 and ids[0, 0] == 100                # a NaN key sorts first, its rank follows the key
    assert lp[3] == -np.inf and np.isfinite(tlp[3]).all()
    assert rank[5] == -1 and rank[7] == -1 and np.isnan(lp[[5, 7]]).all()
    assert rank[6] == 1 + int((logits[6].float() > 0).sum())
    small = logits[5:8, :7].contiguous()                    # fewer entries than top_n
    lp, rank, ids, tlp = _prompt(small, [1, 2, 6], 20)
    assert (ids[:, 7:] == -1).all() and np.isnan(tlp[:, 7:]).all()
    assert np.array_equal(rank, PO.ranks(small, [1, 2, 6]))


@pytest.mark.parametrize("V", [32001, 1001, 128256])
def test_row_strided_and_unaligned_rows(V):
    """Row starts at every alignment: a column slice of wider rows, and odd V (every other row starts off a 16-byte boundary)."""
    big = (torch.randn((6, V + 64), device="cuda") * 2).to(torch.bfloat16)
    targets = [1, 2, 3, 4, 5, V - 1]
    for off in (0, 1, 3, 8):
        view = big[:, off:V + off]
        got = _check_against_token_kernel_and_restatement(view, targets, 5, [0, 5])
        assert _same(got, _prompt(view.contiguous(), targets, 5))
    flat = big.reshape(-1)[: 6 * V].view(6, V)              # odd V: packed rows of alternating alignment
    _check_against_token_kernel_and_restatement(flat, targets, 20, list(range(6)))


# ---------------------------------------------------------------- through LlamaModel
def _models(n=2, **kw):
    from test_sampling_gpu import _model, _weights
    w = _weights()
    return [_model(False, w=w) for _ in range(n)], w


def _pp(n, shift=0):
    from swiftllm_b200 import SamplingParams
    c = [SamplingParams(0.0, prompt_logprobs=5), SamplingParams(0.8, seed=21, prompt_logprobs=0, logprobs=2),
         SamplingParams(0.0, prompt_logprobs=20), SamplingParams(0.7, top_p=0.85, seed=23), SamplingParams(0.0, prompt_logprobs=1)]
    return [c[(i + shift) % len(c)] for i in range(n)]


def _check_prompt_values(m, res, sp, n_prefill):
    """Every scored row's values: the token kernel's on the product's own prompt-row logits, bit for bit; ranks and ids: the
    restatement's."""
    logits = m.post_layer.last_prompt_logits
    off = 0
    for i, (r, p) in enumerate(zip(res, sp)):
        if i >= n_prefill or p.prompt_logprobs is None:
            assert r.prompt is None
            continue
        pl = r.prompt
        k = len(pl.token_ids)
        if k == 0:
            continue
        rows = logits[off:off + k]
        off += k
        n = p.prompt_logprobs
        t_lp, t_ids, t_tlp = _token(rows, pl.token_ids, n)
        assert np.array_equal(_bits(pl.logprobs), _bits(t_lp))
        assert np.array_equal(pl.top_ids, t_ids) and np.array_equal(_bits(pl.top_logprobs), _bits(t_tlp))
        assert np.array_equal(pl.ranks, PO.ranks(rows, pl.token_ids))
        assert pl.top_ids.shape == (k, n) and pl.token_ids.dtype == np.int64
    assert off == logits.shape[0]


def test_model_prompt_logprobs_whole_chunked_and_mixed():
    (a, b, c), w = _models(3)
    rng = np.random.default_rng(8)
    prompts = [rng.integers(0, 1000, size=n).tolist() for n in (70, 9, 1, 33)]
    sids = [3, 9, 0, 5]
    sp = _pp(4)
    nxt = [11, None, 7, None]
    res = a.forward_with_logprobs(prompts, sids, [], sampling_params_list=sp, prompt_next_ids_list=nxt)
    toks = b.forward(prompts, sids, [], sampling_params_list=sp)
    assert [r.token for r in res] == toks
    assert torch.equal(a.k_cache, b.k_cache) and torch.equal(a.v_cache, b.v_cache)
    _check_prompt_values(a, res, sp, 4)
    for r, p, x, q in zip(res, sp, prompts, nxt):
        if p.prompt_logprobs is not None:
            first, rows, tgt = PO.entry_targets(x, 0, q)
            assert r.prompt.first_position == first == 1 and r.prompt.token_ids.tolist() == tgt
    assert res[2].prompt.token_ids.tolist() == [7]          # a 1-token prompt scores its next id only
    whole = res[0].prompt
    whole_logits = a.post_layer.last_prompt_logits[:whole.token_ids.shape[0]].float().cpu()

    # chunks of prompt 0 with the next chunk's first token: the concatenation is the whole prompt's result
    P0 = prompts[0]
    cuts = [0, 20, 45, 70]
    parts, chunk_logits = [], []
    for j in range(3):
        s, e = cuts[j], cuts[j + 1]
        nx = P0[e] if e < 70 else 11
        r = c.forward_with_logprobs([P0[s:e]], [3], [], prefill_prefix_lens_list=[s], sampling_params_list=[sp[0]],
                                    prompt_next_ids_list=[nx])[0]
        assert r.prompt.first_position == s + 1
        parts.append(r.prompt)
        chunk_logits.append(c.post_layer.last_prompt_logits.float().cpu())
    assert np.concatenate([p.token_ids for p in parts]).tolist() == whole.token_ids.tolist()
    tol = 2 ** -5 * float(whole_logits.abs().max())
    assert float((torch.cat(chunk_logits) - whole_logits).abs().max()) <= tol
    lp = np.concatenate([p.logprobs for p in parts])
    assert np.abs(lp - whole.logprobs).max() <= 2 * tol

    # mixed: a new prompt's chunk + decodes; entries without prompt_logprobs and decode entries get None
    lens = [len(x) + 1 for x in prompts[1:]]
    sp2 = _pp(4, 2)
    p5 = rng.integers(0, 1000, size=30).tolist()
    dec = [[t] for t in toks[1:]]
    r1 = a.forward_with_logprobs([p5] + dec, [6] + sids[1:], lens, sampling_params_list=sp2, prompt_next_ids_list=[None])
    r2 = b.forward([p5] + dec, [6] + sids[1:], lens, sampling_params_list=sp2)
    assert [r.token for r in r1] == r2
    assert torch.equal(a.k_cache, b.k_cache) and torch.equal(a.v_cache, b.v_cache)
    _check_prompt_values(a, r1, sp2, 1)
    assert all(r.prompt is None for r in r1[1:])

    # scoring without caching
    r3 = a.forward_with_logprobs([P0], [1], [], ignore_kvcache=True, sampling_params_list=[sp[0]], prompt_next_ids_list=[11])
    assert _same((r3[0].prompt.logprobs, r3[0].prompt.top_ids), (whole.logprobs, whole.top_ids))


def test_prompt_logits_match_the_exact_arithmetic_oracle():
    """Every prompt row's logits against the oracle, which returns the last row's: row j is the last row of the prefix x[:j+1]."""
    from oracle.model import OracleLlama
    from test_model_gpu import TINY2
    (m,), w = _models(1)
    oracle = OracleLlama(TINY2, w, block_size=16, num_blocks=40, num_cpu_blocks=4, max_seqs_in_block_table=16,
                         max_blocks_per_seq=16, attn="exact", dtype=torch.bfloat16)
    x = np.random.default_rng(3).integers(0, 1000, size=24).tolist()
    from swiftllm_b200 import SamplingParams
    res = m.forward_with_logprobs([x], [2], [], sampling_params_list=[SamplingParams(prompt_logprobs=3)])
    got = m.post_layer.last_prompt_logits.float().cpu()
    ref = []
    for j in range(len(x) - 1):
        oracle.forward([x[:j + 1]], [0], [], ignore_kvcache=True)
        ref.append(oracle.last_logits.float()[0])
    ref = torch.stack(ref)
    assert float((got - ref).abs().max() / ref.abs().max()) <= 2 ** -5
    assert res[0].prompt.token_ids.tolist() == x[1:]


def test_prompt_logprobs_stay_within_the_profiled_peak_memory():
    """A max_tokens_in_batch prompt with prompt_logprobs=20 allocates no more above the step's starting point than the profiling
    forward did above the weights, nor than the same step through forward(): the logits are computed in blocks after the layers,
    and no prompt metadata is allocated before them."""
    import swiftllm_b200
    from swiftllm_b200.worker.weight import synthetic_getter
    cfg = dict(model_type="llama", num_hidden_layers=2, num_attention_heads=8, num_key_value_heads=2, hidden_size=1024,
               vocab_size=32000, max_position_embeddings=4096, intermediate_size=1536, rope_theta=500000.0, rms_norm_eps=1e-5,
               hidden_act="silu")
    T = 2048
    ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=2,
                                    max_seqs_in_block_table=4, max_blocks_per_seq=T // 16, max_batch_size=4, max_tokens_in_batch=T,
                                    dtype="bfloat16")
    m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(cfg))
    m.load_weights(synthetic_getter(seed=2, std=0.05))
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    m.profile_num_blocks()
    profiled = torch.cuda.max_memory_allocated() - base
    m.init_kvcache_and_swap(2 * (T // 16) + 4)
    assert m._prompt_block_rows() < T                       # several blocks
    x = np.random.default_rng(0).integers(0, 32000, size=T).tolist()

    def peak(fn):
        # from an empty allocator cache, as profile_num_blocks measures: a cached block is handed out unsplit when less than
        # 1 MB of it would remain, and counts in full, so a warm cache can inflate the peak by up to that much per allocation
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = fn()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base, out

    plain, _ = peak(lambda: m.forward([x], [1], []))
    used, res = peak(lambda: m.forward_with_logprobs([x], [0], [], prompt_next_ids_list=[5],
                                                     sampling_params_list=[swiftllm_b200.SamplingParams(prompt_logprobs=20)]))
    assert res[0].prompt.token_ids.shape == (T,)
    assert used <= profiled, (used, profiled)
    # nothing of the prompt part is live during the layers: the step's peak is forward()'s own
    assert used <= plain, (used, plain)


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
    for shard in (True, False):
        ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=2,
                                        max_seqs_in_block_table=8, max_blocks_per_seq=16, max_batch_size=4, max_tokens_in_batch=256,
                                        dtype="bfloat16", tp_size=world, tp_rank=rank, shard_lm_head=shard)
        m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(CFG))
        m.load_weights(synthetic_getter(seed=11, std=0.05, device=f"cuda:{rank}"))
        m.init_kvcache_and_swap(40)
        res = m.forward_with_logprobs([[1, 2, 3, 4, 5], [7, 8], [9] * 20], [0, 1, 2], [], sampling_params_list=_pp(3, 1),
                                      prompt_next_ids_list=[3, None, 4])
        out.append([(r.token, None if r.prompt is None else tuple(x.tolist() for x in r.prompt[1:])) for r in res])
    got = [None] * world
    dist.all_gather_object(got, out)
    if rank == 0:
        q.put(got)
    dist.destroy_process_group()


def test_tensor_parallel_ranks_return_identical_prompt_logprobs():
    """Two GPUs: sharded lm_head (rows gathered per block) and replicated lm_head give identical results on every rank."""
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_tp_worker, args=(r, 2, 29957, q)) for r in range(2)]
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
    assert got[0] == got[1] and got[0][0] == got[0][1]
