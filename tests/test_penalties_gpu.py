"""GPU: the penalty kernel (csrc/penalties.cu) against the numpy restatement (tests/penalties_oracle.py) bit for bit, the token
pages it writes, and the penalties through LlamaModel (eager vs graph replay, chunked prefill, swaps, default parameters)."""
import numpy as np
import pytest
import torch

import penalties_oracle as PO

pytestmark = pytest.mark.gpu

HIST_LENS = [0, 1, 17, 4096, 20000]
BS = 16


def _word(ids, out):
    """Page words id | is_output << 31 as int32."""
    return (np.asarray(ids, dtype=np.int64) | (np.asarray(out, dtype=np.int64) << 31)).astype(np.uint32).view(np.int32)


def _case(B, V, dtype, vocab_offset=0, v_full=None, seed=0, prefill=True):
    """A launch: logits, per-row parameters, token pages with random histories behind a shuffled block table, and the step's
    new tokens (the first B // 3 rows are prefill entries)."""
    v_full = v_full or V
    rng = np.random.default_rng(seed)
    g = torch.Generator(device="cuda").manual_seed(seed)
    logits = (torch.randn((B, V), generator=g, device="cuda") * 3).to(dtype)
    logits[:, 7] = float("nan"); logits[:, 8] = float("inf"); logits[:, 9] = -float("inf"); logits[:, 10] = -0.0
    n_pre = B // 3 if prefill else 0
    hist = [HIST_LENS[i % 5] for i in range(B)]
    heavy = min(2, B - 1)
    hist[heavy] = 70000
    n_new = [int(rng.integers(1, 40)) if i < n_pre else 1 for i in range(B)]
    pos = [h + n for h, n in zip(hist, n_new)]
    nblk = [(p + BS - 1) // BS for p in pos]
    pool = rng.permutation(sum(nblk) + 7)
    max_blocks = max(nblk)
    seq_ids = rng.permutation(B + 3)[:B]
    bt = np.full((B + 3, max_blocks), -1, dtype=np.int32)
    used = 0
    for i in range(B):
        bt[seq_ids[i], :nblk[i]] = pool[used:used + nblk[i]]
        used += nblk[i]
    tc = rng.integers(-2 ** 31, 2 ** 31, size=(len(pool), BS), dtype=np.int64).astype(np.int32)    # unrecorded: anything
    histories, new_ids = [], []
    for i in range(B):
        ids = rng.integers(0, v_full, size=hist[i])
        if hist[i] >= 17:
            ids[:3] = [0, v_full - 1, v_full + 5]                    # both ends of the vocabulary and an id past it
        if i == heavy:
            ids[:] = vocab_offset + V // 2                             # one id 70000 times
        out = rng.random(hist[i]) < 0.6
        q = np.arange(hist[i])
        tc[bt[seq_ids[i], q // BS], q % BS] = _word(ids, out)
        new = rng.integers(0, v_full, size=n_new[i])
        histories.append((np.concatenate([ids, new]), np.concatenate([out, np.full(n_new[i], i >= n_pre)])))
        new_ids.append(new)
    params = []
    for i in range(B):
        if i % 4 == 3:
            params.append((1.0, 0.0, 0.0))
        else:
            params.append((float(rng.uniform(0.5, 2.0)), float(rng.uniform(-2, 2)) * (i % 4 != 1), float(rng.uniform(-2, 2))))
    flat = np.concatenate(new_ids).astype(np.int32)
    last = np.cumsum(n_new) - 1
    dev = lambda a, dt=torch.int32: torch.as_tensor(np.asarray(a), dtype=dt, device="cuda")
    return dict(logits=logits, params=params, histories=histories, tc=tc, bt=bt, seq_ids=seq_ids, pos=pos, n_pre=n_pre,
                n_new=n_new, hist=hist, args=dict(pos=dev(pos), seq_ids=dev(seq_ids), input_ids=dev(flat), last=dev(last),
                                                  p_lens=dev(n_new[:n_pre]), bt=dev(bt), vocab_offset=vocab_offset))


def _run(c, logits=None, tc=None, rows=None):
    from swiftllm_b200.worker.kernels.penalties import apply_penalties
    a = c["args"]
    sel = slice(None) if rows is None else rows
    lg = (c["logits"] if logits is None else logits)[sel].clone()
    r, f, p = (torch.tensor([x[k] for x in c["params"]], dtype=torch.float32, device="cuda")[sel].contiguous() for k in range(3))
    tok = torch.as_tensor(c["tc"] if tc is None else tc, device="cuda").clone()
    n_pre = c["n_pre"] if rows is None else 0
    apply_penalties(lg, r, f, p, a["pos"][sel].contiguous(), a["seq_ids"][sel].contiguous(), a["input_ids"],
                    a["last"][sel].contiguous(), a["p_lens"], n_pre, a["bt"], tok, vocab_offset=a["vocab_offset"])
    return lg, tok


def _same_bits(a, b):
    a, b = a.cpu(), b.cpu()
    both_nan = torch.isnan(a.float()) & torch.isnan(b.float())
    return bool(((a.view(torch.int16) == b.view(torch.int16)) | both_nan).all())


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V,offset,v_full", [(1000, 0, None), (32001, 0, None), (128256, 0, None), (16032, 3 * 16032, 128256)],
                         ids=["1000", "32001", "128256", "shard16032"])
@pytest.mark.parametrize("B", [1, 3, 64, 257])
def test_kernel_matches_the_restatement_bit_for_bit(B, V, offset, v_full, dtype):
    c = _case(B, V, dtype, offset, v_full, seed=B * 7 + V)
    got, tok = _run(c)
    want = PO.penalize(c["logits"], c["params"], c["histories"], vocab_offset=offset)
    for i in range(B):
        assert _same_bits(got[i], want[i]), (i, c["params"][i], c["hist"][i])
        if c["params"][i] == (1.0, 0.0, 0.0):
            assert torch.equal(got[i].view(torch.int16), c["logits"][i].view(torch.int16))
    # the pages: exactly the step's tokens of the penalised rows at [pos - n_new, pos), nothing else changed
    exp = c["tc"].copy()
    for i in range(B):
        if c["params"][i] == (1.0, 0.0, 0.0):
            continue
        ids, out = c["histories"][i]
        q = np.arange(c["hist"][i], c["pos"][i])
        exp[c["bt"][c["seq_ids"][i], q // BS], q % BS] = _word(ids[q], out[q])
    assert np.array_equal(tok.cpu().numpy(), exp)
    again, tok2 = _run(c)
    assert torch.equal(again.view(torch.int16), got.view(torch.int16)) and torch.equal(tok, tok2)


def test_a_row_alone_equals_the_row_in_a_batch_and_samples_the_same_token():
    """Cluster size 8 (one row) against 4 (64 rows): the same penalised logits, and a seeded sampled row draws the same token."""
    from swiftllm_b200.worker.kernels.sampling import sample_tokens
    c = _case(64, 128256, torch.bfloat16, seed=3, prefill=False)
    batch, _ = _run(c)
    for r in (0, 2, 5):
        alone, _ = _run(c, rows=slice(r, r + 1))
        assert torch.equal(alone.view(torch.int16), batch[r:r + 1].view(torch.int16)), r
        args = [torch.tensor([v], device="cuda", dtype=dt) for v, dt in ((0.9, torch.float32), (0, torch.int32), (1.0, torch.float32),
                                                                          (1234, torch.int64), (c["pos"][r], torch.int32))]
        t1 = sample_tokens(alone, *args)
        tb = sample_tokens(batch, *[a.repeat(64) for a in args])
        assert int(t1[0]) == int(tb[r])


# ---------------------------------------------------------------- through LlamaModel
def _params(sids):
    from swiftllm_b200 import SamplingParams
    c = [SamplingParams(0.0, repetition_penalty=1.3, frequency_penalty=0.4), SamplingParams(0.8, seed=31, presence_penalty=1.2),
         SamplingParams(1.1, top_k=20, seed=32, repetition_penalty=1.2, frequency_penalty=0.7, presence_penalty=0.2),
         SamplingParams(0.0, frequency_penalty=1.5)]
    return [c[s % len(c)] for s in sids]


def _pages(m, sid, n):
    bt = m.gpu_block_manager.block_table.cpu()
    tc = m.token_cache.cpu()
    bs = m.engine_config.block_size
    return [int(tc[int(bt[sid, q // bs]), q % bs]) for q in range(n)]


def _decode(models, prompts, sids, steps, swap_at=None):
    """Prefill + decode steps on every model in lockstep; returns the per-step tokens of each."""
    outs = [[m.forward(prompts, sids, [], sampling_params_list=_params(sids))] for m in models]
    lens = [len(p) for p in prompts]
    for s in range(steps):
        lens = [l + 1 for l in lens]
        for k, m in enumerate(models):
            if swap_at is not None and k == 1 and s == swap_at:
                m.swap_out_seqs(sids[1:2]); m.swap_in_seqs(sids[1:2])
            outs[k].append(m.forward([[t] for t in outs[k][-1]], sids, lens, sampling_params_list=_params(sids)))
    return outs, lens


def test_model_eager_equals_graph_replay_and_swaps_change_nothing():
    from test_sampling_gpu import _model, _weights
    from test_model_gpu import _script
    w = _weights()
    eager, graph, swapped = _model(False, w=w), _model(True, w=w), _model(False, w=w)
    rng = np.random.default_rng(5)
    prompts, sids = _script(rng), [3, 9, 0]
    (a, b, c), lens = _decode([eager, graph, swapped], prompts, sids, 8, swap_at=4)
    assert a == b == c
    assert all(k[-2:] == ("penalties", True) for k in graph._graphs)
    for s, n in zip(sids, lens):
        assert _pages(eager, s, n) == _pages(graph, s, n) == _pages(swapped, s, n)


def test_model_chunked_prefill_records_the_whole_prompt_pages():
    """Chunked and whole-prompt prefill record identical pages; every step's token is the restatement applied to the step's raw
    logits with the history of its sequence."""
    from test_sampling_gpu import _model, _weights
    w = _weights()
    whole, chunked = _model(False, w=w), _model(False, w=w)
    rng = np.random.default_rng(6)
    prompt = rng.integers(0, 1000, size=70).tolist()
    sp = _params([0])
    t1 = whole.forward([prompt], [0], [], sampling_params_list=sp)
    chunked.forward([prompt[:30]], [0], [], prefill_prefix_lens_list=[0], sampling_params_list=sp)
    t2 = chunked.forward([prompt[30:]], [0], [], prefill_prefix_lens_list=[30], sampling_params_list=sp)
    assert _pages(whole, 0, 70) == _pages(chunked, 0, 70) == prompt
    hist = [(x, False) for x in prompt]
    for m, t in ((whole, t1), (chunked, t2)):
        want = PO.penalize(m.post_layer.last_logits, [(1.3, 0.4, 0.0)], [hist])
        assert t == torch.argmax(want, dim=1).tolist()
    toks, n = t1, 70
    for _ in range(5):
        hist.append((toks[0], True)); n += 1
        toks = whole.forward([toks], [0], [n], sampling_params_list=sp)
        want = PO.penalize(whole.post_layer.last_logits, [(1.3, 0.4, 0.0)], [hist])
        assert toks == torch.argmax(want, dim=1).tolist()
    assert _pages(whole, 0, n) == _word([x for x, _ in hist], [o for _, o in hist]).tolist()


def test_default_parameters_run_the_plain_step():
    from swiftllm_b200 import SamplingParams, _lib
    from test_sampling_gpu import _model, _weights
    w = _weights()
    a, b = _model(True, w=w), _model(True, w=w)
    prompts, sids = [[1, 2, 3, 4], [5, 6]], [0, 1]
    ta = a.forward(prompts, sids, [])
    tb = b.forward(prompts, sids, [], sampling_params_list=[SamplingParams()] * 2)
    assert ta == tb
    lens = [4, 2]
    for _ in range(3):
        lens = [l + 1 for l in lens]
        n0 = _lib.LAUNCH_CALLS
        ta = a.forward([[t] for t in ta], sids, lens)
        n1 = _lib.LAUNCH_CALLS
        tb = b.forward([[t] for t in tb], sids, lens, sampling_params_list=[SamplingParams()] * 2)
        assert ta == tb and _lib.LAUNCH_CALLS - n1 == n1 - n0
    assert not b._penalties_used and set(a._graphs) == set(b._graphs)
