"""CPU: the prompt log-probability semantics (tests/prompt_logprobs_oracle.py) against brute-force counts and sorts, the C ABI's
argument checks, SamplingParams.prompt_logprobs and prompt_next_ids_list validation, the unchanged staging, and
LlamaModel.forward_with_logprobs' prompt rows through the product's host path (single GPU and a vocabulary-sharded lm_head over
gloo) with the restatements standing in for the kernels."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import prompt_logprobs_oracle as PO
from test_logprobs_cpu import PATCH as LOGPROBS_PATCH


# ---------------------------------------------------------------- the restatement
def _brute_rank(row, t):
    if not 0 <= t < len(row):
        return -1
    key = lambda v: (2 if v != v else 0, 0.0 if v == 0 else v)      # NaN above everything, -0 == +0
    return 1 + sum(key(v) > key(row[t]) for v in row)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_rank_restatement_matches_brute_force_counts(dtype):
    g = torch.Generator().manual_seed(4)
    V = 300
    lg = (torch.randn((8, V), generator=g) * 4).to(dtype)
    lg[1] = torch.randint(-2, 3, (V,), generator=g).to(dtype)         # ties at the target
    lg[2, 10] = -0.0; lg[2, 11] = 0.0; lg[2] = lg[2].clamp(max=0)     # signed zeros
    lg[3, ::3] = -float("inf")
    lg[4, 5] = float("inf")
    lg[5, 6] = float("nan")
    targets = [0, 7, 10, 3, 5, 6, -1, V]
    rank = PO.ranks(lg, targets)
    for r in range(8):
        row = lg[r].float().tolist()
        if r == 5:                                                     # positive NaN: only other NaN keys could be above it
            assert rank[r] == 1
            continue
        assert rank[r] == _brute_rank(row, targets[r]), r
    assert rank[6] == rank[7] == -1 and rank[4] == 1
    lp, rk, ids, tlp = PO.prompt_logprobs(lg, targets, 5)
    assert np.isnan(lp[[4, 5, 6, 7]]).all() and lp[3] <= 0
    for r in (0, 1, 2, 3):                                             # a target's rank is its place among the sorted keys
        if rk[r] <= 5:
            assert ids[r, rk[r] - 1] == targets[r] or lg[r, ids[r, rk[r] - 1]] == lg[r, targets[r]]


def test_entry_targets():
    assert PO.entry_targets([5, 6, 7], 0) == (1, [0, 1], [6, 7])
    assert PO.entry_targets([5, 6, 7], 10, 9) == (11, [0, 1, 2], [6, 7, 9])
    assert PO.entry_targets([5], 0) == (1, [], [])
    assert PO.entry_targets([5], 3, 2) == (4, [0], [2])


# ---------------------------------------------------------------- C ABI and host validation
def test_prompt_logprobs_rejects_invalid_arguments_before_launch():
    from swiftllm_b200 import _lib
    l = _lib.lib()
    names = ("logits", "rows", "V", "stride", "tgt", "n", "lp", "rank", "ids", "tlp", "dtype", "stream")
    dflt = (1, 2, 1000, 1000, 1, 5, 1, 1, 1, 1, 1, None)
    args = lambda **kw: [kw.get(n, d) for n, d in zip(names, dflt)]
    for kw, msg in (({"dtype": 7}, b"dtype"), ({"V": 0}, b"vocab_size"), ({"V": (1 << 24) + 1, "stride": 1 << 25}, b"vocab_size"),
                    ({"n": -1}, b"top_n"), ({"n": 21}, b"top_n"), ({"stride": 999}, b"row_stride"), ({"rows": -1}, b"num_rows"),
                    ({"rows": (1 << 24) + 1}, b"num_rows"), ({"tgt": None}, b"null pointer"), ({"lp": None}, b"null pointer"),
                    ({"rank": None}, b"null pointer"), ({"ids": None}, b"null pointer"), ({"tlp": None}, b"null pointer"),
                    ({"logits": None}, b"null pointer")):
        assert l.sllm_prompt_logprobs(*args(**kw)) != 0, kw
        assert msg in l.sllm_last_error(), (kw, l.sllm_last_error())
    assert l.sllm_prompt_logprobs(*args(rows=0, logits=None, tgt=None, lp=None, rank=None)) == 0     # nothing to launch
    # a max_tokens_in_batch-sized prefill fits the row bound; 128256 fits the vocabulary bound (no shared-memory limit)
    assert l.sllm_prompt_logprobs(*args(rows=1 << 16, V=128256, stride=128256, dtype=7)) != 0
    assert b"dtype" in l.sllm_last_error()


@pytest.mark.parametrize("bad", [-1, 21, 2.0, True, "5"])
def test_bad_prompt_logprobs_raise_value_error(bad):
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import sampling_words
    with pytest.raises(ValueError, match="prompt_logprobs"):
        sampling_words([SamplingParams(prompt_logprobs=bad)], 1, np.random.default_rng(0))


def test_prompt_logprobs_do_not_change_the_staged_words():
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import prompt_logprobs_top_n, sampling_words
    plain = [SamplingParams(0.7, 5, 0.9, seed=3), SamplingParams(0.0), SamplingParams(1.0, repetition_penalty=1.2)]
    asked = [SamplingParams(0.7, 5, 0.9, seed=3, prompt_logprobs=4), SamplingParams(0.0, prompt_logprobs=0),
             SamplingParams(1.0, repetition_penalty=1.2, prompt_logprobs=20)]
    assert sampling_words(plain, 3, np.random.default_rng(1)) == sampling_words(asked, 3, np.random.default_rng(1))
    assert sampling_words([SamplingParams(prompt_logprobs=3)], 1, np.random.default_rng(1)) is None
    assert prompt_logprobs_top_n(asked) == 20 and prompt_logprobs_top_n(plain) is None and prompt_logprobs_top_n(None) is None
    assert prompt_logprobs_top_n([SamplingParams(prompt_logprobs=0), SamplingParams(logprobs=5)]) == 0


def test_token_logprobs_keeps_its_three_field_form():
    from swiftllm_b200 import PromptLogprobs, TokenLogprobs
    t = TokenLogprobs(5, -0.5, [(5, -0.5)])
    assert t == (5, -0.5, [(5, -0.5)], None) and t.prompt is None and t.token == 5
    assert TokenLogprobs(3) == TokenLogprobs(3, None, None) and TokenLogprobs(3).top is None
    assert PromptLogprobs._fields == ("first_position", "token_ids", "logprobs", "ranks", "top_ids", "top_logprobs")


# ---------------------------------------------------------------- host path with the restatements standing in for the kernels
def _prompt_stand_in(logits, targets, top_n, out=None):
    res = tuple(torch.from_numpy(np.ascontiguousarray(x)) for x in PO.prompt_logprobs(logits, targets.tolist(), top_n))
    if out is None:
        return res
    for o, r in zip(out, res):
        o.copy_(r)
    return out


PATCH = LOGPROBS_PATCH + [("swiftllm_b200.worker.layers.post_layer", "prompt_logprobs", _prompt_stand_in)]


def _pp(n, shift=0):
    from swiftllm_b200 import SamplingParams
    c = [SamplingParams(0.0, prompt_logprobs=5), SamplingParams(0.8, seed=11, prompt_logprobs=0, logprobs=3),
         SamplingParams(1.2, top_k=7, seed=12), SamplingParams(0.0, prompt_logprobs=20), SamplingParams(0.9, seed=14, prompt_logprobs=1)]
    return [c[(i + shift) % len(c)] for i in range(n)]


def _check_prompt(m, res, sp, prompts, prefixes, nexts, n_prefill):
    """Each asking prefill entry's PromptLogprobs: positions and targets as the restatement builds them, values the restatement's
    on the product's own prompt-row logits (kept in batch order)."""
    logits = m.post_layer.last_prompt_logits
    off = 0
    for i, (r, p) in enumerate(zip(res, sp)):
        if i >= n_prefill or p.prompt_logprobs is None:
            assert r.prompt is None
            continue
        first, rows, tgt = PO.entry_targets(prompts[i], prefixes[i], nexts[i])
        pl = r.prompt
        assert pl.first_position == first and pl.token_ids.tolist() == tgt and pl.token_ids.dtype == np.int64
        k, n = len(tgt), min(p.prompt_logprobs, logits.shape[1] if logits is not None else 1 << 30)
        assert pl.logprobs.shape == (k,) and pl.ranks.shape == (k,) and pl.top_ids.shape == (k, n)
        if k == 0:
            continue
        lp, rank, ids, tlp = PO.prompt_logprobs(logits[off:off + k], tgt, p.prompt_logprobs)
        assert np.array_equal(pl.logprobs.view(np.uint32), lp.view(np.uint32)) and np.array_equal(pl.ranks, rank)
        assert np.array_equal(pl.top_ids, ids[:, :n]) and np.array_equal(pl.top_logprobs.view(np.uint32), tlp[:, :n].view(np.uint32))
        off += k
    if off:
        assert off == logits.shape[0]


def test_prompt_logprobs_host_path_on_cpu():
    """Whole prompts (with and without next ids, 1-token prompts), chunks whose results concatenate to the whole prompt's, mixed
    prefill + decode batches, ignore_kvcache and several row blocks: forward_with_logprobs returns forward's tokens (two models in
    lockstep) and the restatement's values on the rows it scored; every step stages exactly forward()'s words."""
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200 import SamplingParams
    from test_host_path_cpu import CFG, _product
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=2, std=0.08)
    rng = np.random.default_rng(3)
    with product_on_cpu(PATCH):
        a, b, c = _product(w), _product(w), _product(w)
        c.engine_config.max_tokens_in_batch = 8             # blocks of a few rows
        assert c._prompt_block_rows() < 12
        staged = {id(a): [], id(b): []}
        for m in (a, b):
            orig = m._stage_metadata
            m._stage_metadata = (lambda o, k: lambda *parts: (staged[k].append([list(p) for p in parts]), o(*parts))[1])(orig, id(m))

        prompts = [rng.integers(0, 300, size=n).tolist() for n in (30, 5, 1, 12)]
        sids = [0, 1, 2, 3]
        sp = _pp(4)
        nexts = [17, None, 4, None]
        res = b.forward_with_logprobs(prompts, sids, [], sampling_params_list=sp, prompt_next_ids_list=nexts)
        toks = a.forward(prompts, sids, [], sampling_params_list=sp)
        assert [r.token for r in res] == toks
        assert torch.equal(a.k_cache, b.k_cache) and torch.equal(a.v_cache, b.v_cache)
        _check_prompt(b, res, sp, prompts, [0] * 4, nexts, 4)
        assert res[2].prompt is None                         # SamplingParams without prompt_logprobs
        whole = res[0].prompt
        whole_logits = b.post_layer.last_prompt_logits[:30].clone()

        # several row blocks: the same rows, values of its own logits
        r_c = c.forward_with_logprobs(prompts, sids, [], sampling_params_list=sp, prompt_next_ids_list=nexts)
        assert [r.token for r in r_c] == toks
        _check_prompt(c, r_c, sp, prompts, [0] * 4, nexts, 4)
        assert float((c.post_layer.last_prompt_logits[:30].float() - whole_logits.float()).abs().max()) <= 1e-2

        # a 1-token prompt scores its next id only, and nothing without one
        one = b.forward_with_logprobs([[9], [8]], [4, 5], [], sampling_params_list=[sp[0], sp[0]], prompt_next_ids_list=[None, 3])
        a.forward([[9], [8]], [4, 5], [], sampling_params_list=[sp[0], sp[0]])
        assert one[0].prompt.token_ids.shape == (0,) and one[0].prompt.top_ids.shape == (0, 5) and one[0].prompt.first_position == 1
        assert one[1].prompt.token_ids.tolist() == [3]

        # chunks of prompt 0, each given the next chunk's first token: concatenation == the whole prompt's result
        P0, cuts, parts = prompts[0], [0, 9, 21, 30], []
        for j in range(3):
            s, e = cuts[j], cuts[j + 1]
            nx = P0[e] if e < 30 else 17
            r = b.forward_with_logprobs([P0[s:e]], [6], [], prefill_prefix_lens_list=[s], sampling_params_list=[sp[0]],
                                        prompt_next_ids_list=[nx])
            t = a.forward([P0[s:e]], [6], [], prefill_prefix_lens_list=[s], sampling_params_list=[sp[0]])
            assert [x.token for x in r] == t
            _check_prompt(b, r, [sp[0]], [P0[s:e]], [s], [nx], 1)
            parts.append(r[0].prompt)
        assert [p.first_position for p in parts] == [1, 10, 22]
        assert np.concatenate([p.token_ids for p in parts]).tolist() == whole.token_ids.tolist()
        assert np.abs(np.concatenate([p.logprobs for p in parts]) - whole.logprobs).max() <= 2e-2

        # mixed: one prefill chunk + decodes; decode entries get prompt None even when their parameters ask
        lens = [len(x) + 1 for x in prompts]
        sp2 = _pp(5, 3)
        p7 = rng.integers(0, 300, size=14).tolist()
        r = b.forward_with_logprobs([p7] + [[t] for t in toks], [7] + sids, lens, sampling_params_list=sp2,
                                    prompt_next_ids_list=[1])
        t = a.forward([p7] + [[t] for t in toks], [7] + sids, lens, sampling_params_list=sp2)
        assert [x.token for x in r] == t
        _check_prompt(b, r, sp2, [p7], [0], [1], 1)
        assert all(x.prompt is None for x in r[1:])
        assert torch.equal(a.k_cache, b.k_cache) and torch.equal(a.v_cache, b.v_cache)

        # every step above staged exactly forward()'s words: the prompt rows are built on the device after the layers
        assert len(staged[id(b)]) == 6 and staged[id(a)] == staged[id(b)]
        # no entry asks: forward()'s staged words, prompt None
        del staged[id(a)][:], staged[id(b)][:]
        lens = [l + 1 for l in lens]
        plain = [SamplingParams(0.0), SamplingParams(0.8, seed=3, logprobs=2)]
        r = b.forward_with_logprobs([p7[:6], [t[1]]], [5, 0], [lens[0]], sampling_params_list=plain)
        a.forward([p7[:6], [t[1]]], [5, 0], [lens[0]], sampling_params_list=plain)
        assert staged[id(a)] == staged[id(b)] and all(x.prompt is None for x in r)

        # scoring without caching
        r = b.forward_with_logprobs([P0], [3], [], ignore_kvcache=True, sampling_params_list=[sp[0]], prompt_next_ids_list=[17])
        _check_prompt(b, r, [sp[0]], [P0], [0], [17], 1)
        assert np.abs(r[0].prompt.logprobs - whole.logprobs).max() <= 2e-2


def test_prompt_next_ids_list_is_validated_before_anything_is_enqueued():
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200 import SamplingParams
    from test_host_path_cpu import CFG, _product
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=2, std=0.08)
    with product_on_cpu(PATCH):
        m = _product(w)
        calls = []
        m._stage_metadata = lambda *parts: calls.append(parts)
        sp = [SamplingParams(prompt_logprobs=2), SamplingParams()]
        for nexts, msg in (([1], "entries"), ([1, 2, 3], "entries"), ([300, None], "token id"), ([-1, None], "token id"),
                           ([True, None], "token id"), ([1.0, None], "token id")):
            with pytest.raises(ValueError, match=msg):
                m.forward_with_logprobs([[1, 2], [3]], [0, 1], [], sampling_params_list=sp, prompt_next_ids_list=nexts)
        with pytest.raises(ValueError, match="entries"):                 # one entry per PREFILL entry
            m.forward_with_logprobs([[1, 2], [3]], [0, 1], [5], sampling_params_list=sp, prompt_next_ids_list=[1, 2])
        assert calls == []
        m2 = _product(w)                                                 # an entry that does not ask: its id is not used
        r = m2.forward_with_logprobs([[1, 2], [3]], [0, 1], [], sampling_params_list=sp, prompt_next_ids_list=[None, 999])
        assert r[0].prompt.token_ids.tolist() == [2] and r[1].prompt is None


def _tp_worker(rank, world, port, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import warnings
    import swiftllm_b200
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200.worker.weight import dict_getter
    from test_host_path_cpu import _hf_tensors
    from test_tp_gloo import CFG
    cfg = dict(CFG, num_hidden_layers=2, vocab_size=96)
    if world == 3:
        cfg.update(num_attention_heads=6, num_key_value_heads=3, hidden_size=96, intermediate_size=192)
    w = OracleWeights.random(cfg, dtype=torch.float16, seed=12, std=0.08)
    ok, out = True, []
    with product_on_cpu(PATCH), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        models = []
        for shard in (True, False):
            ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=2,
                                            max_seqs_in_block_table=8, max_blocks_per_seq=8, max_batch_size=8,
                                            max_tokens_in_batch=4, dtype="float16", tp_size=world, tp_rank=rank,
                                            shard_lm_head=shard, fused_allreduce=False, sampling_seed=5)
            m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(cfg))
            m.load_weights(dict_getter(_hf_tensors(w, cfg["intermediate_size"])))
            assert m.post_layer.sharded == shard
            m.init_kvcache_and_swap(20)
            m.post_layer.keep_logits = True
            models.append(m)
        sharded, full = models
        rng = np.random.default_rng(2)
        ids = [rng.integers(0, 96, size=n).tolist() for n in (21, 3, 9)]
        sp = _pp(3)
        res = sharded.forward_with_logprobs(ids, [4, 1, 2], [], sampling_params_list=sp, prompt_next_ids_list=[5, 6, None])
        ref = full.forward_with_logprobs(ids, [4, 1, 2], [], sampling_params_list=sp, prompt_next_ids_list=[5, 6, None])
        flat = lambda rs: [(r.token, r.logprob, r.top, None if r.prompt is None else [x.tolist() if hasattr(x, "tolist") else x
                                                                                     for x in r.prompt]) for r in rs]
        ok &= flat(res) == flat(ref)
        ok &= torch.equal(sharded.post_layer.last_prompt_logits, full.post_layer.last_prompt_logits)
        try:
            _check_prompt(sharded, res, sp, ids, [0] * 3, [5, 6, None], 3)
        except AssertionError:
            ok = False
        out.append(flat(res))
    gathered = [None] * world
    dist.all_gather_object(gathered, (bool(ok), out))
    if rank == 0:
        ret.put(gathered)
    dist.destroy_process_group()
    ret.close()
    ret.join_thread()
    os._exit(0)


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_lm_head_prompt_logprobs_equal_the_unsharded_ones_on_every_rank(world):
    """Vocabulary-sharded lm_head over gloo: each block's rows are gathered and every rank computes the prompt log-probabilities
    of whole rows; the result equals an unsharded lm_head's and is identical on every rank."""
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_tp_worker, args=(r, world, 29880 + world, ret)) for r in range(world)]
    for p in procs:
        p.start()
    out = ret.get(timeout=240)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(ok for ok, _ in out), out
    assert all(t == out[0][1] for _, t in out)
