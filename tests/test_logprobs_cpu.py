"""CPU: the log-probability semantics (tests/logprobs_oracle.py) against fp64 log_softmax and brute-force sorts, the C ABI's
argument checks, SamplingParams.logprobs validation, the unchanged staging, and LlamaModel.forward_with_logprobs through the
product's host path (single GPU and a vocabulary-sharded lm_head over gloo) with the restatements standing in for the kernels."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import logprobs_oracle as LO
from test_sampling_cpu import PATCH as SAMPLING_PATCH, _record_sampling


# ---------------------------------------------------------------- the restatement
def _brute_top(row, n):
    vals = [0.0 if v == 0 else float(v) for v in row]           # -0 == +0
    return sorted(range(len(vals)), key=lambda i: (-vals[i], i))[:n]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_restatement_matches_fp64_log_softmax_and_sorts(dtype):
    g = torch.Generator().manual_seed(3)
    B, V = 9, 700
    lg = (torch.randn((B, V), generator=g) * 6).clamp(-64, 64).to(dtype)
    lg[1] = torch.randint(-2, 3, (V,), generator=g).to(dtype)         # heavy ties, also at the top-N boundary
    lg[2, ::3] = -float("inf")                                         # -inf entries of a finite row
    lg[3, :] = 64.0; lg[3, 5] = -64.0                                  # extreme range
    lg[4, 10] = -0.0; lg[4, 11] = 0.0; lg[4] = lg[4].clamp(max=0)      # signed zeros tied at the top
    tok = torch.randint(0, V, (B,), generator=g)
    for n in (0, 1, 5, 20):
        tl, ids, tlp = LO.token_logprobs(lg, tok.tolist(), n)
        ref = LO.log_softmax64(lg)
        for r in range(B):
            assert ids[r].tolist() == _brute_top(lg[r].float().tolist(), n)
            fin = np.isfinite(ref[r, ids[r]])
            assert np.abs(tlp[r][fin] - ref[r, ids[r]][fin]).max(initial=0) <= LO.TOL
            assert (tlp[r][~fin] == -np.inf).all()
            want = ref[r, tok[r]]
            assert (tl[r] == want == -np.inf) or abs(tl[r] - want) <= LO.TOL
            pos = [j for j, i in enumerate(ids[r]) if i == tok[r]]
            if pos:
                assert tlp[r, pos[0]] == tl[r]                        # the same value, bit for bit


def test_restatement_edge_rows():
    V = 40
    lg = torch.linspace(-3, 3, V).to(torch.bfloat16)[None].repeat(5, 1)
    lg[0, 7] = float("nan"); lg[1, 3] = float("inf"); lg[2, :] = -float("inf"); lg[3, 0] = -float("inf")
    tl, ids, tlp = LO.token_logprobs(lg, [7, 3, 0, 0, V + 2], 3)
    assert np.isnan(tl[:3]).all() and np.isnan(tlp[:3]).all()
    assert tl[3] == -np.inf and np.isfinite(tlp[3]).all()
    assert np.isnan(tl[4]) and np.isfinite(tlp[4]).all()              # an id outside [0, V)
    assert ids[1, 0] == 3 and ids[0, 0] == 7                           # +inf and +NaN keys sort first
    tl, ids, tlp = LO.token_logprobs(lg[3:4, :2], [1], 5)             # N clamped to V
    assert ids[0].tolist() == [1, 0, -1, -1, -1] and tlp[0, 1] == -np.inf and np.isnan(tlp[0, 2:]).all()


# ---------------------------------------------------------------- C ABI and host validation
def test_token_logprobs_rejects_invalid_arguments_before_launch():
    from swiftllm_b200 import _lib
    l = _lib.lib()
    args = lambda **kw: [kw.get(n, d) for n, d in (("logits", 1), ("rows", 2), ("V", 1000), ("stride", 1000), ("tok", 1),
                                                      ("n", 5), ("out", 1), ("ids", 1), ("lp", 1), ("dtype", 1), ("stream", None))]
    for kw, msg in (({"dtype": 7}, b"dtype"), ({"V": 0}, b"vocab_size"), ({"V": 1 << 21, "stride": 1 << 21}, b"shared memory"),
                    ({"n": -1}, b"top_n"), ({"n": 21}, b"top_n"), ({"stride": 999}, b"row_stride"), ({"rows": -1}, b"num_rows"),
                    ({"rows": (1 << 20) + 1}, b"num_rows"), ({"tok": None}, b"null pointer"), ({"out": None}, b"null pointer"),
                    ({"ids": None}, b"null pointer"), ({"logits": None}, b"null pointer")):
        assert l.sllm_token_logprobs(*args(**kw)) != 0, kw
        assert msg in l.sllm_last_error(), (kw, l.sllm_last_error())
    assert l.sllm_token_logprobs(*args(rows=0, logits=None, tok=None, out=None)) == 0      # empty batch: nothing to launch


@pytest.mark.parametrize("bad", [-1, 21, 2.0, True, "5"])
def test_bad_logprobs_raise_value_error(bad):
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import sampling_words
    with pytest.raises(ValueError):
        sampling_words([SamplingParams(logprobs=bad)], 1, np.random.default_rng(0))


def test_logprobs_do_not_change_the_staged_words():
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import logprobs_top_n, sampling_words
    plain = [SamplingParams(0.7, 5, 0.9, seed=3), SamplingParams(0.0), SamplingParams(1.0)]
    asked = [SamplingParams(0.7, 5, 0.9, seed=3, logprobs=4), SamplingParams(0.0, logprobs=0), SamplingParams(1.0, logprobs=20)]
    assert sampling_words(plain, 3, np.random.default_rng(1)) == sampling_words(asked, 3, np.random.default_rng(1))
    assert sampling_words([SamplingParams(logprobs=3)], 1, np.random.default_rng(1)) is None      # greedy stays greedy
    assert logprobs_top_n(asked) == 20 and logprobs_top_n(plain) is None and logprobs_top_n(None) is None
    assert logprobs_top_n([SamplingParams(logprobs=0), SamplingParams()]) == 0


# ---------------------------------------------------------------- host path with the restatements standing in for the kernels
def _lp_stand_in(logits, token_ids, top_n):
    tl, ids, tlp = LO.token_logprobs(logits, token_ids.tolist(), top_n)
    return torch.from_numpy(tl), torch.from_numpy(ids), torch.from_numpy(tlp)


PATCH = SAMPLING_PATCH + [("swiftllm_b200.worker.layers.post_layer", "token_logprobs", _lp_stand_in)]


def _lp_params(n, shift=0):
    from swiftllm_b200 import SamplingParams
    c = [SamplingParams(0.0, logprobs=5), SamplingParams(0.8, seed=11, logprobs=0), SamplingParams(1.2, top_k=7, seed=12),
         SamplingParams(0.6, top_p=0.9, seed=13, logprobs=20), SamplingParams(0.0), SamplingParams(0.9, seed=14, logprobs=1)]
    return [c[(i + shift) % len(c)] for i in range(n)]


def _check_logprobs(res, logits, sp_list):
    """forward_with_logprobs' entries against the restatement on the step's logits."""
    tl, ids, tlp = LO.token_logprobs(logits, [r.token for r in res], 20)
    V = logits.shape[1]
    for i, (r, sp) in enumerate(zip(res, sp_list)):
        if sp.logprobs is None:
            assert r.logprob is None and r.top is None
            continue
        assert r.logprob == float(tl[i])
        n = min(sp.logprobs, V)
        assert r.top == [(int(a), float(b)) for a, b in zip(ids[i][:n], tlp[i][:n])]
        if sp.temperature == 0:
            assert r.top == [] or r.top[0] == (r.token, r.logprob)      # a greedy token is top[0], same value


def test_forward_with_logprobs_host_path_on_cpu():
    """Prefill, decode, mixed and chunked steps: forward_with_logprobs returns forward's tokens (two models in lockstep, staging
    identical) and the restatement's log-probabilities of the step's logits; entries without logprobs get None."""
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG, _product
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=2, std=0.08)
    rng = np.random.default_rng(1)
    with product_on_cpu(PATCH):
        a, b = _product(w), _product(w)
        staged = {id(a): [], id(b): []}
        for m in (a, b):
            _record_sampling(m)
            orig = m._stage_metadata
            m._stage_metadata = (lambda o, k: lambda *parts: (staged[k].append([list(p) for p in parts]), o(*parts))[1])(orig, id(m))

        def both(ids, sids, lens, sp, **kw):
            t = a.forward(ids, sids, lens, sampling_params_list=sp, **kw)
            res = b.forward_with_logprobs(ids, sids, lens, sampling_params_list=sp, **kw)
            assert [r.token for r in res] == t
            assert torch.equal(a.post_layer.last_logits, b.post_layer.last_logits)
            _check_logprobs(res, b.post_layer.last_logits, sp)
            return t

        prompts = [rng.integers(0, 300, size=n).tolist() for n in (12, 5, 30)]
        sids = [0, 1, 2]
        t = both(prompts, sids, [], _lp_params(3))
        lens = [13, 6, 31]
        for step in range(3):
            t = both([[x] for x in t], sids, lens, _lp_params(3, step + 1))
            lens = [l + 1 for l in lens]
        p4 = rng.integers(0, 300, size=40).tolist()
        both([p4[:16]], [3], [], _lp_params(1, 2), prefill_prefix_lens_list=[0])
        t = both([p4[16:40]] + [[x] for x in t], [3] + sids, lens, _lp_params(4, 3), prefill_prefix_lens_list=[16])
        assert staged[id(a)] == staged[id(b)]
        # no entry asks: forward()'s step, entries carry None
        res = b.forward_with_logprobs([[x] for x in t[1:]], sids, [l + 1 for l in lens])
        assert all(r.logprob is None and r.top is None for r in res)
        with pytest.raises(ValueError):
            b.forward_with_logprobs([[1]], [7], [], sampling_params_list=[_lp_params(1)[0].__class__(logprobs=21)])


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
                                            max_tokens_in_batch=128, dtype="float16", tp_size=world, tp_rank=rank,
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
        sids, dec = [4, 1, 2], []
        lens = [21, 3, 9]
        for step in range(4):
            # the last step samples without top-k / top-p: forward() merges per-shard pairs there instead of gathering rows
            sp = _lp_params(3, step) if step < 3 else [swiftllm_b200.SamplingParams(0.9, seed=5 + i, logprobs=3) for i in range(3)]
            plain = sharded.forward(ids, sids, dec, sampling_params_list=sp)      # the same step twice: same KV writes
            res = sharded.forward_with_logprobs(ids, sids, dec, sampling_params_list=sp)
            ref = full.forward_with_logprobs(ids, sids, dec, sampling_params_list=sp)
            ok &= [r.token for r in res] == plain
            ok &= res == ref                                  # sharded == unsharded, tokens and log-probabilities
            ok &= torch.equal(sharded.post_layer.last_logits, full.post_layer.last_logits)
            try:
                _check_logprobs(res, sharded.post_layer.last_logits, sp)
            except AssertionError:
                ok = False
            out.append(res)
            lens = [l + 1 for l in lens]
            ids, dec = [[r.token] for r in res], lens
    gathered = [None] * world
    dist.all_gather_object(gathered, (bool(ok), out))
    if rank == 0:
        ret.put(gathered)
    dist.destroy_process_group()
    ret.close()
    ret.join_thread()
    os._exit(0)


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_lm_head_logprobs_equal_the_unsharded_ones_on_every_rank(world):
    """Vocabulary-sharded lm_head over gloo: the full rows are gathered, every rank chooses the token and computes the
    log-probabilities of whole rows; the result equals an unsharded lm_head's and is identical on every rank."""
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_tp_worker, args=(r, world, 29870 + world, ret)) for r in range(world)]
    for p in procs:
        p.start()
    out = ret.get(timeout=240)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(ok for ok, _ in out), out
    assert all(t == out[0][1] for _, t in out)
