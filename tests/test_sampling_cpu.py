"""CPU: the sampling semantics (tests/sampling_oracle.py, restated from csrc/sampling.cu), the C ABI's argument checks, the host
validation of SamplingParams, the staging of the per-row parameters, and the sampled host path of LlamaModel (single GPU and
tensor parallel over gloo) with the restatement standing in for the kernel."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import sampling_oracle as SO


def test_philox_known_answer_vectors():
    """Random123's kat_vectors for philox4x32_10."""
    cases = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
             ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
             ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
              (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in cases:
        assert tuple(int(x) for x in SO.philox4x32_10(*ctr, *key)) == want


def test_uniforms_stay_inside_the_open_interval():
    x = np.array([0, 1, 511, 512, 2 ** 32 - 1], dtype=np.uint32)
    u = ((x >> 9).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)
    assert (u > 0).all() and (u < 1).all() and np.isfinite(-np.log(-np.log(u))).all()


def _row(vals, dtype=torch.float16):
    return torch.tensor([vals], dtype=dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_greedy_is_torch_argmax_including_ties_and_signed_zeros(dtype):
    g = torch.Generator().manual_seed(0)
    for _ in range(30):
        lg = torch.randint(-3, 3, (4, 50), generator=g).to(dtype)
        lg[0, 7] = -0.0
        res = SO.sample_tokens(lg, [0.0] * 4, [5] * 4, [0.5] * 4, [1] * 4, [1] * 4)
        assert [r.token for r in res] == torch.argmax(lg, dim=1).tolist()
    lg = _row([-0.0, 0.0, -1.0])
    assert SO.sample_tokens(lg, [0.0], [0], [1.0], [0], [0])[0].token == 0 == int(torch.argmax(lg))


def _brute_topk(vals, k):
    order = sorted(vals, reverse=True)
    return np.array([v >= order[k - 1] for v in vals]) if 0 < k < len(vals) else np.ones(len(vals), bool)


def _brute_topp(vals, kept, T, p):
    """Sort the survivors, add fp64 masses from the top one distinct value at a time, stop at p * Z."""
    vals = np.asarray(vals, dtype=np.float64)
    m = vals[kept].max()
    q = np.where(kept, np.exp((vals - m) / T), 0)
    Z, acc = q.sum(), 0.0
    for v in sorted(set(vals[kept].tolist()), reverse=True):
        acc += q[vals == v].sum()
        if acc >= np.float32(p) * Z:
            return kept & (vals >= v)
    return kept


@pytest.mark.parametrize("case", ["ties_at_k", "k_ge_V", "k_one", "tiny_p", "p_tie_boundary", "k_and_p", "negative"])
def test_kept_sets_equal_brute_force_sorts(case):
    vals, k, p, T = {
        "ties_at_k": ([1, 3, 3, 3, 2, 0, 3, -1], 2, 1.0, 1.0),        # the 2nd largest is tied with three more: all kept
        "k_ge_V": ([1, 2, 3, 4], 9, 1.0, 0.7),
        "k_one": ([1, 5, 5, 2], 1, 1.0, 0.7),                          # k = 1 with a tie at the top keeps both
        "tiny_p": ([0.5, 4, 1, 3.5], 0, 1e-6, 1.0),                    # only the max survives
        "p_tie_boundary": ([2, 2, 1, 1, 1, 0], 0, 0.5, 1.0),           # the boundary value's ties are all kept
        "k_and_p": ([4, 3, 3, 2, 2, 2, 1, 0], 5, 0.8, 2.0),
        "negative": ([-8, -7.5, -0.0, 0.0, -3, -2], 3, 0.9, 0.5),
    }[case]
    lg = _row([float(v) for v in vals])
    res = SO.sample_tokens(lg, [T], [k], [p], [123], [4])[0]
    fv = lg[0].float().tolist()
    want = _brute_topk(fv, k)
    if p < 1:
        want = _brute_topp(fv, want, T, p)
    assert res.kept.tolist() == want.tolist()
    assert res.kept[res.token]


def test_empirical_frequencies_match_the_filtered_softmax():
    from scipy.stats import chisquare
    V, S, T, k, p = 40, 20000, 0.8, 25, 0.9
    lg = torch.linspace(-3, 2, V).to(torch.bfloat16)[None]
    vals = lg[0].float().numpy()
    res = SO.sample_tokens(lg, [T], [k], [p], [0], [9])[0]
    kept = res.kept
    prob = np.where(kept, np.exp((vals - vals.max()) / T), 0)
    prob /= prob.sum()
    # 20 000 seeds at once: the restatement's draw, vectorised over seeds
    seeds = np.arange(S, dtype=np.uint64)
    gidx = np.arange(V, dtype=np.int64)
    w = SO.philox4x32_10((gidx >> 2)[None], np.uint32(9), 0, 0, (seeds & np.uint64(0xFFFFFFFF))[:, None], (seeds >> np.uint64(32))[:, None])
    x = np.choose(np.broadcast_to(gidx & 3, (S, V)), w)
    u = ((x >> 9).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)
    score = np.where(kept, vals.astype(np.float32) / np.float32(T) - np.log(-np.log(u)), -np.inf)
    tok = score.argmax(axis=1)
    for s in (0, 1, 777):                                   # the vectorised draw is the restatement's
        assert tok[s] == SO.sample_tokens(lg, [T], [k], [p], [s], [9])[0].token
    assert kept[tok].all()
    cnt = np.bincount(tok, minlength=V)[kept]
    assert chisquare(cnt, prob[kept] * S).pvalue > 1e-3


@pytest.mark.parametrize("shards", [2, 3, 8])
def test_sharded_pairs_merge_to_the_unsharded_token(shards):
    g = torch.Generator().manual_seed(shards)
    B, V = 6, 24 * 5
    lg = (torch.randn((B, V), generator=g) * 2).to(torch.bfloat16)
    temp, seed, pos = [0.0, 0.7, 1.0, 1.3, 0.0, 2.0], [1, 2, 3, 4, 5, 2 ** 63 + 7], [3, 3, 9, 100, 1, 2]
    full = [r.token for r in SO.sample_tokens(lg, temp, [0] * B, [1.0] * B, seed, pos)]
    Vs = V // shards
    per = [SO.sample_tokens(lg[:, n * Vs:(n + 1) * Vs], temp, [0] * B, [1.0] * B, seed, pos, vocab_offset=n * Vs)
           for n in range(shards)]
    assert SO.merge_pairs(per) == full


# ---------------------------------------------------------------- C ABI and host validation
def test_sample_tokens_rejects_invalid_arguments_before_launch():
    from swiftllm_b200 import _lib
    l = _lib.lib()
    args = lambda **kw: [kw.get(n, d) for n, d in (("logits", 1), ("rows", 2), ("V", 1000), ("stride", 1000), ("off", 0),
                                                      ("t", 1), ("k", 1), ("p", 1), ("s", 1), ("pos", 1), ("out", 1),
                                                      ("pairs", None), ("dtype", 1), ("stream", None))]
    for kw, msg in (({"dtype": 7}, b"dtype"), ({"V": 0}, b"vocab_size"), ({"V": 1 << 21, "stride": 1 << 21}, b"shared memory"),
                    ({"stride": 999}, b"row_stride"), ({"off": (1 << 24) - 10}, b"2^24"), ({"rows": -1}, b"num_rows"),
                    ({"t": None}, b"null pointer")):
        assert l.sllm_sample_tokens(*args(**kw)) != 0, kw
        assert msg in l.sllm_last_error(), (kw, l.sllm_last_error())
    assert l.sllm_sample_tokens(*args(rows=0, logits=None)) == 0          # empty batch: nothing to launch


@pytest.mark.parametrize("bad", [dict(temperature=-0.1), dict(temperature=float("nan")), dict(temperature=float("inf")),
                                 dict(top_k=-1), dict(top_k=2.5), dict(top_k=True), dict(top_p=0.0), dict(top_p=1.5),
                                 dict(top_p=float("nan")), dict(seed=-1), dict(seed=2 ** 64), dict(seed=1.0)])
def test_bad_sampling_params_raise_value_error(bad):
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import sampling_words
    with pytest.raises(ValueError):
        sampling_words([SamplingParams(**bad)], 1, np.random.default_rng(0))


def test_sampling_list_must_match_the_batch():
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import sampling_words
    rng = np.random.default_rng(0)
    with pytest.raises(ValueError):
        sampling_words([SamplingParams()], 2, rng)
    with pytest.raises(ValueError):
        sampling_words([SamplingParams(), dict(temperature=1.0)], 2, rng)
    assert sampling_words([SamplingParams(), SamplingParams(top_k=3)], 2, rng) is None       # all greedy: the argmax path


def test_sampling_words_layout():
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import sampling_words
    from swiftllm_b200.worker.infer_state import SamplingState
    sp = [SamplingParams(0.7, 5, 0.9, seed=2 ** 64 - 3), SamplingParams(0.0), SamplingParams(1.0, top_p=1.0, seed=None)]
    words, filtered = sampling_words(sp, 3, np.random.default_rng(5))
    assert filtered and len(words) == 15
    st = SamplingState.from_staged(torch.tensor(words, dtype=torch.int32), torch.tensor([4, 5, 6], dtype=torch.int32), filtered)
    assert st.seed[0].item() == -3 and 0 <= st.seed[2].item() < 2 ** 63
    assert st.temperature.tolist() == [np.float32(0.7), 0.0, 1.0] and st.top_k.tolist() == [5, 0, 0]
    assert st.top_p.tolist() == [np.float32(0.9), 1.0, 1.0]
    again, _ = sampling_words(sp, 3, np.random.default_rng(5))
    assert again == words                                   # unseeded rows: reproducible from the generator's seed
    assert sampling_words([SamplingParams(0.5)], 1, np.random.default_rng(0))[1] is False


# ---------------------------------------------------------------- host path with the restatement standing in for the kernel
def _stand_in(logits, temperature, top_k, top_p, seed, pos, vocab_offset=0, out_pairs=None):
    res = SO.sample_tokens(logits, temperature.tolist(), top_k.tolist(), top_p.tolist(), seed.tolist(), pos.tolist(), vocab_offset)
    if out_pairs is not None:
        out_pairs.copy_(torch.tensor([[r.score, float(r.token)] for r in res], dtype=torch.float32))
    return torch.tensor([r.token for r in res], dtype=torch.int64)


PATCH = [("swiftllm_b200.worker.layers.post_layer", "sample_tokens", _stand_in)]


def _params(n, seed0=0):
    from swiftllm_b200 import SamplingParams
    choices = [SamplingParams(0.0), SamplingParams(0.8, seed=11), SamplingParams(1.2, top_k=7, seed=12),
               SamplingParams(0.6, top_p=0.9, seed=13), SamplingParams(1.0, top_k=20, top_p=0.8), SamplingParams(0.9)]
    return [choices[(i + seed0) % len(choices)] for i in range(n)]


def _expect(m, sp_list, seq_lens):
    """The restatement on the model's logits of the step, with the seeds the model staged."""
    st = m._last_sampling
    return [r.token for r in SO.sample_tokens(m.post_layer.last_logits, [s.temperature for s in sp_list],
                                              [s.top_k for s in sp_list], [s.top_p for s in sp_list], st.seed.tolist(), seq_lens)]


def _record_sampling(m):
    """Wrap post_layer.forward to keep the step's SamplingState (its seeds, pos) for the checks."""
    fwd = m.post_layer.forward

    def wrapped(x, st, **kw):
        m._last_sampling = st.sampling
        return fwd(x, st, **kw)
    m.post_layer.forward = wrapped


def test_sampled_host_path_on_cpu():
    """Prefill, decode, mixed and chunked-prefill steps: the staged parameters reach the kernel with pos = the sequence length
    after the step; the tokens equal the restatement on the step's logits; sampling_params_list=None and all-greedy lists stage
    exactly what the greedy path stages."""
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG, _product
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=2, std=0.08)
    rng = np.random.default_rng(1)
    with product_on_cpu(PATCH):
        m = _product(w)
        _record_sampling(m)
        staged = []
        orig = m._stage_metadata
        m._stage_metadata = lambda *parts: (staged.append([list(p) for p in parts]), orig(*parts))[1]
        prompts = [rng.integers(0, 300, size=n).tolist() for n in (12, 5, 30)]
        sids = [0, 1, 2]
        sp = _params(3)
        t = m.forward(prompts, sids, [], sampling_params_list=sp)
        assert t == _expect(m, sp, [12, 5, 30])
        assert m._last_sampling.pos.tolist() == [12, 5, 30]
        lens = [13, 6, 31]
        sp = _params(3, 1)
        t = m.forward([[x] for x in t], sids, lens, sampling_params_list=sp)
        assert t == _expect(m, sp, lens)
        # mixed: a chunk of a new prompt (prefix 16) + three decodes
        p4 = rng.integers(0, 300, size=40).tolist()
        m.forward([p4[:16]], [3], [], prefill_prefix_lens_list=[0])
        lens = [14, 7, 32]
        sp = _params(4, 2)
        t = m.forward([p4[16:40]] + [[x] for x in t], [3] + sids, lens, prefill_prefix_lens_list=[16], sampling_params_list=sp)
        assert t == _expect(m, sp, [40] + lens)
        assert m._last_sampling.pos.tolist() == [40] + lens
        # greedy: None and an all-greedy list stage the same words as each other and as before this feature (8 parts)
        staged.clear()
        from swiftllm_b200 import SamplingParams
        lens = [l + 1 for l in lens]
        a = m.forward([[1], [2], [3]], sids, lens)
        m.free_seqs_resources([0, 1, 2])
        b = m.forward([[1, 2], [3], [4, 5, 6]], sids, [])
        c = m.forward([[1, 2], [3], [4, 5, 6]], [4, 5, 6], [], sampling_params_list=[SamplingParams(top_k=3)] * 3)
        assert b == c and len(staged) == 3 and all(len(s) == 8 for s in staged)
        assert staged[1][0] == staged[2][0] and staged[1][2:] == staged[2][2:]
        assert m._last_sampling is None and len(a) == 3
        with pytest.raises(ValueError):
            m.forward([[1]], [7], [], sampling_params_list=[SamplingParams(top_p=0)])
        assert len(staged) == 3                             # rejected before anything was staged


def _tp_worker(rank, world, port, ret, filtered):
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
    ok = True
    toks = []
    with product_on_cpu(PATCH), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=2,
                                        max_seqs_in_block_table=8, max_blocks_per_seq=8, max_batch_size=8, max_tokens_in_batch=128,
                                        dtype="float16", tp_size=world, tp_rank=rank, shard_lm_head=True, fused_allreduce=False,
                                        sampling_seed=5)
        m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(cfg))
        m.load_weights(dict_getter(_hf_tensors(w, cfg["intermediate_size"])))
        assert m.post_layer.sharded
        m.init_kvcache_and_swap(20)
        m.post_layer.keep_logits = True
        _record_sampling(m)
        called = []
        import swiftllm_b200.worker.layers.post_layer as PL
        PL.sample_tokens = lambda lg, *a, **kw: (called.append((lg.shape[1], kw.get("out_pairs") is not None)), _stand_in(lg, *a, **kw))[1]
        rng = np.random.default_rng(2)
        prompts = [rng.integers(0, 96, size=n).tolist() for n in (21, 3, 9)]
        sids, lens = [4, 1, 2], [21, 3, 9]
        sp = [swiftllm_b200.SamplingParams(t, top_k=(5 if filtered and i == 1 else 0), top_p=(0.9 if filtered and i == 2 else 1.0))
              for i, t in enumerate([0.9, 1.1, 0.0])]
        sp[0].seed = 77
        ids, dec, pos = prompts, [], lens
        for _ in range(3):
            t = m.forward(ids, sids, dec, sampling_params_list=sp)
            ok &= t == _expect(m, sp, pos)
            toks.append(t)
            pos = [l + 1 for l in pos]
            ids, dec = [[x] for x in t], pos
        Vs = cfg["vocab_size"] // world
        ok &= all(c == ((cfg["vocab_size"], False) if filtered else (Vs, True)) for c in called) and len(called) == 3
    gathered = [None] * world
    dist.all_gather_object(gathered, (bool(ok), toks))
    if rank == 0:
        ret.put(gathered)
    dist.destroy_process_group()
    # flush the result, then leave without running C++ static destructors: a library thread still alive at interpreter
    # teardown can abort the process after the work has finished
    ret.close()
    ret.join_thread()
    os._exit(0)


@pytest.mark.parametrize("filtered", [False, True], ids=["shard-pairs", "gathered-rows"])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_lm_head_sampling_equals_the_unsharded_tokens(world, filtered):
    """Vocabulary-sharded lm_head over gloo: without top-k / top-p every rank samples its shard and the (score, index) pairs
    merge to the unsharded token; with them, the logits are gathered and every rank samples the full rows.  Both return the
    restatement's token for the full logits, identical on every rank."""
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = 29850 + world * 2 + int(filtered)
    procs = [ctx.Process(target=_tp_worker, args=(r, world, port, ret, filtered)) for r in range(world)]
    for p in procs:
        p.start()
    out = ret.get(timeout=240)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(ok for ok, _ in out), out
    assert all(t == out[0][1] for _, t in out)
