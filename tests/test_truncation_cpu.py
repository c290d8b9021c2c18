"""CPU: min-p, typical-p and XTC - the restatement (tests/truncation_oracle.py) against literal transcriptions of vLLM's min-p
processor, Hugging Face's TypicalLogitsWarper and llama.cpp's XTC sampler; parameter validation, the staged words and their
views, the host path's graph keys and speculative row words, and the C ABI's checks before launch."""
import dataclasses

import numpy as np
import pytest
import torch

import truncation_oracle as TO


# ---------------------------------------------------------------- the restatement against the libraries' definitions (fp64)
def _softmax(z):
    z = z - z[np.isfinite(z)].max()
    e = np.exp(z)
    return e / e.sum()


def vllm_min_p(logits, T, min_p):
    """vLLM's min-p processor: probs = softmax(logits / T); tokens with p < min_p * max p get -inf."""
    probs = _softmax(logits / T)
    top = probs.max()
    out = logits.copy()
    out[probs < min_p * top] = -np.inf
    return out


def hf_typical(scores, mass):
    """Hugging Face TypicalLogitsWarper.__call__ (min_tokens_to_keep = 1) on one row of temperature-scaled scores."""
    normalized = scores - np.log(np.exp(scores - scores.max()).sum()) - scores.max()            # log_softmax
    p = np.exp(normalized)
    with np.errstate(invalid="ignore"):
        ent = -np.nansum(normalized * p)
    shifted_scores = np.abs(-normalized - ent)
    sorted_indices = np.argsort(shifted_scores, kind="stable")
    sorted_scores = shifted_scores[sorted_indices]
    sorted_logits = scores[sorted_indices]
    cumulative_probs = np.cumsum(_softmax(sorted_logits))
    last_ind = int((cumulative_probs < mass).sum())
    last_ind = min(last_ind, sorted_scores.shape[-1] - 1)
    sorted_indices_to_remove = sorted_scores > sorted_scores[last_ind]
    sorted_indices_to_remove[:1] = False
    indices_to_remove = np.zeros_like(sorted_indices_to_remove)
    indices_to_remove[sorted_indices] = sorted_indices_to_remove
    return np.where(indices_to_remove, -np.inf, scores)


def llama_cpp_xtc(scores, probability, threshold, chance, min_keep=1):
    """llama.cpp's llama_sampler_xtc_apply on one row (the uniform draw passed in as `chance`): the kept ids."""
    ids = np.nonzero(np.isfinite(scores))[0]
    if probability <= 0 or threshold > 0.5 or ids.size < 2:
        return set(ids.tolist())
    if chance > probability:
        return set(ids.tolist())
    p = _softmax(scores[ids])
    order = np.argsort(-p, kind="stable")                                  # llama_sampler_softmax_impl: sorted by p desc
    data = [(int(ids[i]), float(p[i])) for i in order]
    pos_last = 0
    for i in range(len(data)):
        if data[i][1] >= threshold:
            pos_last = i
        else:
            break
    if len(data) - pos_last >= min_keep and pos_last > 0:
        data = data[pos_last:]
    return {i for i, _ in data}


def _row(V, rng, scale):
    vals = (rng.standard_normal(V) * scale).astype(np.float32)
    t = torch.from_numpy(vals).to(torch.bfloat16)
    return t.view(torch.int16).numpy().view(np.uint16), t.float().numpy()


def _distinct(vals):
    return np.unique(vals).size == vals.size


@pytest.mark.parametrize("T", [0.5, 1.0, 1.7])
def test_min_p_is_vllms(T):
    rng = np.random.default_rng(int(T * 10))
    checked = 0
    for _ in range(40):
        bits, vals = _row(int(rng.integers(20, 400)), rng, 2.0)
        mp = float(np.float32(rng.choice([0.01, 0.05, 0.2, 0.6, 1.0])))
        res = TO.sample_row(bits, vals, T, 0, 1.0, 1, 1, min_p=mp)
        if res.boundary_margin <= 1e-6:
            continue
        want = np.isfinite(vllm_min_p(vals.astype(np.float64), np.float32(T), mp))
        assert np.array_equal(res.kept, want)
        checked += 1
    assert checked >= 30


@pytest.mark.parametrize("T", [0.6, 1.0, 1.5])
def test_typical_p_is_hugging_faces(T):
    rng = np.random.default_rng(int(T * 100))
    checked = 0
    for _ in range(40):
        bits, vals = _row(int(rng.integers(20, 400)), rng, 1.5)          # equal logits: equal distances on both sides
        tp = float(np.float32(rng.choice([0.2, 0.5, 0.9, 0.95])))
        res = TO.sample_row(bits, vals, T, 0, 1.0, 1, 1, typical_p=tp)
        if res.boundary_margin <= 1e-5:
            continue
        want = np.isfinite(hf_typical(vals.astype(np.float64) / np.float32(T), tp))
        assert np.array_equal(res.kept, want), (tp, np.nonzero(res.kept != want))
        checked += 1
    assert checked >= 25


def test_typical_p_after_min_p_top_k_and_top_p_is_hugging_faces_chain():
    rng = np.random.default_rng(7)
    for _ in range(30):
        bits, vals = _row(300, rng, 2.0)
        res = TO.sample_row(bits, vals, 1.0, 100, 0.9, 1, 1, min_p=0.01, typical_p=0.8)
        if res.boundary_margin <= 1e-5:
            continue
        s = vllm_min_p(vals.astype(np.float64), 1.0, float(np.float32(0.01)))
        s[vals < np.sort(vals)[::-1][99]] = -np.inf                             # top-k
        p = _softmax(s)                                                          # top-p over the survivors
        order = np.argsort(-p, kind="stable")
        cum = np.cumsum(p[order])
        s[p < p[order[int(np.argmax(cum >= float(np.float32(0.9))))]]] = -np.inf      # ties at the cut kept
        want = np.isfinite(hf_typical(s, float(np.float32(0.8))))
        assert np.array_equal(res.kept, want)


def test_xtc_is_llama_cpps():
    rng = np.random.default_rng(3)
    checked = 0
    for trial in range(200):
        bits, vals = _row(int(rng.integers(5, 60)), rng, 2.0)
        if not _distinct(vals):
            continue
        th = float(np.float32(rng.choice([0.0, 0.02, 0.1, 0.3])))
        xp = float(np.float32(rng.choice([0.3, 0.7, 1.0])))
        seed, pos = int(rng.integers(0, 2 ** 63)), int(rng.integers(1, 9999))
        res = TO.sample_row(bits, vals, 1.0, 0, 1.0, seed, pos, xtc_threshold=th, xtc_probability=xp)
        if res.boundary_margin <= 1e-6:
            continue
        u = float(TO.xtc_draw(seed, pos))
        # the kernel removes when u < probability; llama.cpp when its draw <= probability (equal draws have measure 0)
        want = llama_cpp_xtc(vals.astype(np.float64), xp, th, u)
        assert set(np.nonzero(res.kept)[0].tolist()) == want, (trial, th, xp, u)
        checked += 1
    assert checked >= 100


def test_edges():
    bits, vals = _row(50, np.random.default_rng(0), 2.0)
    top = int(np.argmax(vals))
    assert np.nonzero(TO.sample_row(bits, vals, 1.0, 0, 1.0, 1, 1, min_p=1.0).kept)[0].tolist() == [top]
    # XTC with threshold 0 and probability 1 keeps the least likely survivor (and its ties) only
    kept = TO.sample_row(bits, vals, 1.0, 0, 1.0, 1, 1, xtc_threshold=0.0, xtc_probability=1.0).kept
    assert np.array_equal(kept, vals == vals.min())
    # ties at the XTC boundary are all kept (llama.cpp keeps one)
    t = torch.tensor([3.0, 1.0, 1.0, -2.0], dtype=torch.bfloat16)
    b, v = t.view(torch.int16).numpy().view(np.uint16), t.float().numpy()
    assert TO.sample_row(b, v, 1.0, 0, 1.0, 1, 1, xtc_threshold=0.05, xtc_probability=1.0).kept.tolist() == [False, True, True, True]
    # a tiny typical_p keeps the tokens nearest the entropy
    assert TO.sample_row(bits, vals, 1.0, 0, 1.0, 1, 1, typical_p=1e-4).kept.sum() >= 1
    # greedy and bad rows ignore the filters
    assert TO.sample_row(bits, vals, 0.0, 0, 1.0, 1, 1, min_p=0.5).token == top
    v2 = vals.copy()
    v2[3] = np.nan
    b2 = torch.from_numpy(v2).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    assert TO.sample_row(b2, v2, 1.0, 0, 1.0, 1, 1, typical_p=0.5).kept is None


# ---------------------------------------------------------------- parameters and staging
@pytest.mark.parametrize("field,bad", [("min_p", -0.1), ("min_p", 1.5), ("min_p", float("nan")), ("min_p", True),
                                       ("typical_p", 0.0), ("typical_p", 1.01), ("typical_p", float("inf")),
                                       ("typical_p", False), ("xtc_threshold", -1e-3), ("xtc_threshold", 2.0),
                                       ("xtc_threshold", "0.1"), ("xtc_probability", 1.5), ("xtc_probability", float("nan")),
                                       ("xtc_probability", True)])
def test_bad_truncation_parameters_raise_value_error(field, bad):
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import sampling_words
    with pytest.raises(ValueError, match=field):
        SamplingParams(**{field: bad}).validate()
    with pytest.raises(ValueError, match=field):
        sampling_words([SamplingParams(1.0, **{field: bad})], 1, np.random.default_rng(0))


def test_good_truncation_parameters_and_defaults():
    from swiftllm_b200 import SamplingParams
    d = SamplingParams()
    assert (d.min_p, d.typical_p, d.xtc_threshold, d.xtc_probability) == (0.0, 1.0, 0.1, 0.0) and not d.has_truncation()
    for sp in (SamplingParams(min_p=1.0, typical_p=1e-6, xtc_threshold=0.0, xtc_probability=1.0),
               SamplingParams(min_p=np.float32(0.05), typical_p=1, xtc_threshold=1, xtc_probability=0)):
        sp.validate()
    assert SamplingParams(min_p=0.1).has_truncation() and SamplingParams(typical_p=0.9).has_truncation()
    assert SamplingParams(xtc_probability=0.5).has_truncation() and not SamplingParams(xtc_threshold=0.3).has_truncation()


def _parent_words(params_list, rng):
    """sampling_words of the parent commit without penalties, transcribed."""
    seeds = np.array([int(rng.integers(0, 2 ** 63)) if sp.seed is None else int(sp.seed) for sp in params_list], dtype=np.uint64)
    if all(sp.temperature == 0 for sp in params_list):
        return None
    i32 = lambda w: w.astype(np.uint32).view(np.int32).tolist()    # noqa: E731
    temp = np.array([sp.temperature for sp in params_list], dtype=np.float32)
    top_p = np.array([sp.top_p for sp in params_list], dtype=np.float32)
    words = i32(seeds.view(np.uint32)) + i32(temp.view(np.uint32)) + [int(sp.top_k) for sp in params_list] + \
        i32(top_p.view(np.uint32))
    return words, any(sp.temperature > 0 and (sp.top_k > 0 or sp.top_p < 1) for sp in params_list)


def test_lists_without_truncation_stage_the_parent_words():
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import has_truncation, sampling_words
    lists = [[SamplingParams()] * 3, [SamplingParams(0.7, top_k=5, seed=3)], [SamplingParams(0.5, top_p=0.8, xtc_threshold=0.4)],
             [SamplingParams(0.0, min_p=0.3, typical_p=0.5, xtc_probability=1.0), SamplingParams(0.9, seed=2)],
             [SamplingParams(min_p=0.2)] * 2]
    for sp in lists:
        assert not has_truncation(sp)
        assert sampling_words(sp, len(sp), np.random.default_rng(4)) == _parent_words(sp, np.random.default_rng(4))


def test_truncation_layout_and_state_views():
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import has_truncation, sampling_words
    from swiftllm_b200.worker.infer_state import SamplingState
    for pen in (False, True):
        extra = dict(repetition_penalty=1.2) if pen else {}
        sp = [SamplingParams(0.8, seed=5, min_p=0.05, **extra), SamplingParams(),
              SamplingParams(1.0, seed=6, typical_p=0.9, xtc_threshold=0.2, xtc_probability=0.5)]
        words, filtered = sampling_words(sp, 3, np.random.default_rng(0))
        assert filtered and has_truncation(sp)
        base = (8 if pen else 5) * 3
        assert len(words) == base + 12
        off = [dataclasses.replace(s, min_p=0.0, typical_p=1.0, xtc_threshold=0.1, xtc_probability=0.0) for s in sp]
        assert words[:base] == sampling_words(off, 3, np.random.default_rng(0))[0]
        tail = np.array(words[base:], dtype=np.int32).view(np.float32).reshape(4, 3)
        assert np.array_equal(tail, np.float32([[0.05, 0, 0], [1, 1, 0.9], [0.1, 0.1, 0.2], [0, 0, 0.5]]))
        st = SamplingState.from_staged(torch.tensor(words, dtype=torch.int32), torch.zeros(3, dtype=torch.int32), filtered,
                                       truncated=True)
        assert st.truncated and st.penalized == pen
        assert st.min_p.tolist() == [np.float32(0.05), 0, 0] and st.xtc_probability.tolist() == [0, 0, 0.5]
        assert st.typical_p.tolist() == [1, 1, np.float32(0.9)] and st.top_p.tolist() == [1, 1, 1]
        assert set(st.truncation_kwargs()) == {"min_p", "typical_p", "xtc_threshold", "xtc_probability"}
        plain = SamplingState.from_staged(torch.tensor(words[:base], dtype=torch.int32), torch.zeros(3, dtype=torch.int32), False)
        assert not plain.truncated and plain.truncation_kwargs() == {}
    # only a sampled row's filters count: a greedy row with them stages nothing new, a sampled one filters
    assert sampling_words([SamplingParams(0.5, typical_p=0.9)], 1, np.random.default_rng(0))[1] is True


def test_sample_tokens_truncated_rejects_invalid_arguments_before_launch():
    from swiftllm_b200 import _lib
    l = _lib.lib()
    names = (("logits", 1), ("rows", 2), ("V", 1000), ("stride", 1000), ("off", 0), ("t", 1), ("k", 1), ("p", 1), ("seed", 1),
             ("pos", 1), ("out", 1), ("pairs", None), ("min_p", 1), ("typ", 1), ("xt", 1), ("xp", 1), ("dtype", 1),
             ("stream", None))
    args = lambda **kw: [kw.get(n, d) for n, d in names]      # noqa: E731
    vmax = 8 * (200 * 1024 // 2)
    for kw, msg in (({"dtype": 7}, b"dtype"), ({"V": 0}, b"vocab_size"), ({"V": vmax + 8, "stride": vmax + 8}, b"shared memory"),
                    ({"stride": 999}, b"row_stride"), ({"rows": -1}, b"num_rows"), ({"off": (1 << 24)}, b"2^24"),
                    ({"logits": None}, b"null pointer"), ({"seed": None}, b"null pointer"),
                    ({"min_p": None}, b"null filter array"), ({"typ": None}, b"null filter array"),
                    ({"xt": None}, b"null filter array"), ({"xp": None}, b"null filter array")):
        assert l.sllm_sample_tokens_truncated(*args(**kw)) != 0, kw
        assert msg in l.sllm_last_error() and b"sample_tokens_truncated" in l.sllm_last_error(), (kw, l.sllm_last_error())
    assert l.sllm_sample_tokens_truncated(*args(rows=0, logits=None, min_p=None)) == 0       # empty batch: nothing to launch


# ---------------------------------------------------------------- the host path: graph keys, speculative row words
def test_graph_keys_and_meta_without_and_with_truncation():
    """Steps without the filters keep their graph keys and staged words; a step with them replays its own graph, keyed by one
    more tag, with 4 * B more meta words."""
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200 import SamplingParams
    from test_constraints_cpu import PATCH
    from test_host_path_cpu import CFG, _product
    from test_speculative_cpu import SPEC
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=5, std=0.08)
    with product_on_cpu(PATCH + SPEC):
        m = _product(w, use_cuda_graph=True)
        caps, staged = [], []
        orig = m._stage_metadata

        def fake_capture(B, bucket, filtered=None, top_n=None, penalized=False, sampled=True, con=None, ngram=False,
                         truncated=False):
            caps.append((B, filtered, penalized, truncated))
            nw = 0 if filtered is None else (28 if ngram else 8 if penalized else 5) * B + (4 * B if truncated else 0)
            g = type("G", (), {"replay": lambda self: None})()
            return dict(graph=g, meta=torch.zeros((nw + 3 * B,), dtype=torch.int32), tokens=torch.zeros((B,), dtype=torch.int64),
                        logprobs=None)
        m._capture_decode_graph = fake_capture
        m._stage_metadata = lambda *parts, **kw: (staged.append([len(p) for p in parts]), orig(*parts, **kw))[1]
        m.forward([[1, 2, 3], [4, 5]], [0, 1], [])
        m.forward([[1], [2]], [0, 1], [4, 3], sampling_params_list=[SamplingParams(0.7, seed=1)] * 2)
        m.forward([[1], [2]], [0, 1], [5, 4], sampling_params_list=[SamplingParams(0.0, min_p=0.3)] * 2)   # greedy: ignored
        m.forward([[1], [2]], [0, 1], [6, 5], sampling_params_list=[SamplingParams(0.7, seed=1, min_p=0.1), SamplingParams()])
        m.forward([[1], [2]], [0, 1], [7, 6], sampling_params_list=[SamplingParams(0.7, seed=1, repetition_penalty=1.1,
                                                                                    xtc_probability=0.5)] * 2)
        assert set(m._graphs) == {(2, 1024), (2, 1024, True, False), (2, 1024, True, False, "truncated"),
                                  (2, 1024, True, False, "penalties", True, "truncated")}
        assert staged[1:] == [[10, 2, 2, 2], [2, 2, 2], [18, 2, 2, 2], [24, 2, 2, 2]]
        assert [c[-1] for c in caps] == [False, False, True, True]


def test_speculative_row_words_carry_the_filters_per_row():
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.worker.infer_state import SamplingState
    from test_constraints_cpu import PATCH
    from test_host_path_cpu import CFG, _product
    from test_speculative_cpu import SPEC
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=5, std=0.08)
    with product_on_cpu(PATCH + SPEC):
        m = _product(w)
        m.forward([[1, 2, 3], [4, 5]], [0, 1], [])
        seen = []
        m._forward = lambda ids, st: (seen.append(st.sampling), torch.zeros((st.num_tokens,), dtype=torch.int64))[1]
        sp = [SamplingParams(0.8, seed=3, min_p=0.05), SamplingParams(1.0, seed=4, typical_p=0.7, xtc_probability=0.25)]
        m.forward_speculative([[7, 8, 9], [6]], [0, 1], [3, 2], sampling_params_list=sp)
        st = seen[0]
        assert st.truncated
        assert st.min_p.tolist() == [np.float32(0.05)] * 3 + [0.0]
        assert st.typical_p.tolist() == [1.0] * 3 + [np.float32(0.7)]
        assert st.xtc_probability.tolist() == [0.0] * 3 + [0.25] and st.xtc_threshold.tolist() == [np.float32(0.1)] * 4
        assert st.seed.tolist() == [3, 3, 3, 4] and st.pos.tolist() == [4, 5, 6, 3]
        m.forward_speculative([[7, 8], [6]], [0, 1], [3, 2], sampling_params_list=[SamplingParams(0.8, seed=3)] * 2)
        assert not seen[1].truncated


def test_xtc_threshold_zero_never_keeps_only_masked_ids():
    """A -inf id is never an XTC top choice: threshold 0 stops at the least likely finite survivor."""
    t = torch.tensor([3.0, 1.0, float("-inf"), 0.5, float("-inf")], dtype=torch.bfloat16)
    b, v = t.view(torch.int16).numpy().view(np.uint16), t.float().numpy()
    for seed in range(20):
        res = TO.sample_row(b, v, 1.0, 0, 1.0, seed, 7, xtc_threshold=0.0, xtc_probability=1.0)
        assert res.token == 3 and res.kept[3] and res.boundary_margin == np.inf, res


# ---------------------------------------------------------------- tensor parallelism over gloo
def _trunc_stand_in(logits, temperature, top_k, top_p, seed, pos, vocab_offset=0, out_pairs=None, min_p=None, typical_p=None,
                    xtc_threshold=None, xtc_probability=None):
    """The kernel restated on CPU; records the shape and offset of every launch with the filters."""
    B = logits.shape[0]
    f = [min_p, typical_p, xtc_threshold, xtc_probability]
    if min_p is not None:
        _trunc_stand_in.calls.append((logits.shape[1], vocab_offset))
    f = [[0.0] * B, [1.0] * B, [0.1] * B, [0.0] * B] if min_p is None else [x.tolist() for x in f]
    res = TO.sample_tokens(logits, temperature.tolist(), top_k.tolist(), top_p.tolist(), seed.tolist(), pos.tolist(), *f,
                           vocab_offset=vocab_offset)
    if out_pairs is not None:
        out_pairs.copy_(torch.tensor([[r.score, float(r.token)] for r in res], dtype=torch.float32))
    return torch.tensor([r.token for r in res], dtype=torch.int64)


_trunc_stand_in.calls = []


def _tp_params(step):
    from swiftllm_b200 import SamplingParams
    if step % 2:                                        # no filter, no top-k / top-p: the pair exchange of a sharded lm_head
        return [SamplingParams(0.9, seed=50 + i) for i in range(2)]
    return [SamplingParams(1.0, seed=60 + step, min_p=0.05, typical_p=0.9),
            SamplingParams(0.8, seed=70 + step, top_k=30, xtc_threshold=0.02, xtc_probability=1.0)]


def _tp_worker(rank, world, port, ret, shard_lm_head):
    """The product model with tp_size = world on CPU against the unsharded oracle model: the restatement applied to the
    unsharded logits gives the tokens every rank returns, and the filters only ever see whole rows."""
    import os
    import sys
    import warnings
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import swiftllm_b200
    from cpu_shim import product_on_cpu
    from oracle.model import OracleLlama, OracleWeights
    from swiftllm_b200.worker.weight import dict_getter
    from test_host_path_cpu import _hf_tensors
    from test_tp_gloo import CFG
    cfg = dict(CFG, num_hidden_layers=2, vocab_size=96)
    w = OracleWeights.random(cfg, dtype=torch.float16, seed=12, std=0.08)
    ok, toks_all = True, []
    with product_on_cpu([("swiftllm_b200.worker.layers.post_layer", "sample_tokens", _trunc_stand_in)]), \
            warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=2,
                                        max_seqs_in_block_table=8, max_blocks_per_seq=8, max_batch_size=8, max_tokens_in_batch=128,
                                        dtype="float16", tp_size=world, tp_rank=rank, shard_lm_head=shard_lm_head,
                                        fused_allreduce=False)
        m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(cfg))
        m.load_weights(dict_getter(_hf_tensors(w, cfg["intermediate_size"])))
        m.init_kvcache_and_swap(20)
        o = OracleLlama(cfg, w, block_size=16, num_blocks=20, num_cpu_blocks=2, max_seqs_in_block_table=8, max_blocks_per_seq=8,
                        attn="exact", dtype=torch.float16)
        rng = np.random.default_rng(2)
        ids = [rng.integers(0, 96, size=n).tolist() for n in (21, 3)]
        sids, lens, dec = [4, 1], [21, 3], []
        for step in range(6):
            sp = _tp_params(step)
            _trunc_stand_in.calls.clear()
            got = m.forward(ids, sids, dec, sampling_params_list=sp)
            o.forward(ids, sids, dec)
            if step % 2 == 0:
                ok &= _trunc_stand_in.calls == [(96, 0)]           # whole rows: gathered when the lm_head is sharded
            f = [[getattr(s, n) for s in sp] for n in ("min_p", "typical_p", "xtc_threshold", "xtc_probability")]
            ref = TO.sample_tokens(o.last_logits, [s.temperature for s in sp], [s.top_k for s in sp], [s.top_p for s in sp],
                                   [s.seed for s in sp], lens, *f)
            for t, r in zip(got, ref):
                ok &= t == r.token or r.gap <= 2e-2 or r.boundary_margin <= 1e-2     # fp16 logits within tolerance
            toks_all.append(got)
            lens = [l + 1 for l in lens]
            ids, dec = [[t] for t in got], lens
    gathered = [None] * world
    dist.all_gather_object(gathered, (bool(ok), toks_all))
    if rank == 0:
        ret.put(gathered)
    dist.destroy_process_group()


@pytest.mark.parametrize("shard_lm_head", [False, True], ids=["replicated-lm_head", "vocab-sharded-lm_head"])
def test_tensor_parallel_truncation_equals_unsharded_on_cpu(shard_lm_head):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    port = 29711 + (7 if shard_lm_head else 0)
    procs = [ctx.Process(target=_tp_worker, args=(r, 2, port, ret, shard_lm_head)) for r in range(2)]
    for p in procs:
        p.start()
    got = ret.get(timeout=240)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(ok for ok, _ in got), got
    assert got[0][1] == got[1][1]                               # every rank returns the same tokens
