"""CPU: constrained decoding (allowed-token masks and logit bias).  The semantics (tests/constraints_oracle.py) on hand-made rows,
the C ABI's argument checks, the host-side validation, and the constraints through the product's host path with a torch stand-in
of the kernel - greedy and seeded rows, mixed and chunked steps, masks that change every step, penalties on top, raw
log-probabilities, speculative verification, the graph path's key and staging, and a vocabulary-sharded lm_head over gloo."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import constraints_oracle as CO
import penalties_oracle as PO
import sampling_oracle as SO
from test_penalties_cpu import PATCH as PEN_PATCH, _History

V_CFG = 300                                     # tests/test_host_path_cpu.py: CFG["vocab_size"]


def _row(vals, dtype=torch.float16):
    return torch.tensor(vals, dtype=torch.float32).to(dtype)


def _bits(t):
    return t.view(torch.int16)


def _mask(V, ids):
    from swiftllm_b200 import token_mask
    return token_mask(V, ids)


# ---------------------------------------------------------------- the restatement
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_mask_only_bias_only_and_both(dtype):
    row = _row([1.0, 2.0, -3.0, 0.5, 4.0, -0.25], dtype)
    ninf = float("-inf")
    assert CO.constrain_row(row, _mask(6, [1, 3])).tolist() == [ninf, 2.0, ninf, 0.5, ninf, ninf]
    assert CO.constrain_row(row, None, {0: 1.0, 5: -2.0}).tolist() == [2.0, 2.0, -3.0, 0.5, 4.0, -2.25]
    assert CO.constrain_row(row, _mask(6, [0, 2, 4]), {0: 0.5, 2: 3.0, 3: 10.0}).tolist() == [1.5, ninf, 0.0, ninf, 4.0, ninf]
    assert torch.equal(_bits(CO.constrain(row[None], [None], [None])), _bits(row[None]))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_allowed_unbiased_special_values_keep_their_bits(dtype):
    row = _row([float("nan"), float("inf"), float("-inf"), -0.0, 1.0, 0.0], dtype)
    out = CO.constrain_row(row, _mask(6, [0, 1, 2, 3]), {4: 1.0, 1: 5.0, 2: 3.0})
    assert torch.equal(_bits(out[:4])[[0, 3]], _bits(row)[[0, 3]])
    assert out[1].item() == float("inf") and out[2].item() == float("-inf")     # inf + b = inf, -inf + b = -inf
    assert out[4].item() == float("-inf") and out[5].item() == float("-inf")    # masked, bias or not
    nan_b = CO.constrain_row(_row([float("nan"), -float("nan")], dtype), None, {0: 2.0, 1: -1.0})
    assert _bits(nan_b).tolist() == [CO.CANONICAL_NAN, CO.CANONICAL_NAN]      # a biased NaN stays NaN (the device's NaN)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_bias_is_one_fp32_add_rounded_once(dtype):
    g = torch.Generator().manual_seed(1)
    row = (torch.randn(500, generator=g) * 8).to(dtype)
    bias = {int(v): float(b) for v, b in zip(torch.randperm(500, generator=g)[:200], torch.rand(200, generator=g) * 200 - 100)}
    out = CO.constrain_row(row, None, bias)
    for v in range(500):
        if v not in bias:
            assert _bits(out[v:v + 1]) == _bits(row[v:v + 1])
            continue
        s = np.float32(np.float32(row[v].float().item()) + np.float32(bias[v]))
        assert out[v].item() == torch.tensor(float(s)).to(dtype).item()
    if dtype == torch.float16:                  # overflow of the rounding: 65504 + 100 -> inf
        assert CO.constrain_row(_row([65504.0], dtype), None, {0: 100.0}).item() == float("inf")
        assert CO.constrain_row(_row([65504.0], dtype), None, {0: 8.0}).item() == 65504.0


def test_tail_bits_past_the_vocabulary_are_ignored_and_shards_use_global_ids():
    from swiftllm_b200 import token_mask
    m = ~token_mask(70, [3, 40, 69])                         # bans 3, 40, 69; bits 70..95 set and ignored
    out = CO.constrain_row(_row([1.0] * 70), m)
    assert [i for i in range(70) if out[i].item() == float("-inf")] == [3, 40, 69]
    # a shard starting at global id 45 (not a multiple of 32) of V = 70: local i is global 45 + i
    full = _row(np.arange(70) * 0.5)
    allowed = [1, 44, 45, 63, 64, 69]
    bias = {45: 1.0, 64: -1.0, 10: 5.0, 63: 2.0}
    want = CO.constrain_row(full, token_mask(70, allowed), bias)
    got = torch.cat([CO.constrain_row(full[:45], token_mask(70, allowed), bias, 0),
                     CO.constrain_row(full[45:], token_mask(70, allowed), bias, 45)])
    assert torch.equal(_bits(got), _bits(want))


# ---------------------------------------------------------------- token_mask, validation, the C ABI
def test_token_mask_round_trips():
    from swiftllm_b200 import token_mask
    rng = np.random.default_rng(0)
    for V in (1, 31, 32, 33, 1000, 128256):
        ids = np.unique(rng.integers(0, V, size=min(V, 50)))
        m = token_mask(V, ids)
        assert m.dtype == np.int32 and m.shape == ((V + 31) // 32,)
        assert np.flatnonzero(CO.allowed_ids(m, 0, V)).tolist() == ids.tolist()
        assert np.flatnonzero(CO.allowed_ids(~m, 0, V)).tolist() == sorted(set(range(V)) - set(ids.tolist()))
    assert token_mask(40, []).tolist() == [0, 0]
    for bad in ([-1], [40], [1.5]):
        with pytest.raises(ValueError):
            token_mask(40, bad)


@pytest.mark.parametrize("bad", [[1], {1: float("nan")}, {1: float("inf")}, {1: 100.5}, {1: -101}, {-1: 1.0}, {True: 1.0},
                                 {"3": 1.0}, {1: "2"}, {1: None}, {i: 0.0 for i in range(1025)}])
def test_bad_logit_bias_raises_value_error(bad):
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import sampling_words
    with pytest.raises(ValueError, match="logit_bias"):
        sampling_words([SamplingParams(logit_bias=bad)], 1, np.random.default_rng(0))


def test_mask_and_list_validation():
    from swiftllm_b200 import MAX_LOGIT_BIAS, SamplingParams, token_mask
    from swiftllm_b200.sampling_params import constraint_words
    V, W = 100, 4
    ok = token_mask(V, [7])
    SamplingParams(logit_bias={i: 100.0 for i in range(MAX_LOGIT_BIAS)}).validate()
    assert constraint_words(None, None, 2, V) is None and constraint_words([None, None], [SamplingParams()] * 2, 2, V) is None
    assert constraint_words([None], [SamplingParams(logit_bias={})], 1, V) is None
    for masks, msg in (([ok], "2 entries|1 entries"), ([ok, ok, ok], "entries"), ([ok.astype(np.int64), None], "int32"),
                       ([ok[:3], None], "shape"), ([np.zeros(W, np.int32), None], "allows no token"),
                       ([(~token_mask(V, range(V))), None], "allows no token"), ([[1, 2, 3, 4], None], "numpy"),
                       ([torch.from_numpy(ok).to(torch.int16), None], "int32")):
        with pytest.raises(ValueError, match=msg):
            constraint_words(masks, None, 2, V)
    with pytest.raises(ValueError, match="outside"):
        constraint_words(None, [SamplingParams(logit_bias={V: 1.0})], 1, V)
    # uint32 arrays and CPU tensors of either dtype are accepted and stage the same words
    a = constraint_words([ok], None, 1, V).words
    for m in (ok.view(np.uint32), torch.from_numpy(ok.copy()), torch.from_numpy(ok.copy()).view(torch.uint32)):
        assert np.array_equal(constraint_words([m], None, 1, V).words, a)
    # speculative: [rows_i, W] per entry
    two = np.stack([ok, token_mask(V, [1, 2])])
    constraint_words([two, None], None, 2, V, rows=[2, 3])
    for m in (two[:1], ok):
        with pytest.raises(ValueError, match="shape"):
            constraint_words([m, None], None, 2, V, rows=[2, 3])
    with pytest.raises(ValueError, match="row 1"):
        constraint_words([np.stack([ok, np.zeros(W, np.int32)])], None, 1, V, rows=[2])


def test_staged_region_layout_and_graph_padding():
    from swiftllm_b200 import SamplingParams, token_mask
    from swiftllm_b200.sampling_params import ConstraintWords, constraint_words
    from swiftllm_b200.worker.infer_state import ConstraintState
    V = 70
    m0, m2 = token_mask(V, [1, 69]), token_mask(V, [5])
    sp = [SamplingParams(logit_bias={9: 1.5, 3: -2.0}), SamplingParams(), SamplingParams(logit_bias={4: 0.25})]
    for graph in (False, True):
        cw = constraint_words([m0, None, m2], sp, 3, V, graph=graph)
        assert len(cw.words) == ConstraintWords.size(*cw[1:])
        st = ConstraintState.from_staged(torch.from_numpy(cw.words), *cw[1:])
        assert st.bias_index.tolist() == [0, -1, 2] and st.bias_starts.tolist() == [0, 2, 2, 3]
        assert st.bias_ids.tolist()[:3] == [3, 9, 4] and st.bias_values.tolist()[:3] == [-2.0, 1.5, 0.25]
        if graph:                                           # one mask slot per row, bias arrays padded to 4 with id -1
            assert st.mask_index.tolist() == [0, -1, 2] and cw.num_masks == 3 and cw.num_bias == 4
            assert st.bias_ids.tolist()[3] == -1 and not st.masks[1].any()
        else:
            assert st.mask_index.tolist() == [0, -1, 1] and cw.num_masks == 2 and cw.num_bias == 3
        assert np.array_equal(st.masks[st.mask_index[2]].numpy(), m2)
    assert constraint_words(None, [SamplingParams(logit_bias={i: 1.0 for i in range(5)})], 1, V, graph=True).num_bias == 8
    assert constraint_words([m0], None, 1, V, graph=True).num_bias == 0


def test_constrain_logits_rejects_invalid_arguments_before_launch():
    from swiftllm_b200 import _lib
    l = _lib.lib()
    names = (("logits", 1), ("rows", 2), ("V", 1000), ("stride", 1000), ("off", 0), ("mi", 1), ("masks", 1), ("nm", 2),
             ("mw", 32), ("bi", 1), ("bs", 1), ("ne", 2), ("bids", 1), ("bvals", 1), ("nb", 3), ("dtype", 1), ("stream", None))
    args = lambda **kw: [kw.get(n, d) for n, d in names]
    for kw, msg in (({"dtype": 7}, b"dtype"), ({"V": 0}, b"vocab_size"), ({"stride": 999}, b"row_stride"),
                    ({"rows": -1}, b"num_rows"), ({"rows": 2 ** 31}, b"num_rows"), ({"off": -1}, b"2^31"),
                    ({"off": 2 ** 31 - 1000}, b"2^31"), ({"mw": 31}, b"mask_words"), ({"mw": 0}, b"mask_words"),
                    ({"off": 100, "mw": 32}, b"mask_words"), ({"nm": -1}, b"num_masks"), ({"ne": -1}, b"num_entries"),
                    ({"nb": -1}, b"num_bias"), ({"logits": None}, b"null pointer"), ({"mi": None}, b"null pointer"),
                    ({"masks": None}, b"null pointer"), ({"bi": None}, b"null pointer"), ({"bs": None}, b"null pointer"),
                    ({"bids": None}, b"null pointer"), ({"bvals": None}, b"null pointer")):
        assert l.sllm_constrain_logits(*args(**kw)) != 0, kw
        assert msg in l.sllm_last_error(), (kw, l.sllm_last_error())
    # the largest shard below 2^31 passes the range check; empty arrays may be NULL
    assert l.sllm_constrain_logits(*args(off=2 ** 31 - 1001, mw=2 ** 26, dtype=7)) != 0 and b"dtype" in l.sllm_last_error()
    assert l.sllm_constrain_logits(*args(masks=None, nm=0, bs=None, ne=0, bids=None, bvals=None, nb=0, dtype=7)) != 0
    assert b"dtype" in l.sllm_last_error()
    assert l.sllm_constrain_logits(*args(rows=0, logits=None, mi=None, bi=None)) == 0     # empty batch: nothing to launch


# ---------------------------------------------------------------- host path with a stand-in of the kernel
CON_CALLS = []


def _con_stand_in(logits, mask_index, masks, bias_index, bias_starts, bias_ids, bias_values, vocab_offset=0):
    """csrc/constraints.cu on CPU tensors: the staged arrays decoded row by row, the restatement applied in place."""
    CON_CALLS.append((tuple(logits.shape), vocab_offset))
    ms, bs = [], []
    for r in range(logits.shape[0]):
        mi, bi = int(mask_index[r]), int(bias_index[r])
        ms.append(None if mi < 0 else masks[mi].numpy())
        bs.append(None if bi < 0 else {int(bias_ids[j]): float(bias_values[j])
                                       for j in range(int(bias_starts[bi]), int(bias_starts[bi + 1]))})
    logits.copy_(CO.constrain(logits, ms, bs, vocab_offset))


PATCH = PEN_PATCH + [("swiftllm_b200.worker.layers.post_layer", "constrain_logits", _con_stand_in)]


def _biases(sp_list):
    return [None if sp is None else sp.logit_bias for sp in sp_list]


def _expected(m, sp_list, masks, hists=None):
    """The step's token restated from its raw logits: constraints, then penalties, then argmax or the sampling restatement."""
    x = CO.constrain(m.post_layer.last_logits, masks, _biases(sp_list) if sp_list else [None] * len(masks))
    if sp_list is not None and any(s.has_penalties() for s in sp_list):
        x = PO.penalize(x, [(s.repetition_penalty, s.frequency_penalty, s.presence_penalty) for s in sp_list], hists)
    if sp_list is None or all(s.temperature == 0 for s in sp_list):
        return torch.argmax(x, dim=1).tolist()
    st = m._last_sampling
    return [r.token for r in SO.sample_tokens(x, [s.temperature for s in sp_list], [s.top_k for s in sp_list],
                                              [s.top_p for s in sp_list], st.seed.tolist(), st.pos.tolist())]


def _random_masks(rng, n, V, p_none=0.25):
    from swiftllm_b200 import token_mask
    out = []
    for _ in range(n):
        r = rng.random()
        if r < p_none:
            out.append(None)
        elif r < 0.45:
            out.append(token_mask(V, [int(rng.integers(0, V))]))                        # one id
        else:
            ids = np.flatnonzero(rng.random(V) < rng.choice([0.02, 0.3, 0.8]))
            out.append(token_mask(V, ids if ids.size else [0]))
    return out


def _params(rng, n, penalties=False):
    from swiftllm_b200 import SamplingParams
    out = []
    for i in range(n):
        t = float(rng.choice([0.0, 0.0, 0.8, 1.3]))
        bias = None if rng.random() < 0.4 else {int(v): float(rng.uniform(-100, 100)) for v in rng.choice(V_CFG, 5, replace=False)}
        kw = dict(top_k=int(rng.choice([0, 7])), top_p=float(rng.choice([1.0, 0.9])), seed=int(rng.integers(0, 99)))
        if penalties:
            kw.update(repetition_penalty=1.3, frequency_penalty=0.5)
        out.append(SamplingParams(t, logit_bias=bias, **kw))
    return out


@pytest.mark.parametrize("kind", ["greedy", "sampled", "penalised"])
def test_constrained_host_path_on_cpu(kind):
    """prefill -> decodes -> chunked prefill -> mixed batch, with fresh masks and biases every step: every token is the restatement
    applied to the step's raw logits (then the penalties over the tracked history), and every masked token is allowed."""
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200 import SamplingParams
    from test_host_path_cpu import _product
    from test_sampling_cpu import _record_sampling
    w = OracleWeights.random(__import__("test_host_path_cpu").CFG, dtype=torch.float16, seed=4, std=0.08)
    rng = np.random.default_rng({"greedy": 1, "sampled": 2, "penalised": 3}[kind])
    with product_on_cpu(PATCH):
        m = _product(w)
        _record_sampling(m)
        H = _History()
        CON_CALLS.clear()
        fixed = {}

        def step(ids, sids, lens, n_pre, prefix=None):
            if kind == "greedy":
                sp = None if rng.random() < 0.5 else [SamplingParams(logit_bias=_params(rng, 1)[0].logit_bias) for _ in sids]
            else:
                sp = [fixed.setdefault(s, _params(rng, 1, kind == "penalised")[0]) for s in sids]
                if kind == "sampled":      # biases change every step too
                    sp = [SamplingParams(p.temperature, p.top_k, p.top_p, p.seed, logit_bias=_params(rng, 1)[0].logit_bias)
                          for p in sp]
            masks = _random_masks(rng, len(ids), V_CFG)
            hists = H.step(ids, sids, n_pre, prefix)
            kw = {} if prefix is None else dict(prefill_prefix_lens_list=prefix)
            t = m.forward(ids, sids, lens, sampling_params_list=sp, token_masks_list=masks, **kw)
            assert t == _expected(m, sp, masks, hists)
            for tok, mk in zip(t, masks):
                assert mk is None or CO.allowed_ids(mk, tok, tok + 1)[0]
            return dict(zip(sids, t))

        prompts = [rng.integers(0, 300, size=n).tolist() for n in (12, 5, 30, 9)]
        sids = [0, 1, 2, 4]
        t = step(prompts, sids, [], 4)
        lens = {0: 12, 1: 5, 2: 30, 4: 9}
        for _ in range(4):
            lens = {s: l + 1 for s, l in lens.items()}
            t = step([[t[s]] for s in sids], sids, [lens[s] for s in sids], 0)
        p3 = rng.integers(0, 300, size=40).tolist()
        step([p3[:16]], [3], [], 1, prefix=[0])
        lens = {s: l + 1 for s, l in lens.items()}
        step([p3[16:40]] + [[t[s]] for s in sids], [3] + sids, [lens[s] for s in sids], 1, prefix=[16])
        assert CON_CALLS and all(shape[1] == V_CFG and off == 0 for shape, off in CON_CALLS)


def test_a_single_allowed_id_forces_the_token():
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200 import SamplingParams, token_mask
    from test_host_path_cpu import CFG, _product
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=8, std=0.08)
    with product_on_cpu(PATCH):
        a = _product(w)
        prompts = [[1, 2, 3], [4, 5, 6, 7], [8, 9]]
        forced = [17, 299, 0]
        sp = [SamplingParams(1.5, seed=3), SamplingParams(0.0), SamplingParams(0.7, top_k=3, seed=4, logit_bias={0: -100.0})]
        t = a.forward(prompts, [0, 1, 2], [], sampling_params_list=sp, token_masks_list=[token_mask(V_CFG, [f]) for f in forced])
        assert t == forced
        masks = [None, ~token_mask(V_CFG, range(0, 290)), token_mask(V_CFG, range(5, 200))]
        t = a.forward([[x] for x in t], [0, 1, 2], [4, 5, 3], sampling_params_list=sp, token_masks_list=masks)
        assert 290 <= t[1] < 300 and 5 <= t[2] < 200


def test_logprobs_stay_raw_next_to_constrained_tokens():
    """forward_with_logprobs with masks and biases (and penalties on one row): the log-probabilities are bit-equal to those of an
    unconstrained call on the same state, the tokens respect the masks, and last_logits stays raw."""
    import logprobs_oracle as LO
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200 import SamplingParams
    from test_host_path_cpu import CFG, _product
    from test_sampling_cpu import _record_sampling
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=6, std=0.08)
    rng = np.random.default_rng(5)
    with product_on_cpu(PATCH):
        a, b = _product(w), _product(w)
        for m in (a, b):
            _record_sampling(m)
        H = _History()
        sp = [SamplingParams(0.0, logprobs=3, repetition_penalty=2.0, logit_bias={5: 30.0}),
              SamplingParams(0.9, seed=3, logprobs=0), SamplingParams(0.0, logprobs=2, logit_bias={1: -5.0, 2: 5.0})]
        plain = [SamplingParams(s.temperature, seed=s.seed, logprobs=s.logprobs) for s in sp]
        ids, sids, lens = [[5, 6, 5, 7], [9, 9], [1, 2, 3]], [0, 1, 2], []
        moved = 0
        for s in range(4):
            masks = _random_masks(rng, 3, V_CFG, p_none=0.0)
            hists = H.step(ids, sids, 3 if s == 0 else 0)
            ref = a.forward_with_logprobs(ids, sids, lens, sampling_params_list=plain)
            res = b.forward_with_logprobs(ids, sids, lens, sampling_params_list=sp, token_masks_list=masks)
            assert torch.equal(a.post_layer.last_logits, b.post_layer.last_logits)
            t = [r.token for r in res]
            assert t == _expected(b, sp, masks, hists)
            tl, ids_top, tlp = LO.token_logprobs(b.post_layer.last_logits, t, 3)
            for i, (r, q) in enumerate(zip(res, ref)):
                assert CO.allowed_ids(masks[i], r.token, r.token + 1)[0]
                assert r.top == q.top and r.logprob == float(tl[i])
            moved += sum(r.token != q.token for r, q in zip(res, ref))
            lens = [len(h) + 1 for h in hists]
            ids = [[x] for x in t]                       # both models are fed b's tokens: their caches stay identical
        assert moved > 0


def test_constraints_with_ignore_kvcache_and_bad_arguments_raise_before_anything_is_enqueued():
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200 import SamplingParams, token_mask
    from test_host_path_cpu import CFG, _product
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=2, std=0.08)
    with product_on_cpu(PATCH):
        m = _product(w)
        staged = []
        orig = m._stage_metadata
        m._stage_metadata = lambda *parts, **kw: (staged.append(1), orig(*parts, **kw))[1]
        CON_CALLS.clear()
        ok = token_mask(V_CFG, [3])
        for call, msg in ((lambda: m.forward([[1, 2]], [0], [], ignore_kvcache=True, token_masks_list=[ok]), "ignore_kvcache"),
                          (lambda: m.forward([[1, 2]], [0], [], token_masks_list=[ok, ok]), "entries"),
                          (lambda: m.forward([[1, 2]], [0], [], token_masks_list=[ok[:-1]]), "shape"),
                          (lambda: m.forward([[1, 2]], [0], [], token_masks_list=[np.zeros_like(ok)]), "allows no"),
                          (lambda: m.forward_with_logprobs([[1, 2]], [0], [], token_masks_list=[ok.astype(np.float32)]), "int32"),
                          (lambda: m.forward([[1, 2]], [0], [], sampling_params_list=[SamplingParams(logit_bias={300: 1.0})]),
                           "outside"),
                          (lambda: m.forward_speculative([[1, 2]], [0], [0], token_masks_list=[ok]), "shape")):
            with pytest.raises(ValueError, match=msg):
                call()
        assert staged == [] and CON_CALLS == [] and m.gpu_block_manager.num_free_blocks == m.gpu_block_manager.num_blocks
        # the profiling forward takes a bias (no token history needed)
        m.forward([[1, 2]], [0], [], ignore_kvcache=True, sampling_params_list=[SamplingParams(logit_bias={3: 1.0})])


# ---------------------------------------------------------------- unconstrained steps do what the parent did
def test_unconstrained_steps_stage_launch_and_key_their_graphs_as_before():
    """No masks (None, or a list of None) and no logit_bias (None or {}): the staged parts are exactly those of a call without
    the new arguments - the parent's staging, restated in test_penalties_cpu / test_sampling_cpu - no constraint kernel runs,
    and the graph path keeps its key and meta length.  A constrained graph step adds ("constrained", bias capacity) to the key
    and the region to meta."""
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200 import SamplingParams, token_mask
    from swiftllm_b200.sampling_params import ConstraintWords
    from test_host_path_cpu import CFG, _product
    from test_speculative_cpu import SPEC
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=5, std=0.08)
    with product_on_cpu(PATCH + SPEC):
        runs = []
        for variant in range(3):
            m = _product(w)
            staged = []
            orig = m._stage_metadata
            m._stage_metadata = lambda *parts, **kw: (staged.append([list(p) for p in parts]), orig(*parts, **kw))[1]
            CON_CALLS.clear()
            kw = [dict(), dict(token_masks_list=[None, None]), dict(token_masks_list=[None, None])][variant]
            mk = lambda sp: [SamplingParams(s.temperature, s.top_k, s.top_p, s.seed, s.logprobs,
                                            logit_bias=[None, None, {}][variant]) for s in sp]
            toks = []
            for sp in (None, [SamplingParams()] * 2, [SamplingParams(0.9, seed=4), SamplingParams(0.0, logprobs=2)]):
                t = m.forward([[1, 2, 3], [4, 5]], [0, 1], [], sampling_params_list=sp and mk(sp), **kw)
                t += m.forward([[t[0]], [t[1]]], [0, 1], [4, 3], sampling_params_list=sp and mk(sp), **kw)
                t += [r.token for r in m.forward_with_logprobs([[t[2]], [t[3]]], [0, 1], [5, 4], sampling_params_list=sp and mk(sp),
                                                                **kw)]
                m.free_seqs_resources([0, 1])
                toks.append(t)
            spec = m.forward_speculative([[1, 2, 3]], [0], [0], **({} if not kw else dict(token_masks_list=[None])))
            runs.append((staged, toks, spec))
            assert CON_CALLS == []
        assert runs[0] == runs[1] == runs[2]

        # graph path: the key and the staged meta, with a stand-in capture (capturing needs a device)
        for variant in ("plain", "constrained"):
            m = _product(w, use_cuda_graph=True)
            caps, staged = [], []
            orig = m._stage_metadata

            def fake_capture(B, bucket, filtered=None, top_n=None, penalized=False, sampled=True, con=None):
                caps.append((B, filtered, top_n, penalized, sampled, con))
                nw = 0 if filtered is None else (8 if penalized else 5) * B
                nc = 0 if con is None else ConstraintWords.size(*con[1:])
                g = type("G", (), {"replay": lambda self: None})()
                return dict(graph=g, meta=torch.zeros((nw + nc + 3 * B,), dtype=torch.int32), tokens=torch.zeros((B,), dtype=torch.int64),
                            logprobs=None)
            m._capture_decode_graph = fake_capture
            m._stage_metadata = lambda *parts, **kw: (staged.append([len(p) for p in parts]), orig(*parts, **kw))[1]
            m.forward([[1, 2, 3], [4, 5]], [0, 1], [])
            if variant == "plain":
                m.forward([[1], [2]], [0, 1], [4, 3], token_masks_list=[None, None])
                m.forward([[1], [2]], [0, 1], [5, 4], sampling_params_list=[SamplingParams(0.5, seed=1, logit_bias={})] * 2)
                assert [c[-1] for c in caps] == [None, None] and all(len(k) == 2 or k[2:] == (True, False) for k in m._graphs)
                assert staged[1:] == [[2, 2, 2], [10, 2, 2, 2]]
            else:
                bias = {i: 1.0 for i in range(3)}
                m.forward([[1], [2]], [0, 1], [4, 3], token_masks_list=[token_mask(V_CFG, [4]), None])
                m.forward([[1], [2]], [0, 1], [5, 4], sampling_params_list=[SamplingParams(logit_bias=bias)] * 2)
                keys = list(m._graphs)
                assert keys[0][-2:] == ("constrained", 0) and keys[1][-2:] == ("constrained", 8)
                W = (V_CFG + 31) // 32
                assert staged[1:] == [[ConstraintWords.size(2, 2, W, 2, 0), 2, 2, 2], [ConstraintWords.size(2, 2, W, 2, 8), 2, 2, 2]]
                assert caps[0][-1][1:] == (2, 2, W, 2, 0)


# ---------------------------------------------------------------- speculative verification
@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "seeded-sampling"])
def test_speculative_with_per_row_masks_returns_the_plain_masked_steps(sampled):
    """Drafts from a plain run with masks (row j's mask = the plain step's at that position), one of them replaced by an id its
    row's mask disallows: forward_speculative returns exactly the plain steps' tokens up to and including that row."""
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200 import SamplingParams, token_mask
    from test_host_path_cpu import CFG, _product
    from test_speculative_cpu import SPEC
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=9, std=0.08)
    rng = np.random.default_rng(7 + sampled)
    sp = SamplingParams(0.9 if sampled else 0.0, seed=21, logit_bias={7: 3.0, 11: -4.0})
    with product_on_cpu(PATCH + SPEC):
        plain, spec = _product(w), _product(w)
        for sid, (k, wrong) in enumerate(((5, 2), (7, None), (3, 0), (6, 5))):
            prompt = rng.integers(0, 300, size=13 + sid).tolist()
            x = plain.forward([prompt], [sid], [], sampling_params_list=[sp])[0]
            assert spec.forward([prompt], [sid], [], sampling_params_list=[sp])[0] == x
            L = len(prompt)
            masks = [token_mask(V_CFG, np.flatnonzero(rng.random(V_CFG) < 0.2)) for _ in range(k + 1)]
            ys, inp = [], x
            for j in range(k + 1):
                ys.append(plain.forward([[inp]], [sid], [L + j + 1], sampling_params_list=[sp], token_masks_list=[masks[j]])[0])
                inp = ys[-1]
            drafts = list(ys[:k])
            if wrong is not None:                   # an id row `wrong`'s mask disallows
                drafts[wrong] = int(np.flatnonzero(~CO.allowed_ids(masks[wrong], 0, V_CFG))[0])
            out = spec.forward_speculative([[x] + drafts], [sid], [L], sampling_params_list=[sp],
                                           token_masks_list=[np.stack(masks)])[0]
            assert out == ys[:(k if wrong is None else wrong) + 1]


# ---------------------------------------------------------------- vocabulary-sharded lm_head over gloo
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
    V = 104 if world == 4 else 96                    # shards of 26 / 48 ids: boundaries off the 32-id words
    cfg = dict(CFG, num_hidden_layers=2, vocab_size=V)
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
        CON_CALLS.clear()
        rng = np.random.default_rng(2)
        ids = [rng.integers(0, V, size=n).tolist() for n in (21, 3, 9, 4)]
        sids, dec, lens = [4, 1, 2, 3], [], [21, 3, 9, 4]
        Vs = V // world
        for step in range(4):
            sp = [swiftllm_b200.SamplingParams(t, top_k=(5 if filtered and i == 1 else 0), seed=30 + i,
                                               logit_bias={int(v): 40.0 - 20 * i for v in rng.choice(V, 3, replace=False)})
                  for i, t in enumerate([0.9, 1.1, 0.0, 0.0])]
            masks = [swiftllm_b200.token_mask(V, rng.choice(Vs, 2, replace=False) + Vs * (world - 1)),     # last shard only
                     swiftllm_b200.token_mask(V, np.flatnonzero(rng.random(V) < 0.3)),
                     swiftllm_b200.token_mask(V, [Vs + 1]),                                              # one id, second shard
                     None]
            got = sharded.forward(ids, sids, dec, sampling_params_list=sp, token_masks_list=masks)
            ref = full.forward(ids, sids, dec, sampling_params_list=sp, token_masks_list=masks)
            ok &= got == ref
            ok &= torch.equal(sharded.post_layer.last_logits, full.post_layer.last_logits)
            ok &= all(m is None or CO.allowed_ids(m, t, t + 1)[0] for m, t in zip(masks, got))
            out.append(got)
            lens = [l + 1 for l in lens]
            ids, dec = [[x] for x in got], lens
        calls = CON_CALLS[0::2]                      # the sharded model's calls (the unsharded model's follow each)
        ok &= all(c == ((4, V), 0) for c in calls) if filtered else all(c == ((4, Vs), rank * Vs) for c in calls)
    gathered = [None] * world
    dist.all_gather_object(gathered, (bool(ok), out))
    if rank == 0:
        ret.put(gathered)
    dist.destroy_process_group()
    ret.close()
    ret.join_thread()
    os._exit(0)


@pytest.mark.parametrize("filtered", [False, True], ids=["shard-pairs", "gathered-rows"])
@pytest.mark.parametrize("world", [2, 4])
def test_sharded_lm_head_constraints_equal_the_unsharded_tokens(world, filtered):
    """Vocabulary-sharded lm_head over gloo: the pair-merge path constrains each rank's shard at its vocabulary offset (a shard
    with no allowed id yields a -inf pair the merge never picks), the gather path the full rows; both return the unsharded
    model's tokens on every rank, with masks whose only allowed ids lie in one shard."""
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_tp_worker, args=(r, world, 29930 + world * 2 + int(filtered), ret, filtered))
             for r in range(world)]
    for p in procs:
        p.start()
    out = ret.get(timeout=240)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(ok for ok, _ in out), out
    assert all(t == out[0][1] for _, t in out)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_staged_form_of_the_restatement_equals_the_row_form(dtype):
    """constraints_oracle.constrain_staged (the GPU tests' reference at large batch) against constrain_row, on a shard."""
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import constraint_words
    from swiftllm_b200.worker.infer_state import ConstraintState
    rng = np.random.default_rng(4)
    V, off, n = 1000, 333, 12
    masks = _random_masks(rng, n, V)
    sp = [SamplingParams(logit_bias=None if i % 3 == 0 else {int(v): float(rng.uniform(-100, 100))
                                                             for v in rng.choice(V, 40, replace=False)}) for i in range(n)]
    cw = constraint_words(masks, sp, n, V)
    st = ConstraintState.from_staged(torch.from_numpy(cw.words), *cw[1:])
    logits = (torch.randn((n, V - off)) * 30).to(dtype)
    logits[:, 5] = float("nan"); logits[:, 6] = -0.0
    got = CO.constrain_staged(logits, st.mask_index.numpy(), st.masks.numpy(), st.bias_index.numpy(), st.bias_starts.numpy(),
                              st.bias_ids.numpy(), st.bias_values.numpy(), off)
    want = CO.constrain(logits, masks, [s.logit_bias for s in sp], off)
    assert torch.equal(_bits(got), _bits(want))
