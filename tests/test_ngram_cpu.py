"""CPU: the n-gram controls' restatement (tests/ngram_oracle.py) against literal transcriptions of Hugging Face's n-gram ban and
text-generation-webui's DRY loop, hand-made rows, SamplingParams validation, the staging of lists with and without the new
fields, the C ABI's argument checks, and the graph path's keys."""
import numpy as np
import pytest
import torch

import ngram_oracle as NO


def _histories():
    rng = np.random.default_rng(0)
    out = []
    for t in range(400):
        L, k = int(rng.integers(1, 160)), int(rng.integers(1, 7))
        out.append(rng.integers(0, k, size=L).tolist())                               # random over a small vocabulary
    out += [[7] * L for L in (1, 2, 3, 49, 50, 51, 52, 120)]                            # one repeated token
    out += [np.resize(rng.integers(0, 9, size=p), L).tolist() for p in (2, 3, 5) for L in (10, 60, 130)]   # periodic
    for m in (48, 49, 50, 51, 53):                                                      # a match of length m ending the sequence
        body = rng.permutation(200)[:m].tolist()
        out.append([500] + body + [501, 502] + body)
    return out


def test_ban_is_hugging_faces_no_repeat_ngram():
    for x in _histories():
        for n in (1, 2, 3, 4, 7, 50):
            assert NO.banned_ids(x, n) == NO.hf_banned_tokens(x, n), (x, n)


def test_ban_edges():
    assert NO.banned_ids([1, 2, 3], 1) == {1, 2, 3}                    # n = 1: every id in the history
    assert NO.banned_ids([1, 2], 4) == set() and NO.banned_ids([1, 1, 1], 4) == set()    # shorter than n: nothing
    assert NO.banned_ids([1, 2, 3, 1, 2], 3) == {3}
    assert NO.banned_ids([1, None, 3, 1, None], 3) == set()          # unmapped positions match nothing, not even each other
    assert NO.banned_ids([1, 2, None, 1, 2], 3) == set()


@pytest.mark.parametrize("allowed", [1, 2, 3, 5])
def test_dry_is_text_generation_webuis_loop(allowed):
    rng = np.random.default_rng(allowed)
    for x in _histories():
        br = tuple(int(b) for b in rng.choice(8, size=int(rng.integers(0, 3)), replace=False))
        for mult, base in ((0.8, 1.75), (2.0, 1.1), (0.5, 3.0)):
            got = NO.dry_penalties(x, mult, base, allowed, br)
            want = NO.webui_dry(x, mult, base, allowed, br)
            assert set(got) == set(want), (x, br)
            for v in got:
                assert abs(float(got[v]) - want[v]) <= 2e-6 * want[v] * (1 + abs(np.log(base)) * 50), (v, got[v], want[v])


def test_dry_edges():
    x = [1, 2, 3, 4, 1, 2, 3]
    assert set(NO.dry_penalties(x, 1.0, 2.0, 2, ())) == {4}             # "1 2 3" repeats: 4 would extend a 3-token repeat
    assert NO.dry_penalties(x, 1.0, 2.0, 2, ())[4] == np.float32(2.0)   # multiplier * base^(3 - 2)
    assert NO.dry_penalties(x, 1.0, 2.0, 2, (3,)) == {}                 # the last token is a breaker: no penalty
    assert NO.dry_penalties(x, 1.0, 2.0, 2, (1,)) == {4: np.float32(1.0)}   # an inner breaker cuts the repeat at 2
    assert NO.dry_penalties(x, 1.0, 2.0, 2, (4,)) == {}                 # a breaker is never penalised
    assert NO.dry_penalties(x, 1.0, 2.0, 4, ()) == {}                   # shorter than allowed_length
    # matches are capped at 50: a 51-token repeat counts as 50, like the reference
    body = list(range(100, 151))
    x = [9] + body + [8] + body
    assert NO.match_lengths(x)[8] == 50 and NO.webui_dry(x, 1.0, 1.0, 50, ()) == {8: 1.0}
    # an overflowing q is inf, so the logit becomes -inf
    row = NO.apply_row(torch.zeros(200, dtype=torch.bfloat16), x, multiplier=1.0, base=1e30, allowed=1)
    assert row[8].item() == float("-inf")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_order_and_untouched_entries(dtype):
    row = torch.tensor([1.0, 2.0, -3.0, 0.5, float("nan"), -0.0], dtype=torch.float32).to(dtype)
    x = [0, 1, 2, 0, 1]
    # repetition first, then DRY: id 2 would extend "0 1" (D = 2, A = 1): q = 0.5 * 2 = 1.0
    out = NO.apply_row(row, x, r=2.0, multiplier=0.5, base=2.0, allowed=1)
    assert out.float().tolist()[:3] == [0.5, 1.0, -7.0]
    assert torch.equal(out[3:].view(torch.int16)[[0, 2]], row[3:].view(torch.int16)[[0, 2]])   # untouched entries keep bits
    out = NO.apply_row(row, x, r=2.0, n=3, multiplier=0.5, base=2.0, allowed=1)
    assert out[2].item() == float("-inf") and out[0].item() == 0.5
    # ids outside the shard are absent; a shard gives the same values as the whole row
    whole = NO.apply_row(row, x, n=2, multiplier=0.7, allowed=1)
    assert torch.equal(NO.apply_row(row[2:], x, vocab_offset=2, n=2, multiplier=0.7, allowed=1).view(torch.int16),
                       whole[2:].view(torch.int16))


# ---------------------------------------------------------------- SamplingParams
@pytest.mark.parametrize("field,bad", [("no_repeat_ngram_size", -1), ("no_repeat_ngram_size", 51), ("no_repeat_ngram_size", 2.0),
                                       ("no_repeat_ngram_size", True), ("dry_multiplier", -0.1), ("dry_multiplier", float("inf")),
                                       ("dry_multiplier", float("nan")), ("dry_multiplier", "1"), ("dry_base", 0.99),
                                       ("dry_base", float("inf")), ("dry_base", None), ("dry_allowed_length", 0),
                                       ("dry_allowed_length", 51), ("dry_allowed_length", 1.5),
                                       ("dry_sequence_breakers", (1, 1)), ("dry_sequence_breakers", (-1,)),
                                       ("dry_sequence_breakers", tuple(range(17))), ("dry_sequence_breakers", (True,)),
                                       ("dry_sequence_breakers", "ab"), ("dry_sequence_breakers", (2 ** 31,))])
def test_bad_ngram_parameters_raise_value_error(field, bad):
    from swiftllm_b200 import SamplingParams
    with pytest.raises(ValueError, match=field):
        SamplingParams(**{field: bad}).validate()


def test_good_ngram_parameters_and_defaults():
    from swiftllm_b200 import SamplingParams
    for sp in (SamplingParams(no_repeat_ngram_size=50, dry_multiplier=0.0, dry_base=1.0, dry_allowed_length=50),
               SamplingParams(no_repeat_ngram_size=1, dry_multiplier=1e6, dry_base=1e30, dry_allowed_length=1,
                              dry_sequence_breakers=tuple(range(16))),
               SamplingParams(dry_multiplier=0.8, dry_sequence_breakers=[np.int64(5), 198])):
        sp.validate()
        assert sp.has_ngram_controls()
    d = SamplingParams()
    assert (d.no_repeat_ngram_size, d.dry_multiplier, d.dry_base, d.dry_allowed_length, d.dry_sequence_breakers) == \
        (0, 0.0, 1.75, 2, ())
    assert not d.has_ngram_controls() and not SamplingParams(dry_base=3.0, dry_allowed_length=7).has_ngram_controls()


def _parent_words(params_list, rng):
    """sampling_words of the parent commit, transcribed: the staging of lists without the new fields must not change."""
    seeds = np.array([int(rng.integers(0, 2 ** 63)) if sp.seed is None else int(sp.seed) for sp in params_list], dtype=np.uint64)
    penalized = any(sp.has_penalties() for sp in params_list)
    if not penalized and all(sp.temperature == 0 for sp in params_list):
        return None
    i32 = lambda w: w.astype(np.uint32).view(np.int32).tolist()    # noqa: E731
    temp = np.array([sp.temperature for sp in params_list], dtype=np.float32)
    top_p = np.array([sp.top_p for sp in params_list], dtype=np.float32)
    words = i32(seeds.view(np.uint32)) + i32(temp.view(np.uint32)) + [int(sp.top_k) for sp in params_list] + \
        i32(top_p.view(np.uint32))
    if penalized:
        for name in ("repetition_penalty", "frequency_penalty", "presence_penalty"):
            words += i32(np.array([getattr(sp, name) for sp in params_list], dtype=np.float32).view(np.uint32))
    return words, any(sp.temperature > 0 and (sp.top_k > 0 or sp.top_p < 1) for sp in params_list)


def test_lists_without_ngram_controls_stage_the_parent_words():
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import has_ngram_controls, sampling_words
    lists = [[SamplingParams()] * 3, [SamplingParams(0.7, top_k=5, seed=3)], [SamplingParams(repetition_penalty=1.2)] * 2,
             [SamplingParams(0.5, top_p=0.8, frequency_penalty=0.3, dry_base=2.0, dry_allowed_length=4,
                             dry_sequence_breakers=(1, 2))],
             [SamplingParams(seed=9, no_repeat_ngram_size=0, dry_multiplier=0.0), SamplingParams(0.9)]]
    for sp in lists:
        assert not has_ngram_controls(sp)
        assert sampling_words(sp, len(sp), np.random.default_rng(4)) == _parent_words(sp, np.random.default_rng(4))


def test_ngram_layout_and_state_views():
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import sampling_words
    from swiftllm_b200.worker.infer_state import SamplingState
    sp = [SamplingParams(no_repeat_ngram_size=3), SamplingParams(0.8, seed=5, repetition_penalty=1.3),
          SamplingParams(dry_multiplier=0.8, dry_base=2.5, dry_allowed_length=4, dry_sequence_breakers=(198, 25, 7))]
    words, filtered = sampling_words(sp, 3, np.random.default_rng(0))
    B = 3
    assert len(words) == 28 * B and not filtered
    assert words[:8 * B] == _parent_words(sp, np.random.default_rng(0))[0]        # the parent's words, then the new ones
    assert words[8 * B:10 * B] == [3, 0, 0] + [2, 2, 4]
    assert np.array(words[10 * B:12 * B], dtype=np.int32).view(np.float32).tolist() == [0.0, 0.0, 0.800000011920929, 1.75, 1.75, 2.5]
    assert words[12 * B:] == [-1] * 16 + [-1] * 16 + [198, 25, 7] + [-1] * 13
    st = SamplingState.from_staged(torch.tensor(words, dtype=torch.int32), torch.tensor([4, 5, 6], dtype=torch.int32), False)
    assert st.penalized and st.ngram
    assert st.repetition_penalty.tolist() == [1.0, pytest.approx(1.3), 1.0]
    assert st.no_repeat_ngram_size.tolist() == [3, 0, 0] and st.dry_allowed_length.tolist() == [2, 2, 4]
    assert st.dry_breakers.shape == (3, 16) and st.dry_breakers[2, :3].tolist() == [198, 25, 7]
    kw = st.ngram_kwargs()
    assert set(kw) == {"no_repeat_ngram_size", "dry_allowed_length", "dry_multiplier", "dry_base", "dry_breakers"}
    plain = SamplingState.from_staged(torch.tensor(words[:8 * B], dtype=torch.int32), st.pos, False)
    assert plain.penalized and not plain.ngram and plain.ngram_kwargs() == {}


def test_breaker_ids_are_checked_against_the_vocabulary():
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import check_breaker_ids
    check_breaker_ids([SamplingParams(dry_multiplier=1.0, dry_sequence_breakers=(0, 299))], 300)
    with pytest.raises(ValueError, match="dry_sequence_breakers has token id 300"):
        check_breaker_ids([SamplingParams(), SamplingParams(dry_multiplier=1.0, dry_sequence_breakers=(5, 300))], 300)


def test_apply_penalties_ngram_rejects_invalid_arguments_before_launch():
    from swiftllm_b200 import _lib
    l = _lib.lib()
    names = (("logits", 1), ("rows", 2), ("V", 1000), ("stride", 1000), ("off", 0), ("r", 1), ("f", 1), ("p", 1), ("sid", 1),
             ("pos", 1), ("ids", 1), ("last", 1), ("plens", 1), ("npre", 1), ("bt", 1), ("bts", 8), ("bs", 16), ("tok", 1),
             ("nblk", 10), ("n", 1), ("A", 1), ("mult", 1), ("base", 1), ("brk", 1), ("dtype", 1), ("stream", None))
    args = lambda **kw: [kw.get(n, d) for n, d in names]      # noqa: E731
    vmax = 8 * (200 * 1024 // 8)
    for kw, msg in (({"dtype": 7}, b"dtype"), ({"V": 0}, b"vocab_size"), ({"V": vmax + 8, "stride": vmax + 8}, b"shared memory"),
                    ({"stride": 999}, b"row_stride"), ({"rows": -1}, b"num_rows"), ({"off": -1}, b"2^31"),
                    ({"bs": 0}, b"block_size"), ({"nblk": -1}, b"num_blocks"), ({"npre": 3}, b"num_prefill_rows"),
                    ({"logits": None}, b"null pointer"), ({"tok": None}, b"null pointer"), ({"n": None}, b"null pointer"),
                    ({"A": None}, b"null pointer"), ({"mult": None}, b"null pointer"), ({"base": None}, b"null pointer"),
                    ({"brk": None}, b"null pointer")):
        assert l.sllm_apply_penalties_ngram(*args(**kw)) != 0, kw
        assert msg in l.sllm_last_error() and b"apply_penalties_ngram" in l.sllm_last_error(), (kw, l.sllm_last_error())
    assert l.sllm_apply_penalties_ngram(*args(V=vmax, stride=vmax, dtype=7)) != 0     # the largest vocabulary passes the size check
    assert b"dtype" in l.sllm_last_error()
    assert l.sllm_apply_penalties(*args(V=vmax + 8, stride=vmax + 8, dtype=7)[:19], 7, None) != 0   # 4-byte slots: still fits
    assert b"dtype" in l.sllm_last_error()


# ---------------------------------------------------------------- the host path: refusals, graph keys
def test_graph_keys_and_meta_without_and_with_ngram_controls():
    """Steps without n-gram controls keep their graph keys and meta lengths; a step with them replays its own graph, keyed by
    one more tag, with 28 * B meta words of parameters."""
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

        def fake_capture(B, bucket, filtered=None, top_n=None, penalized=False, sampled=True, con=None, ngram=False):
            caps.append((B, filtered, penalized, sampled, ngram))
            nw = 0 if filtered is None else (28 if ngram else 8 if penalized else 5) * B
            g = type("G", (), {"replay": lambda self: None})()
            return dict(graph=g, meta=torch.zeros((nw + 3 * B,), dtype=torch.int32), tokens=torch.zeros((B,), dtype=torch.int64),
                        logprobs=None)
        m._capture_decode_graph = fake_capture
        m._stage_metadata = lambda *parts, **kw: (staged.append([len(p) for p in parts]), orig(*parts, **kw))[1]
        m.forward([[1, 2, 3], [4, 5]], [0, 1], [])
        m.forward([[1], [2]], [0, 1], [4, 3])
        m.forward([[1], [2]], [0, 1], [5, 4], sampling_params_list=[SamplingParams(repetition_penalty=1.2)] * 2)
        m.forward([[1], [2]], [0, 1], [6, 5], sampling_params_list=[SamplingParams(dry_base=3.0)] * 2)    # DRY off: plain
        m.forward([[1], [2]], [0, 1], [7, 6], sampling_params_list=[SamplingParams(no_repeat_ngram_size=3), SamplingParams()])
        m.forward([[1], [2]], [0, 1], [8, 7], sampling_params_list=[SamplingParams(0.5, seed=1, dry_multiplier=0.8)] * 2)
        assert set(m._graphs) == {(2, 1024), (2, 1024, True, False, "penalties", False),
                                  (2, 1024, True, False, "penalties", False, "ngram"), (2, 1024, True, False, "penalties", True, "ngram")}
        assert staged[1:] == [[2, 2, 2], [16, 2, 2, 2], [2, 2, 2], [56, 2, 2, 2], [56, 2, 2, 2]]
        assert [c[-1] for c in caps] == [False, False, True, True]
        assert m._penalties_used


def test_refusals():
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from swiftllm_b200 import SamplingParams
    from test_constraints_cpu import PATCH
    from test_host_path_cpu import CFG, _product
    from test_speculative_cpu import SPEC
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=5, std=0.08)
    with product_on_cpu(PATCH + SPEC):
        m = _product(w)
        for sp in (SamplingParams(no_repeat_ngram_size=2), SamplingParams(dry_multiplier=0.5)):
            with pytest.raises(ValueError, match="DRY"):
                m.forward_speculative([[1, 2]], [0], [0], sampling_params_list=[sp])
            with pytest.raises(ValueError, match="ignore_kvcache"):
                m.forward([[1, 2]], [0], [], ignore_kvcache=True, sampling_params_list=[sp])
        with pytest.raises(ValueError, match="outside"):
            m.forward([[1, 2]], [0], [], sampling_params_list=[SamplingParams(dry_multiplier=0.5, dry_sequence_breakers=(300,))])
        assert m.gpu_block_manager.num_free_blocks == m.gpu_block_manager.num_blocks and not m._penalties_used
