"""CPU: the penalty semantics (tests/penalties_oracle.py) on hand-computed rows, SamplingParams validation, the unchanged staging
of lists without penalties, the C ABI's argument checks, and the penalties through the product's host path - token pages through
prefill, decode, chunked and mixed steps, swaps on every swap path, seq-id reuse, log-probabilities, and a vocabulary-sharded
lm_head over gloo - with a torch stand-in of the kernel that reads and writes the model's real token pages."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import penalties_oracle as PO
import sampling_oracle as SO
from test_logprobs_cpu import PATCH as LOGPROBS_PATCH


# ---------------------------------------------------------------- the restatement on hand-computed rows
def _row(vals, dtype=torch.float32):
    return torch.tensor(vals, dtype=torch.float32).to(dtype)


def test_each_penalty_alone_and_combined():
    row = _row([2.0, -1.0, 0.5, 3.0, -4.0])
    hist = [(0, False), (1, False), (2, True), (2, True), (3, True)]      # prompt 0, 1; outputs 2 x2, 3 x1; 4 unseen
    assert PO.penalize_row(row, 2.0, 0, 0, hist).tolist() == [1.0, -2.0, 0.25, 1.5, -4.0]
    assert PO.penalize_row(row, 1.0, 0.5, 0, hist).tolist() == [2.0, -1.0, -0.5, 2.5, -4.0]
    assert PO.penalize_row(row, 1.0, 0, 0.25, hist).tolist() == [2.0, -1.0, 0.25, 2.75, -4.0]
    # combined, in order: repetition, then t = f * c + p
    assert PO.penalize_row(row, 2.0, 0.5, 0.25, hist).tolist() == [1.0, -2.0, 0.25 - 1.25, 1.5 - 0.75, -4.0]
    assert PO.penalize_row(row, 1.0, 0, 0, hist).tolist() == row.tolist()                     # all off
    # negative penalties reward repeats; repetition < 1 raises positive logits and lowers negative ones
    assert PO.penalize_row(row, 0.5, -1.0, -0.5, hist).tolist() == [4.0, -0.5, 1.0 + 2.5, 6.0 + 1.5, -4.0]


def test_negative_logits_and_zero_under_repetition():
    row = _row([-3.0, 0.0, -0.0, 1e-3])
    out = PO.penalize_row(row, 1.5, 0, 0, [(0, False), (1, False), (2, False), (3, False)])
    assert out[0].item() == -4.5 and out[1].item() == 0.0 and str(out[2].item()) == "-0.0"
    assert out[3].item() == np.float32(np.float32(1e-3) / np.float32(1.5))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_unseen_nan_inf_and_negative_zero_keep_their_bits(dtype):
    row = _row([float("nan"), float("inf"), -float("inf"), -0.0, 1.0, 2.0], dtype)
    out = PO.penalize_row(row, 1.7, 1.1, 0.3, [(4, True), (5, False), (17, True), (-3, True)])
    assert torch.equal(out[:4].view(torch.int16), row[:4].view(torch.int16))
    assert out[4].item() != 1.0 and out[5].item() == (torch.tensor(2.0 / np.float32(1.7)).to(dtype)).item()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_one_rounding_to_the_storage_dtype(dtype):
    g = torch.Generator().manual_seed(0)
    row = (torch.randn(200, generator=g) * 4).to(dtype)
    hist = [(int(v), bool(v % 3)) for v in torch.randint(0, 200, (500,), generator=g)]
    out = PO.penalize_row(row, 1.3, 0.7, 0.2, hist)
    seen, cnt = PO.counts_of(hist, 0, 200)
    for v in range(200):
        l = np.float32(row[v].float().item())
        if not seen[v]:
            assert out[v].view(torch.int16) == row[v].view(torch.int16)
            continue
        l = np.float32(l / np.float32(1.3)) if l > 0 else np.float32(l * np.float32(1.3))
        t = np.float32(np.float32(0.7) * np.float32(cnt[v]))
        if cnt[v]:
            t = np.float32(t + np.float32(0.2))
        assert out[v].item() == torch.tensor(float(np.float32(l - t))).to(dtype).item()


def test_counts_above_65535_are_exact():
    row = _row([10.0, 10.0, 10.0])
    hist = [(1, True)] * 70001 + [(2, True)] * 65535
    out = PO.penalize_row(row, 1.0, 1.0 / 1024, 0.0, hist)
    assert out.tolist() == [10.0, np.float32(10.0 - 70001 / 1024), np.float32(10.0 - 65535 / 1024)]


def test_shard_offsets_and_out_of_range_ids():
    row = _row([1.0, 1.0, 1.0, 1.0])
    out = PO.penalize_row(row, 2.0, 0, 0, [(100, False), (103, True), (99, True), (104, True), (-1, True)], vocab_offset=100)
    assert out.tolist() == [0.5, 1.0, 1.0, 0.5]


# ---------------------------------------------------------------- validation and staging
@pytest.mark.parametrize("field,bad", [("repetition_penalty", 0.0), ("repetition_penalty", -1.0), ("repetition_penalty", float("inf")),
                                       ("repetition_penalty", float("nan")), ("repetition_penalty", True), ("repetition_penalty", "1"),
                                       ("frequency_penalty", 2.5), ("frequency_penalty", -2.01), ("frequency_penalty", float("nan")),
                                       ("frequency_penalty", None), ("presence_penalty", 3.0), ("presence_penalty", float("-inf")),
                                       ("presence_penalty", False)])
def test_bad_penalties_raise_value_error(field, bad):
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import sampling_words
    with pytest.raises(ValueError, match=field):
        sampling_words([SamplingParams(**{field: bad})], 1, np.random.default_rng(0))


def test_edge_values_are_valid():
    from swiftllm_b200 import SamplingParams
    for sp in (SamplingParams(repetition_penalty=1e-3, frequency_penalty=-2, presence_penalty=2),
               SamplingParams(repetition_penalty=40, frequency_penalty=2, presence_penalty=-2)):
        sp.validate()
        assert sp.has_penalties()
    assert not SamplingParams().has_penalties() and not SamplingParams(frequency_penalty=-0.0).has_penalties()


def _parent_words(params_list, rng):
    """The staging of the parent commit, restated: seeds [2B], temperature bits [B], top_k [B], top_p bits [B]; None if greedy."""
    seeds = np.array([int(rng.integers(0, 2 ** 63)) if sp.seed is None else int(sp.seed) for sp in params_list], dtype=np.uint64)
    if all(sp.temperature == 0 for sp in params_list):
        return None
    i32 = lambda a: a.astype(np.uint32).view(np.int32).tolist()
    temp = np.array([sp.temperature for sp in params_list], dtype=np.float32)
    top_p = np.array([sp.top_p for sp in params_list], dtype=np.float32)
    filtered = any(sp.temperature > 0 and (sp.top_k > 0 or sp.top_p < 1) for sp in params_list)
    return i32(seeds.view(np.uint32)) + i32(temp.view(np.uint32)) + [int(sp.top_k) for sp in params_list] + \
        i32(top_p.view(np.uint32)), filtered


def test_lists_without_penalties_stage_the_parent_words():
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import has_penalties, sampling_words
    lists = [[SamplingParams()] * 3, [SamplingParams(top_k=4, repetition_penalty=1.0)],
             [SamplingParams(0.7, seed=3), SamplingParams(1.1)], [SamplingParams(0.7, 5, 0.9, seed=9), SamplingParams(0.0)],
             [SamplingParams(0.5, top_p=0.8, frequency_penalty=0.0, presence_penalty=0.0)]]
    for sp in lists:
        assert sampling_words(sp, len(sp), np.random.default_rng(4)) == _parent_words(sp, np.random.default_rng(4))
        assert not has_penalties(sp)
    assert not has_penalties(None)


def test_penalised_lists_append_three_float_words_even_when_greedy():
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.sampling_params import sampling_words
    from swiftllm_b200.worker.infer_state import SamplingState
    sp = [SamplingParams(repetition_penalty=1.25), SamplingParams(0.0), SamplingParams(frequency_penalty=-0.5, presence_penalty=2)]
    words, filtered = sampling_words(sp, 3, np.random.default_rng(2))
    assert len(words) == 24 and not filtered
    assert words[:15] == _parent_words([SamplingParams(0.0)] * 2 + [SamplingParams(1.0)], np.random.default_rng(2))[0][:6] + \
        [0] * 3 + [0] * 3 + [np.float32(1).view(np.int32)] * 3
    st = SamplingState.from_staged(torch.tensor(words, dtype=torch.int32), torch.tensor([4, 5, 6], dtype=torch.int32), filtered, False)
    assert st.penalized and not st.sampled
    assert st.repetition_penalty.tolist() == [1.25, 1.0, 1.0]
    assert st.frequency_penalty.tolist() == [0.0, 0.0, -0.5] and st.presence_penalty.tolist() == [0.0, 0.0, 2.0]
    assert not SamplingState.from_staged(torch.tensor(words[:15], dtype=torch.int32), st.pos, False).penalized


def test_apply_penalties_rejects_invalid_arguments_before_launch():
    from swiftllm_b200 import _lib
    l = _lib.lib()
    names = (("logits", 1), ("rows", 2), ("V", 1000), ("stride", 1000), ("off", 0), ("r", 1), ("f", 1), ("p", 1), ("sid", 1),
             ("pos", 1), ("ids", 1), ("last", 1), ("plens", 1), ("npre", 1), ("bt", 1), ("bts", 8), ("bs", 16), ("tok", 1),
             ("nblk", 10), ("dtype", 1), ("stream", None))
    args = lambda **kw: [kw.get(n, d) for n, d in names]
    for kw, msg in (({"dtype": 7}, b"dtype"), ({"V": 0}, b"vocab_size"), ({"V": 409601, "stride": 409601}, b"shared memory"),
                    ({"stride": 999}, b"row_stride"), ({"rows": -1}, b"num_rows"), ({"rows": (1 << 20) + 1}, b"num_rows"),
                    ({"off": -1}, b"2^31"), ({"off": 2 ** 31 - 1000}, b"2^31"), ({"bs": 0}, b"block_size"),
                    ({"bs": 1 << 17}, b"block_size"), ({"bts": 0}, b"block_table_stride"),
                    ({"bts": 1 << 20, "bs": 1 << 12}, b"block_table_stride"), ({"nblk": -1}, b"num_blocks"),
                    ({"npre": 3}, b"num_prefill_rows"), ({"npre": -1}, b"num_prefill_rows"),
                    ({"logits": None}, b"null pointer"), ({"r": None}, b"null pointer"), ({"f": None}, b"null pointer"),
                    ({"p": None}, b"null pointer"), ({"sid": None}, b"null pointer"), ({"pos": None}, b"null pointer"),
                    ({"ids": None}, b"null pointer"), ({"last": None}, b"null pointer"), ({"plens": None}, b"null pointer"),
                    ({"bt": None}, b"null pointer"), ({"tok": None}, b"null pointer")):
        assert l.sllm_apply_penalties(*args(**kw)) != 0, kw
        assert msg in l.sllm_last_error(), (kw, l.sllm_last_error())
    assert l.sllm_apply_penalties(*args(V=409600, stride=409600, dtype=7)) != 0            # the largest vocabulary passes the size check
    assert b"dtype" in l.sllm_last_error()
    assert l.sllm_apply_penalties(*args(rows=0, npre=0, logits=None, r=None, tok=None)) == 0      # empty batch: nothing to launch


# ---------------------------------------------------------------- host path with a stand-in of the kernel over the real pages
PEN_CALLS = []


def _pen_stand_in(logits, rep, freq, pres, pos, seq_ids, input_ids, last, p_lens, n_pre, block_table, token_cache, vocab_offset=0):
    """csrc/penalties.cu on CPU tensors: the history from the token pages + the step's new tokens, the restatement, the pages
    written."""
    PEN_CALLS.append(logits.shape)
    bs = token_cache.shape[1]
    new_logits = logits.clone()
    writes = []
    for i in range(logits.shape[0]):
        r, f, p = float(rep[i]), float(freq[i]), float(pres[i])
        if r == 1 and f == 0 and p == 0:
            continue
        n_new = int(p_lens[i]) if i < n_pre else 1
        P, first, sid = int(pos[i]), int(last[i]) - n_new + 1, int(seq_ids[i])
        hist = []
        for q in range(P - n_new):
            w = int(token_cache[int(block_table[sid, q // bs]), q % bs]) & 0xffffffff
            hist.append((w & 0x7fffffff, bool(w >> 31)))
        new = [(int(input_ids[first + j]), i >= n_pre) for j in range(n_new)]
        new_logits[i] = PO.penalize_row(logits[i], r, f, p, hist + new, vocab_offset)
        writes += [(sid, P - n_new + j, t | (int(o) << 31)) for j, (t, o) in enumerate(new)]
    logits.copy_(new_logits)
    for sid, q, w in writes:
        token_cache[int(block_table[sid, q // bs]), q % bs] = np.int32(np.uint32(w))


PATCH = LOGPROBS_PATCH + [("swiftllm_b200.worker.layers.post_layer", "apply_penalties", _pen_stand_in)]


def _pen_params(sids):
    """Fixed parameters per sequence (a request keeps its SamplingParams from its first prefill chunk on); seq 4 has none."""
    from swiftllm_b200 import SamplingParams
    c = [SamplingParams(0.0, repetition_penalty=1.4), SamplingParams(0.8, seed=11, frequency_penalty=0.6, presence_penalty=0.3),
         SamplingParams(0.0, frequency_penalty=0.9, presence_penalty=-0.2, repetition_penalty=0.9),
         SamplingParams(1.1, top_k=9, seed=12, repetition_penalty=1.2, presence_penalty=1.0), SamplingParams(0.7, seed=13)]
    return [c[s % len(c)] for s in sids]


class _History:
    """The history each sequence should have, tracked from the test's own calls."""

    def __init__(self):
        self.h = {}

    def step(self, ids, sids, n_prefill, prefix=None):
        for i, (toks, sid) in enumerate(zip(ids, sids)):
            if i < n_prefill and (prefix is None or prefix[i] == 0):
                self.h[sid] = []
            self.h[sid] = self.h[sid] + [(t, i >= n_prefill) for t in toks]
        return [list(self.h[s]) for s in sids]


def _expected(m, sp_list, hists, seeds):
    raw = m.post_layer.last_logits
    pen = PO.penalize(raw, [(s.repetition_penalty, s.frequency_penalty, s.presence_penalty) for s in sp_list], hists)
    if all(s.temperature == 0 for s in sp_list):
        return torch.argmax(pen, dim=1).tolist()
    return [r.token for r in SO.sample_tokens(pen, [s.temperature for s in sp_list], [s.top_k for s in sp_list],
                                              [s.top_p for s in sp_list], seeds, [len(h) for h in hists])]


def _seeds(m):
    return m._last_sampling.seed.tolist()


def _check_pages(m, hist, sid):
    bs = m.engine_config.block_size
    bt = m.gpu_block_manager.block_table
    words = [int(m.token_cache[int(bt[sid, q // bs]), q % bs]) & 0xffffffff for q in range(len(hist))]
    assert words == [t | (int(o) << 31) for t, o in hist]


@pytest.mark.parametrize("swap", ["host-ids", "device-ids", "copy-stream"])
def test_penalised_host_path_on_cpu(swap):
    """prefill -> decodes -> chunked prefill -> mixed batch -> swap out / in -> decode: every token equals the restatement applied
    to the step's raw logits with the history the test tracks; the pages hold the history through every swap path."""
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import _product
    from test_sampling_cpu import _record_sampling
    import swiftllm_b200.swiftllm_c as C
    w = OracleWeights.random(__import__("test_host_path_cpu").CFG, dtype=torch.float16, seed=2, std=0.08)
    rng = np.random.default_rng(3)
    kw = dict(device_swap=swap == "device-ids", swap_on_copy_stream=swap == "copy-stream")
    with product_on_cpu(PATCH):
        m = _product(w, **kw)
        _record_sampling(m)
        H = _History()

        def step(ids, sids, lens, n_pre, prefix=None):
            sp = _pen_params(sids)
            hists = H.step(ids, sids, n_pre, prefix)
            kw2 = {} if prefix is None else dict(prefill_prefix_lens_list=prefix)
            t = m.forward(ids, sids, lens, sampling_params_list=sp, **kw2)
            assert t == _expected(m, sp, hists, _seeds(m))
            for s, h, p in zip(sids, hists, sp):
                if p.has_penalties():
                    _check_pages(m, h, s)
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
        t = step([p3[16:40]] + [[t[s]] for s in sids], [3] + sids, [lens[s] for s in sids], 1, prefix=[16])
        lens[3] = 40
        # swap seq 1 out, decode the others, swap it back in (its blocks move), decode all
        calls = []
        for name in ("swap_blocks", "swap_blocks_device"):
            orig = getattr(C, name)
            setattr(C, name, (lambda o: lambda *a: (calls.append(a[3].dtype), o(*a))[1])(orig))
        before = m.gpu_block_manager.block_table[1].clone()
        m.swap_out_seqs([1])
        rest = [0, 2, 3, 4]
        lens = {s: l + (s != 1) for s, l in lens.items()}
        t.update(step([[t[s]] for s in rest], rest, [lens[s] for s in rest], 0))
        step([rng.integers(0, 300, size=20).tolist()], [5], [], 1)                # takes seq 1's old block, writes its pages
        m.swap_in_seqs([1])
        assert calls == [m.dtype, torch.int32] * 2                                  # KV, then the token pages, each way
        assert before[0] != m.gpu_block_manager.block_table[1, 0]
        for _ in range(2):
            lens = {s: l + 1 for s, l in lens.items()}
            t = step([[t[s]] for s in sorted(lens)], sorted(lens), [lens[s] for s in sorted(lens)], 0)


def test_seq_id_reuse_after_free_and_unpenalised_steps_stage_and_launch_as_before():
    """A freed seq id's new prompt starts a fresh history; steps without penalties stage the parent's words, launch no penalty
    kernel and swap no token pages until a penalised step has run."""
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG, _product
    from test_sampling_cpu import _record_sampling
    from swiftllm_b200 import SamplingParams
    import swiftllm_b200.swiftllm_c as C
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=5, std=0.08)
    with product_on_cpu(PATCH):
        m = _product(w)
        _record_sampling(m)
        staged, calls = [], []
        orig = m._stage_metadata
        m._stage_metadata = lambda *parts: (staged.append([list(p) for p in parts]), orig(*parts))[1]
        C_orig = C.swap_blocks
        C.swap_blocks = lambda *a: (calls.append(a[3].dtype), C_orig(*a))[1]
        PEN_CALLS.clear()
        plain = [None, [SamplingParams()] * 2, [SamplingParams(0.9, seed=4), SamplingParams(0.0, logprobs=2)]]
        for sp in plain:
            m.forward([[1, 2, 3], [4, 5]], [0, 1], [], sampling_params_list=sp)
            m.free_seqs_resources([0, 1])
        assert [len(s) for s in staged] == [8, 8, 9]
        rng = np.random.default_rng(0)                       # EngineConfig.sampling_seed: two seeds drawn by the greedy list
        rng.integers(0, 2 ** 63); rng.integers(0, 2 ** 63)
        assert staged[2][0] == _parent_words(plain[2], rng)[0]
        assert PEN_CALLS == [] and not m._penalties_used
        m.forward([[1, 2, 3]], [0], [])
        m.swap_out_seqs([0]); m.swap_in_seqs([0])
        assert calls == [m.dtype, m.dtype]                                           # KV only
        m.free_seqs_resources([0])
        H = _History()
        sp = [SamplingParams(frequency_penalty=1.5, presence_penalty=0.5)]
        for prompt in ([7, 7, 9, 7], [9, 8]):                                        # seq 0 twice: the second prompt starts afresh
            t = m.forward([prompt], [0], [], sampling_params_list=sp)
            assert t == _expected(m, sp, H.step([prompt], [0], 1), None)
            n = len(prompt)
            for _ in range(3):
                n += 1
                hist = H.step([t], [0], 0)
                t = m.forward([t], [0], [n], sampling_params_list=sp)
                assert t == _expected(m, sp, hist, None)
            m.free_seqs_resources([0])
        assert len(PEN_CALLS) == 8 and m._penalties_used


def test_logprobs_stay_raw_next_to_penalised_tokens():
    import logprobs_oracle as LO
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG, _product
    from test_sampling_cpu import _record_sampling
    from swiftllm_b200 import SamplingParams
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=6, std=0.08)
    with product_on_cpu(PATCH):
        a, b = _product(w), _product(w)
        for m in (a, b):
            _record_sampling(m)
        H = _History()
        sp = [SamplingParams(0.0, logprobs=3, repetition_penalty=3.0, frequency_penalty=2.0),
              SamplingParams(0.9, seed=3, logprobs=0, presence_penalty=1.0), SamplingParams(0.0, logprobs=2)]
        ids, sids, lens = [[5, 6, 5, 7], [9, 9], [1, 2, 3]], [0, 1, 2], []
        moved = 0
        for s in range(5):
            hists = H.step(ids, sids, 3 if s == 0 else 0)
            t = a.forward(ids, sids, lens, sampling_params_list=sp)
            res = b.forward_with_logprobs(ids, sids, lens, sampling_params_list=sp)
            assert [r.token for r in res] == t == _expected(b, sp, hists, _seeds(b))
            raw = b.post_layer.last_logits
            tl, ids_top, tlp = LO.token_logprobs(raw, t, 3)
            for i, r in enumerate(res):
                assert r.logprob == float(tl[i])
                assert r.top == [(int(x), float(y)) for x, y in zip(ids_top[i][:sp[i].logprobs], tlp[i][:sp[i].logprobs])]
            moved += res[0].top[0][0] != res[0].token
            lens = [len(h) + 1 for h in hists]
            ids = [[x] for x in t]
        assert moved > 0                          # the penalties moved the greedy token off the raw argmax at least once


def test_penalties_with_ignore_kvcache_raise_value_error():
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG, _product
    from swiftllm_b200 import SamplingParams
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=2, std=0.08)
    with product_on_cpu(PATCH):
        m = _product(w)
        with pytest.raises(ValueError, match="ignore_kvcache"):
            m.forward([[1, 2]], [0], [], ignore_kvcache=True, sampling_params_list=[SamplingParams(repetition_penalty=1.1)])
        m.forward([[1, 2]], [0], [], ignore_kvcache=True, sampling_params_list=[SamplingParams(0.5, seed=1)])


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
        shapes = []
        import swiftllm_b200.worker.layers.post_layer as PL
        PL.apply_penalties = lambda lg, *a, **kw: (shapes.append(lg.shape[1]), _pen_stand_in(lg, *a, **kw))[1]
        rng = np.random.default_rng(2)
        ids = [rng.integers(0, 96, size=n).tolist() for n in (21, 3, 9)]
        sids, dec, lens = [4, 1, 2], [], [21, 3, 9]
        for step in range(4):
            sp = [swiftllm_b200.SamplingParams(t, top_k=(5 if filtered and i == 1 else 0), seed=30 + i, repetition_penalty=1.5,
                                               frequency_penalty=0.8 * i, presence_penalty=0.4)
                  for i, t in enumerate([0.9, 1.1, 0.0])]
            got = sharded.forward(ids, sids, dec, sampling_params_list=sp)
            ref = full.forward(ids, sids, dec, sampling_params_list=sp)
            ok &= got == ref
            ok &= torch.equal(sharded.post_layer.last_logits, full.post_layer.last_logits)
            bs = 16
            for s in sids:                                          # every rank records the same pages as the unsharded model
                for mm in (sharded, full):
                    n = lens[sids.index(s)]
                    bt = mm.gpu_block_manager.block_table
                    mm._pages = [int(mm.token_cache[int(bt[s, q // bs]), q % bs]) for q in range(n)]
                ok &= sharded._pages == full._pages
            out.append(got)
            lens = [l + 1 for l in lens]
            ids, dec = [[x] for x in got], lens
        Vs = cfg["vocab_size"] // world
        ok &= set(shapes[0::2]) == {cfg["vocab_size"] if filtered else Vs} and set(shapes[1::2]) == {cfg["vocab_size"]}
    gathered = [None] * world
    dist.all_gather_object(gathered, (bool(ok), out))
    if rank == 0:
        ret.put(gathered)
    dist.destroy_process_group()
    ret.close()
    ret.join_thread()
    os._exit(0)


@pytest.mark.parametrize("filtered", [False, True], ids=["shard-pairs", "gathered-rows"])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_lm_head_penalties_equal_the_unsharded_tokens(world, filtered):
    """Vocabulary-sharded lm_head over gloo: the pair-merge path penalises each rank's shard with its vocabulary offset, the
    gather path the gathered full rows; both return the unsharded model's tokens on every rank and record identical pages."""
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_tp_worker, args=(r, world, 29890 + world * 2 + int(filtered), ret, filtered))
             for r in range(world)]
    for p in procs:
        p.start()
    out = ret.get(timeout=240)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(ok for ok, _ in out), out
    assert all(t == out[0][1] for _, t in out)


def test_steps_choose_tokens_with_the_sampling_kernel_unless_every_penalised_row_is_greedy():
    """What the post layer is handed on eager steps (forward and forward_with_logprobs, over random parameter lists): no sampling
    state for an all-greedy list without penalties, the argmax of penalised logits (sampled False) only when some row has penalties
    and every temperature is 0, and the sampling kernel (sampled True) on every other list."""
    from cpu_shim import product_on_cpu
    from oracle.model import OracleWeights
    from test_host_path_cpu import CFG, _product
    from test_sampling_cpu import _record_sampling
    from swiftllm_b200 import SamplingParams
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=7, std=0.08)
    rng = np.random.default_rng(11)
    with product_on_cpu(PATCH):
        m = _product(w)
        _record_sampling(m)
        seen = set()
        for k in range(24):
            sp = [SamplingParams(float(rng.choice([0.0, 0.0, 0.7])), logprobs=int(rng.integers(0, 3)) if rng.random() < 0.5 else None,
                                 seed=int(rng.integers(0, 100)),
                                 repetition_penalty=1.3 if rng.random() < 0.3 else 1.0) for _ in range(2)]
            call = m.forward_with_logprobs if k % 2 else m.forward
            call([[1, 2, 3], [4, 5]], [0, 1], [], sampling_params_list=sp)
            st = m._last_sampling
            greedy, penalised = all(s.temperature == 0 for s in sp), any(s.has_penalties() for s in sp)
            if greedy and not penalised:
                assert st is None
            else:
                assert st.sampled == (not greedy) and st.penalized == penalised
            seen.add((greedy, penalised))
            m.free_seqs_resources([0, 1])
        assert seen == {(False, False), (False, True), (True, False), (True, True)}
