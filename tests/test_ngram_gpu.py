"""GPU: the n-gram ban and DRY (the penalty kernel's n-gram instantiation, csrc/penalties.cu) against the numpy restatement
(tests/ngram_oracle.py) bit for bit, the token pages it writes, and the controls through LlamaModel (no repeated n-gram, eager
vs graph replay, chunked prefill, swaps, forks, seeded sampling, masks, raw log-probabilities, refusals)."""
import numpy as np
import pytest
import torch

import ngram_oracle as NO

pytestmark = pytest.mark.gpu

BS = 16
# (no_repeat_ngram_size, dry_multiplier, dry_base, dry_allowed_length, (r, f, p)) per row kind
KINDS = [(3, 0.0, 1.75, 2, (1.0, 0.0, 0.0)), (0, 0.8, 1.75, 2, (1.0, 0.0, 0.0)), (2, 1.5, 2.0, 3, (1.0, 0.0, 0.0)),
         (4, 0.5, 1.3, 1, (1.3, 0.4, 0.2)), (0, 0.0, 1.75, 2, (1.2, 0.0, 0.5)), (0, 0.0, 1.75, 2, (1.0, 0.0, 0.0)),
         (1, 0.0, 1.75, 2, (1.0, 0.0, 0.0)), (50, 3.0, 40.0, 1, (1.0, 0.0, 0.0))]


def _word(ids, out):
    return (np.asarray(ids, dtype=np.int64) | (np.asarray(out, dtype=np.int64) << 31)).astype(np.uint32).view(np.int32)


def _history(rng, kind: str, n: int, lo: int, v_full: int):
    if kind == "small":                                 # a few ids: matches of every length
        return rng.integers(lo, lo + 5, size=n)
    if kind == "periodic":
        per = rng.integers(lo, min(v_full, lo + 40), size=int(rng.integers(2, 9)))
        return np.resize(per, n)
    if kind == "repeat":                                # the adversarial one: every position matches 50 deep
        return np.full(n, lo + 3)
    return rng.integers(0, v_full, size=n)


def _case(B, V, dtype, vocab_offset=0, v_full=None, seed=0, hist_lens=(0, 1, 5, 60, 700, 3000), kinds=None,
          holes=True, n_new_max=40):
    """A launch with n-gram controls: per-row parameters of KINDS, histories of every kind (some split between the pages and a
    prefill's new tokens), unmapped positions and invalid block ids in some rows."""
    v_full = v_full or V
    rng = np.random.default_rng(seed)
    g = torch.Generator(device="cuda").manual_seed(seed)
    logits = (torch.randn((B, V), generator=g, device="cuda") * 3).to(dtype)
    n_pre = B // 3
    kinds = kinds or ["small", "periodic", "repeat", "random"]
    lo = vocab_offset + V // 3 if V > 40 else vocab_offset
    hist = [hist_lens[i % len(hist_lens)] for i in range(B)]
    n_new = [int(rng.integers(1, n_new_max)) if i < n_pre else 1 for i in range(B)]
    pos = [h + n for h, n in zip(hist, n_new)]
    nblk = [(p + BS - 1) // BS for p in pos]
    pool = rng.permutation(sum(nblk) + 7)
    seq_ids = rng.permutation(B + 3)[:B]
    bt = np.full((B + 3, max(nblk)), -1, dtype=np.int32)
    used = 0
    for i in range(B):
        bt[seq_ids[i], :nblk[i]] = pool[used:used + nblk[i]]
        used += nblk[i]
    tc = rng.integers(-2 ** 31, 2 ** 31, size=(len(pool), BS), dtype=np.int64).astype(np.int32)
    xs, outs, new_ids = [], [], []
    for i in range(B):
        ids = _history(rng, kinds[i % len(kinds)], pos[i], lo, v_full)
        out = rng.random(pos[i]) < 0.5
        q = np.arange(hist[i])
        tc[bt[seq_ids[i], q // BS], q % BS] = _word(ids[:hist[i]], out[:hist[i]])
        new_ids.append(ids[hist[i]:])
        x = [int(t) for t in ids]
        outs.append([bool(o) if j < hist[i] else i >= n_pre for j, o in enumerate(out)])
        xs.append(x)
    if holes:
        for i in range(B):
            if hist[i] >= 3 * BS and i % 3 == 1:         # an unmapped block and an invalid block id inside the history
                b1, b2 = 1, hist[i] // BS - 1
                bt[seq_ids[i], b1] = -1
                bt[seq_ids[i], b2] = len(pool) + 100
                for b in (b1, b2):
                    for q in range(b * BS, min((b + 1) * BS, pos[i])):
                        xs[i][q] = None
    params = []
    for i in range(B):
        n, mult, base, A, (r, f, p) = KINDS[(i * 5 + seed) % len(KINDS)]
        small = list(range(lo, lo + 5))
        br = [int(t) for t in rng.choice(small + [v_full + 3], size=int(rng.integers(0, 3)), replace=False)]
        params.append(dict(r=r, f=f, p=p, n=n, multiplier=mult, base=base, allowed=A, breakers=br))
    flat = np.concatenate(new_ids).astype(np.int32)
    last = np.cumsum(n_new) - 1
    dev = lambda a, dt=torch.int32: torch.as_tensor(np.asarray(a), dtype=dt, device="cuda")
    return dict(logits=logits, params=params, xs=xs, outs=outs, tc=tc, bt=bt, seq_ids=seq_ids, pos=pos, n_pre=n_pre,
                n_new=n_new, hist=hist, vocab_offset=vocab_offset,
                args=dict(pos=dev(pos), seq_ids=dev(seq_ids), input_ids=dev(flat), last=dev(last), p_lens=dev(n_new[:n_pre]),
                          bt=dev(bt)))


def _tensors(c, ngram=True):
    P = c["params"]
    f32 = lambda k: torch.tensor([p[k] for p in P], dtype=torch.float32, device="cuda")
    i32 = lambda k: torch.tensor([p[k] for p in P], dtype=torch.int32, device="cuda")
    pen = (f32("r"), f32("f"), f32("p"))
    if not ngram:
        return pen, {}
    br = torch.full((len(P), 16), -1, dtype=torch.int32)
    for i, p in enumerate(P):
        br[i, :len(p["breakers"])] = torch.tensor(p["breakers"], dtype=torch.int32)
    return pen, dict(no_repeat_ngram_size=i32("n"), dry_allowed_length=i32("allowed"), dry_multiplier=f32("multiplier"),
                     dry_base=f32("base"), dry_breakers=br.cuda())


def _run(c, ngram=True):
    from swiftllm_b200.worker.kernels.penalties import apply_penalties
    a = c["args"]
    lg = c["logits"].clone()
    tok = torch.as_tensor(c["tc"], device="cuda").clone()
    (r, f, p), kw = _tensors(c, ngram)
    apply_penalties(lg, r, f, p, a["pos"], a["seq_ids"], a["input_ids"], a["last"], a["p_lens"], c["n_pre"], a["bt"], tok,
                    vocab_offset=c["vocab_offset"], **kw)
    return lg, tok


def _want(c, i):
    p = c["params"][i]
    return NO.apply_row(c["logits"][i], c["xs"][i], c["vocab_offset"], p["r"], p["f"], p["p"], c["outs"][i], p["n"],
                        p["multiplier"], p["base"], p["allowed"], p["breakers"])


def _same_bits(a, b):
    a, b = a.cpu(), b.cpu()
    both_nan = torch.isnan(a.float()) & torch.isnan(b.float())
    return bool(((a.view(torch.int16) == b.view(torch.int16)) | both_nan).all())


def _active(p):
    return p["n"] > 0 or p["multiplier"] > 0 or (p["r"], p["f"], p["p"]) != (1.0, 0.0, 0.0)


def _check_pages(c, tok):
    """Exactly the step's tokens of the rows with some control at [pos - n_new, pos) where mapped, nothing else."""
    exp = c["tc"].copy()
    nb = exp.shape[0]
    for i, p in enumerate(c["params"]):
        if not _active(p):
            continue
        for q in range(c["hist"][i], c["pos"][i]):
            b = int(c["bt"][c["seq_ids"][i], q // BS])
            if 0 <= b < nb:
                exp[b, q % BS] = _word([c["xs"][i][q]], [c["outs"][i][q]])[0]
    assert np.array_equal(tok.cpu().numpy(), exp)


# V 128256 runs clusters of 8 (the n-gram slots need 8 CTAs there); at V 1000, B 1 / 3 / 17 / 64 / 257 run 8, 8, 4, 2 and 1
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V,offset,v_full", [(1000, 0, None), (128256, 0, None), (16032, 3 * 16032, 128256)],
                         ids=["1000", "128256", "shard16032"])
@pytest.mark.parametrize("B", [1, 3, 17, 64, 257])
def test_kernel_matches_the_restatement_bit_for_bit(B, V, offset, v_full, dtype):
    c = _case(B, V, dtype, offset, v_full, seed=B * 7 + V % 97)
    got, tok = _run(c)
    for i in range(B):
        assert _same_bits(got[i], _want(c, i)), (i, c["params"][i], c["hist"][i])
        if not _active(c["params"][i]):
            assert torch.equal(got[i].view(torch.int16), c["logits"][i].view(torch.int16))
    _check_pages(c, tok)
    again, tok2 = _run(c)
    assert torch.equal(again.view(torch.int16), got.view(torch.int16)) and torch.equal(tok, tok2)


def test_rows_without_ngram_controls_equal_the_plain_launch_and_write_the_same_pages():
    """Rows with penalties only (or nothing) give the plain instantiation's bits, and its pages."""
    c = _case(64, 128256, torch.bfloat16, seed=11)
    for p in c["params"]:
        p.update(n=0, multiplier=0.0)
    a, ta = _run(c, ngram=True)
    b, tb = _run(c, ngram=False)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)) and torch.equal(ta, tb)


def test_shards_write_what_the_whole_row_writes():
    """Every vocabulary shard of a row, launched at its vocab_offset, equals that slice of the whole row's launch."""
    c = _case(6, 1000, torch.bfloat16, seed=5, holes=False)
    whole, _ = _run(c)
    for off, n in ((0, 250), (250, 250), (500, 333), (833, 167)):
        s = dict(c, logits=c["logits"][:, off:off + n].contiguous(), vocab_offset=off)
        part, _ = _run(s)
        assert torch.equal(part.view(torch.int16), whole[:, off:off + n].view(torch.int16)), off


def test_largest_vocabulary_of_the_variant_and_the_one_past_it():
    """The n-gram slots are 8 bytes: the largest V that fits 8 slices runs against the restatement; one slice more is refused."""
    from swiftllm_b200 import _lib
    vmax = 8 * (200 * 1024 // 8)                      # 8 CTAs of 200 KiB slices of 8-byte slots, multiples of 4 entries
    c = _case(2, vmax, torch.bfloat16, seed=2, hist_lens=(200, 900))
    got, _ = _run(c)
    for i in range(2):
        assert _same_bits(got[i], _want(c, i))
    c2 = _case(1, vmax + 8, torch.bfloat16, seed=2, hist_lens=(10,))
    with pytest.raises(RuntimeError, match="shared memory"):
        _run(c2)


@pytest.mark.parametrize("kind", ["repeat", "periodic"])
def test_32k_token_repeated_histories(kind):
    """32 768-token histories where every position matches 50 deep (one repeated token) or periodically."""
    c = _case(3, 128256, torch.bfloat16, seed=9, hist_lens=(32768, 32700, 32760), kinds=[kind], holes=False)
    for p in c["params"]:
        p.update(n=3, multiplier=0.8, base=1.75, allowed=2)
    got, tok = _run(c)
    for i in range(3):
        assert _same_bits(got[i], _want(c, i)), i
    _check_pages(c, tok)


# ---------------------------------------------------------------- through LlamaModel
def _ngrams(seq, n):
    return [tuple(seq[i:i + n]) for i in range(len(seq) - n + 1)]


def _greedy(m, prompt, steps, sp, sid=0, swap_at=None):
    toks = m.forward([prompt], [sid], [], sampling_params_list=[sp])
    seq = list(prompt) + toks
    for s in range(steps):
        if swap_at == s:
            m.swap_out_seqs([sid]); m.swap_in_seqs([sid])
        toks = m.forward([[seq[-1]]], [sid], [len(seq)], sampling_params_list=[sp])
        seq += toks
    return seq


def test_no_repeat_ngram_over_200_steps_eager_graph_and_swapped():
    """A logit bias on three ids makes plain greedy decoding cycle through them; with no_repeat_ngram_size=3 the 200-step
    sequence, prompt included, has no repeated 3-gram, and eager, graph-replayed and swapped runs agree token for token."""
    from swiftllm_b200 import SamplingParams
    from test_sampling_gpu import _model, _weights
    w = _weights()
    eager, graph, swapped = _model(False, w=w), _model(True, w=w), _model(False, w=w)
    prompt = np.random.default_rng(4).permutation(1000)[:12].tolist()
    bias = {11: 60.0, 22: 60.0, 33: 60.0}
    plain = _greedy(eager, prompt, 60, SamplingParams(logit_bias=bias))
    eager.free_seqs_resources([0])
    assert len(set(_ngrams(plain, 3))) < len(_ngrams(plain, 3))
    sp = SamplingParams(no_repeat_ngram_size=3, logit_bias=bias)
    a = _greedy(eager, prompt, 200, sp)
    b = _greedy(graph, prompt, 200, sp)
    c = _greedy(swapped, prompt, 200, sp, swap_at=30)
    assert a == b == c
    grams = _ngrams(a, 3)
    assert len(set(grams)) == len(grams)
    assert {k[2:] for k in graph._graphs} == {(True, False, "penalties", False, "ngram", "constrained", 4)}


def test_dry_and_ban_with_penalties_match_the_restatement_every_step():
    """Each step's greedy token is the restatement applied to the step's raw logits (post_layer.last_logits) over the history,
    with chunked prefill equal to the whole prompt."""
    from swiftllm_b200 import SamplingParams
    from test_sampling_gpu import _model, _weights
    w = _weights()
    whole, chunked = _model(False, w=w), _model(False, w=w)
    whole.post_layer.keep_logits = chunked.post_layer.keep_logits = True
    rng = np.random.default_rng(6)
    prompt = np.resize(rng.integers(0, 1000, size=7), 70).tolist()
    sp = SamplingParams(repetition_penalty=1.1, frequency_penalty=0.2, no_repeat_ngram_size=5, dry_multiplier=0.8,
                        dry_allowed_length=2, dry_sequence_breakers=(prompt[3],))
    t1 = whole.forward([prompt], [0], [], sampling_params_list=[sp])
    chunked.forward([prompt[:30]], [0], [], prefill_prefix_lens_list=[0], sampling_params_list=[sp])
    t2 = chunked.forward([prompt[30:]], [0], [], prefill_prefix_lens_list=[30], sampling_params_list=[sp])
    x, outs = list(prompt), [False] * 70

    def want(m):
        row = NO.apply_row(m.post_layer.last_logits[0], x, 0, 1.1, 0.2, 0.0, outs, 5, 0.8, 1.75, 2, (prompt[3],))
        return int(torch.argmax(row.float()))
    assert t1[0] == want(whole) and t2[0] == want(chunked)
    bt, tc = chunked.gpu_block_manager.block_table.cpu(), chunked.token_cache.cpu()
    assert [int(tc[int(bt[0, q // 16]), q % 16]) for q in range(70)] == prompt
    toks = t1
    for _ in range(12):
        x.append(toks[0]); outs.append(True)
        toks = whole.forward([toks], [0], [len(x)], sampling_params_list=[sp])
        assert toks[0] == want(whole)


def test_a_fork_bans_its_parents_ngrams():
    """A fork of a 30-token prompt (two shared blocks and a copied tail) continued with the prompt's 6th token bans the 7th: the
    child's token is the restatement over the parent's history."""
    from swiftllm_b200 import SamplingParams
    from test_sampling_gpu import _model, _weights
    m = _model(False, w=_weights())
    m.post_layer.keep_logits = True
    sp = SamplingParams(no_repeat_ngram_size=2)
    rng = np.random.default_rng(8)
    prompt = rng.permutation(1000)[:30].tolist()
    m.forward([prompt], [0], [], sampling_params_list=[sp])
    m.fork_seqs([0], [5], [30])
    toks = m.forward([[prompt[5]]], [5], [31], sampling_params_list=[sp])
    want = NO.apply_row(m.post_layer.last_logits[0], prompt + [prompt[5]], n=2)
    assert NO.banned_ids(prompt + [prompt[5]], 2) == {prompt[6]}
    assert toks[0] != prompt[6] and toks[0] == int(torch.argmax(want.float()))


def test_seeded_sampled_rows_are_reproducible_and_masks_come_first_with_raw_logprobs():
    from swiftllm_b200 import SamplingParams, token_mask
    from test_sampling_gpu import _model, _weights
    w = _weights()
    runs = []
    for _ in range(2):
        m = _model(True, w=w)
        sp = [SamplingParams(0.9, seed=7, no_repeat_ngram_size=2, dry_multiplier=1.0),
              SamplingParams(0.0, dry_multiplier=2.0, dry_allowed_length=1)]
        seqs = [[1, 2, 3, 1, 2], [9, 8, 9, 8]]
        t = m.forward(seqs, [0, 1], [], sampling_params_list=sp)
        out = [t]
        lens = [5, 4]
        for _ in range(30):
            lens = [l + 1 for l in lens]
            t = m.forward([[x] for x in t], [0, 1], lens, sampling_params_list=sp)
            out.append(t)
        runs.append(out)
    assert runs[0] == runs[1]
    # masks first: a mask allowing only a banned id and one other id leaves the other one
    m = _model(False, w=w)
    m.post_layer.keep_logits = True
    sp = SamplingParams(no_repeat_ngram_size=2, logprobs=3)
    V = m.model_config.vocab_size
    r = m.forward_with_logprobs([[4, 5, 6, 4]], [0], [], sampling_params_list=[sp],
                                token_masks_list=[token_mask(V, [5, 11])])
    assert r[0].token == 11
    raw = torch.log_softmax(m.post_layer.last_logits[0].float(), dim=0)
    assert abs(r[0].logprob - float(raw[11])) < 1e-3


def test_speculative_and_ignore_kvcache_refuse():
    from swiftllm_b200 import SamplingParams
    from test_sampling_gpu import _model, _weights
    m = _model(False, w=_weights())
    for sp in (SamplingParams(no_repeat_ngram_size=3), SamplingParams(dry_multiplier=0.5)):
        with pytest.raises(ValueError, match="DRY"):
            m.forward_speculative([[1, 2]], [0], [0], sampling_params_list=[sp])
        with pytest.raises(ValueError, match="ignore_kvcache"):
            m.forward([[1, 2]], [0], [], ignore_kvcache=True, sampling_params_list=[sp])
    V = m.model_config.vocab_size
    with pytest.raises(ValueError, match="dry_sequence_breakers"):
        m.forward([[1, 2]], [0], [], sampling_params_list=[SamplingParams(dry_multiplier=0.5, dry_sequence_breakers=(V,))])
