"""GPU: the constraint kernel (csrc/constraints.cu) against the numpy restatement (tests/constraints_oracle.py) bit for bit, the
sampling kernel on heavily masked rows against tests/sampling_oracle.py, and constrained decoding through LlamaModel (forced tokens,
eager vs graph replay with changing masks, a row alone vs in a batch, penalties and log-probabilities together, speculative
verification, prompt log-probabilities)."""
import numpy as np
import pytest
import torch

import constraints_oracle as CO
import sampling_oracle as SO

pytestmark = pytest.mark.gpu

DENSITIES = ["one", 0.01, 0.5, "all", None]          # None: an unconstrained row inside the constrained batch
BIAS_COUNTS = [0, 1, 300, 1024]


def _case(B, V, dtype, vocab_offset=0, v_full=None, seed=0):
    """Logits of one shard [B, V] and a staged constraint region over the global vocabulary v_full: rows cycle through the mask
    densities and bias counts."""
    from swiftllm_b200 import SamplingParams, token_mask
    from swiftllm_b200.sampling_params import constraint_words
    from swiftllm_b200.worker.infer_state import ConstraintState
    v_full = v_full or V
    rng = np.random.default_rng(seed)
    g = torch.Generator(device="cuda").manual_seed(seed)
    logits = (torch.randn((B, V), generator=g, device="cuda") * 4).to(dtype)
    logits[:, 3] = float("nan"); logits[:, 4] = float("inf"); logits[:, 5] = -float("inf"); logits[:, 6] = -0.0
    masks, sp = [], []
    for i in range(B):
        d = DENSITIES[i % len(DENSITIES)]
        if d is None:
            masks.append(None)
        elif d == "one":
            masks.append(token_mask(v_full, [vocab_offset + int(rng.integers(0, V))]))
        elif d == "all":
            masks.append(~token_mask(v_full, []))
        else:
            ids = np.flatnonzero(rng.random(v_full) < d)
            masks.append(token_mask(v_full, ids if ids.size else [0]))
        n = min(v_full, BIAS_COUNTS[(i // len(DENSITIES)) % len(BIAS_COUNTS)]) if d is not None or i % 2 else 0
        ids = rng.choice(v_full, n, replace=False)
        if n:
            ids[:2] = [vocab_offset + 3, vocab_offset + 5][:n]            # a bias on NaN / -inf entries
        sp.append(SamplingParams(logit_bias={int(v): float(b) for v, b in zip(ids, rng.uniform(-100, 100, n))} or None))
    cw = constraint_words(masks, sp, B, v_full)
    st = ConstraintState.from_staged(torch.from_numpy(cw.words), *cw[1:])
    return logits, st, masks, sp


def _run(logits, st, vocab_offset=0):
    from swiftllm_b200.worker.kernels.constraints import constrain_logits
    out = logits.clone()
    d = {k: getattr(st, k).cuda() for k in ("mask_index", "masks", "bias_index", "bias_starts", "bias_ids", "bias_values")}
    constrain_logits(out, d["mask_index"], d["masks"], d["bias_index"], d["bias_starts"], d["bias_ids"], d["bias_values"],
                     vocab_offset=vocab_offset)
    return out


def _want(logits, st, vocab_offset=0):
    return CO.constrain_staged(logits.cpu(), st.mask_index.numpy(), st.masks.numpy(), st.bias_index.numpy(),
                               st.bias_starts.numpy(), st.bias_ids.numpy(), st.bias_values.numpy(), vocab_offset)


def _bits(t):
    return t.view(torch.int16)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V,offset,v_full", [(128256, 0, None), (32001, 0, None), (1003, 0, None), (5001, 1003, 128256),
                                             (64128, 64128, 128256)],
                         ids=["V128256", "V32001", "V1003", "shard-at-1003", "half-at-64128"])
@pytest.mark.parametrize("B", [1, 7, 64, 1024])
def test_kernel_matches_the_restatement_bit_for_bit(B, V, offset, v_full, dtype):
    if B == 1024 and V == 32001:
        pytest.skip("B = 1024 runs at the other vocabularies")
    logits, st, _, _ = _case(B, V, dtype, offset, v_full, seed=B + V)
    got = _run(logits, st, offset)
    want = _want(logits, st, offset)
    diff = (_bits(got.cpu()) != _bits(want)).nonzero()
    assert diff.shape[0] == 0, (diff[:5].tolist(), [(got[r, c].item(), want[r, c].item()) for r, c in diff[:5].tolist()])
    free = (st.mask_index < 0) & (st.bias_index < 0)
    assert torch.equal(_bits(got[free.cuda()]), _bits(logits[free.cuda()]))        # untouched rows keep their bits
    assert torch.equal(_bits(_run(logits, st, offset)), _bits(got))                 # deterministic


def test_a_row_alone_equals_the_row_in_a_batch():
    logits, st, masks, sp = _case(64, 128256, torch.bfloat16, seed=9)
    batch = _run(logits, st)
    from swiftllm_b200.sampling_params import constraint_words
    from swiftllm_b200.worker.infer_state import ConstraintState
    for r in (0, 1, 2, 33):
        cw = constraint_words([masks[r]], [sp[r]], 1, 128256)
        if cw is None:
            continue
        one = ConstraintState.from_staged(torch.from_numpy(cw.words), *cw[1:])
        assert torch.equal(_bits(_run(logits[r:r + 1], one)), _bits(batch[r:r + 1])), r


@pytest.mark.parametrize("case", ["one-id", "top-k-above-allowed", "small-top-p", "tied-allowed"])
def test_sampling_kernel_on_heavily_masked_rows(case):
    """Constrained logits into the sampling kernel: the token is allowed and matches the sampling restatement."""
    from swiftllm_b200 import token_mask
    from swiftllm_b200.worker.kernels.sampling import sample_tokens
    from swiftllm_b200.worker.infer_state import ConstraintState
    from swiftllm_b200.sampling_params import constraint_words
    B, V = 32, 128256
    rng = np.random.default_rng(3)
    g = torch.Generator(device="cuda").manual_seed(3)
    logits = (torch.randn((B, V), generator=g, device="cuda") * 3).to(torch.bfloat16)
    allowed = [np.sort(rng.choice(V, 1 if case == "one-id" else 7, replace=False)) for _ in range(B)]
    if case == "tied-allowed":
        for i, a in enumerate(allowed):
            logits[i, torch.from_numpy(a).cuda()] = 1.5
    cw = constraint_words([token_mask(V, a) for a in allowed], None, B, V)
    st = ConstraintState.from_staged(torch.from_numpy(cw.words), *cw[1:])
    x = _run(logits, st)
    T = [0.9 + 0.1 * (i % 3) for i in range(B)]
    K = [50 if case == "top-k-above-allowed" else 0] * B
    P = [0.05 if case == "small-top-p" else 1.0] * B
    seeds = [1000 + i for i in range(B)]
    pos = [7 + i for i in range(B)]
    dev = lambda v, dt: torch.tensor(v, dtype=dt, device="cuda")
    tok = sample_tokens(x, dev(T, torch.float32), dev(K, torch.int32), dev(P, torch.float32), dev(seeds, torch.int64),
                        dev(pos, torch.int32)).tolist()
    ref = SO.sample_tokens(x.cpu(), T, K, P, seeds, pos)
    for t, r, a in zip(tok, ref, allowed):
        assert t in a.tolist()
        assert t == r.token or r.gap <= 1e-5 * abs(r.score) or r.boundary_margin <= 1e-4, (t, r.token)


# ---------------------------------------------------------------- through LlamaModel
V_TINY = 1000


def _models(*graphs):
    from test_sampling_gpu import _model, _weights
    w = _weights()
    return [_model(g, w=w) for g in graphs]


def _rand_mask(rng, p=None):
    from swiftllm_b200 import token_mask
    p = p if p is not None else rng.choice([0.005, 0.1, 0.6])
    ids = np.flatnonzero(rng.random(V_TINY) < p)
    return token_mask(V_TINY, ids if ids.size else [int(rng.integers(0, V_TINY))])


def test_a_single_allowed_id_forces_the_token_for_every_row():
    from swiftllm_b200 import SamplingParams, token_mask
    m, = _models(True)
    rng = np.random.default_rng(1)
    prompts, sids = [rng.integers(0, V_TINY, size=n).tolist() for n in (20, 5, 9)], [0, 1, 2]
    sp = [SamplingParams(0.0), SamplingParams(1.2, seed=3, logit_bias={4: 100.0}), SamplingParams(0.8, top_k=5, top_p=0.5, seed=4)]
    lens = [len(p) for p in prompts]
    forced = [[int(x) for x in rng.integers(0, V_TINY, size=3)] for _ in range(6)]
    t = m.forward(prompts, sids, [], sampling_params_list=sp, token_masks_list=[token_mask(V_TINY, [f]) for f in forced[0]])
    assert t == forced[0]
    for s in range(1, 6):
        lens = [l + 1 for l in lens]
        t = m.forward([[x] for x in t], sids, lens, sampling_params_list=sp,
                      token_masks_list=[token_mask(V_TINY, [f]) for f in forced[s]])
        assert t == forced[s]


def test_greedy_tokens_are_allowed_and_eager_equals_graph_replay_with_changing_masks():
    """Every step has fresh masks and biases; eager and graph-replayed steps return the same tokens and the raw logits of both
    constrained by the restatement give those tokens (greedy rows) - and every token is allowed."""
    from swiftllm_b200 import SamplingParams
    eager, graph = _models(False, True)
    rng = np.random.default_rng(2)
    prompts, sids = [rng.integers(0, V_TINY, size=n).tolist() for n in (33, 4, 17, 9)], [3, 1, 0, 2]
    ta = eager.forward(prompts, sids, [])
    tb = graph.forward(prompts, sids, [])
    assert ta == tb
    lens = [len(p) for p in prompts]
    for s in range(8):
        lens = [l + 1 for l in lens]
        masks = [_rand_mask(rng) if (s + i) % 4 else None for i in range(4)]
        bias = [None if (s * i) % 3 == 1 else {int(v): float(rng.uniform(-100, 100)) for v in rng.choice(V_TINY, 1 + s * 40)}
                for i in range(4)]
        sp = [SamplingParams(0.0 if i % 2 == 0 else 0.9, seed=50 + i, logit_bias=bias[i]) for i in range(4)]
        ta = eager.forward([[x] for x in ta], sids, lens, sampling_params_list=sp, token_masks_list=masks)
        tb = graph.forward([[x] for x in tb], sids, lens, sampling_params_list=sp, token_masks_list=masks)
        assert ta == tb
        want = CO.constrain(eager.post_layer.last_logits.cpu(), masks, bias)
        for i in (0, 2):
            assert ta[i] == int(torch.argmax(want[i]))
        for t, mk in zip(ta, masks):
            assert mk is None or CO.allowed_ids(mk, t, t + 1)[0]
    caps = {k[-1] for k in graph._graphs if "constrained" in k}
    assert caps and all(c == 0 or c & (c - 1) == 0 for c in caps)


def test_a_constrained_row_alone_equals_the_row_in_a_batch():
    from swiftllm_b200 import SamplingParams
    batch, alone = _models(False, False)
    rng = np.random.default_rng(4)
    prompts, sids = [rng.integers(0, V_TINY, size=n).tolist() for n in (12, 30, 7)], [0, 1, 2]
    sp = [SamplingParams(0.0, logit_bias={5: 20.0}), SamplingParams(0.8, seed=8), SamplingParams(1.0, top_k=8, seed=9)]
    masks = [_rand_mask(rng, 0.1) for _ in range(3)]
    tb = batch.forward(prompts, sids, [], sampling_params_list=sp, token_masks_list=masks)
    ta = [alone.forward([prompts[i]], [sids[i]], [], sampling_params_list=[sp[i]], token_masks_list=[masks[i]])[0]
          for i in range(3)]
    assert ta == tb


def test_constraints_penalties_and_logprobs_together():
    """forward_with_logprobs with masks, biases and penalties: the tokens are forward()'s, allowed, and the log-probabilities are
    those of an unconstrained call on the same state (raw logits)."""
    from swiftllm_b200 import SamplingParams
    a, b, c = _models(False, False, True)
    rng = np.random.default_rng(5)
    prompts, sids = [rng.integers(0, V_TINY, size=n).tolist() for n in (40, 11)], [0, 1]
    sp = [SamplingParams(0.0, logprobs=5, repetition_penalty=1.4, logit_bias={7: 50.0}),
          SamplingParams(0.9, seed=12, logprobs=2, frequency_penalty=0.8, presence_penalty=0.3)]
    plain = [SamplingParams(s.temperature, seed=s.seed, logprobs=s.logprobs) for s in sp]
    ids, lens = prompts, []
    for s in range(5):
        masks = [_rand_mask(rng, 0.3) for _ in range(2)]
        ra = a.forward_with_logprobs(ids, sids, lens, sampling_params_list=plain)
        rb = b.forward_with_logprobs(ids, sids, lens, sampling_params_list=sp, token_masks_list=masks)
        tc = c.forward(ids, sids, lens, sampling_params_list=sp, token_masks_list=masks)
        assert [r.token for r in rb] == tc
        for x, y, mk in zip(ra, rb, masks):
            assert x.top == y.top and x.logprob is not None and CO.allowed_ids(mk, y.token, y.token + 1)[0]
        lens = [len(p) + s + 1 for p in prompts]
        ids = [[x] for x in tc]


def test_speculative_with_per_row_masks_equals_plain_masked_steps():
    """Per-row masks (row j's = the plain step's at that position), a draft its row's mask disallows in some cases: the returned
    tokens are the restatement applied to the verify rows' own raw logits with the acceptance rule, and, for greedy entries,
    the plain masked steps' tokens (up to a near-tie: the verify GEMMs round differently from a decode step's)."""
    from swiftllm_b200 import SamplingParams
    from test_speculative_gpu import _agrees
    plain, spec = _models(False, False)
    rng = np.random.default_rng(6)
    for sid, (k, wrong, temp) in enumerate(((5, 2, 0.0), (7, None, 0.0), (4, 1, 0.9), (6, None, 0.9))):
        bias = {3: 5.0, 9: -5.0}
        sp = SamplingParams(temp, seed=40 + sid, logit_bias=bias)
        prompt = rng.integers(0, V_TINY, size=20 + sid).tolist()
        x = plain.forward([prompt], [sid], [], sampling_params_list=[sp])[0]
        spec.forward([prompt], [sid], [], sampling_params_list=[sp])
        L = len(prompt)
        masks = [_rand_mask(rng, 0.2) for _ in range(k + 1)]
        ys, inp = [], x
        for j in range(k + 1):
            ys.append(plain.forward([[inp]], [sid], [L + j + 1], sampling_params_list=[sp], token_masks_list=[masks[j]])[0])
            inp = ys[-1]
        drafts = list(ys[:k])
        if wrong is not None:
            drafts[wrong] = int(np.flatnonzero(~CO.allowed_ids(masks[wrong], 0, V_TINY))[0])
        out = spec.forward_speculative([[x] + drafts], [sid], [L], sampling_params_list=[sp], token_masks_list=[np.stack(masks)])[0]
        con = CO.constrain(spec.post_layer.last_logits.cpu(), masks, [bias] * (k + 1))
        if temp == 0:
            y = torch.argmax(con, dim=1).tolist()
        else:
            res = SO.sample_tokens(con, [temp] * (k + 1), [0] * (k + 1), [1.0] * (k + 1), [40 + sid] * (k + 1),
                                   [L + j + 1 for j in range(k + 1)])
            y = [r.token for r in res]
        n = 0
        while n < k and drafts[n] == y[n]:
            n += 1
        assert out == y[:n + 1]
        if wrong is not None:
            assert n <= wrong
        if temp == 0 and _agrees(out, ys, con, 2 ** -5):
            assert out == ys[:(k if wrong is None else wrong) + 1]


def test_prompt_logprobs_are_unchanged_by_constraints():
    from swiftllm_b200 import SamplingParams
    a, b = _models(False, False)
    rng = np.random.default_rng(7)
    prompts, sids = [rng.integers(0, V_TINY, size=n).tolist() for n in (25, 9)], [0, 1]
    sp = [SamplingParams(0.0, prompt_logprobs=3, logit_bias={1: 9.0}), SamplingParams(0.7, seed=2, prompt_logprobs=0, logprobs=1)]
    plain = [SamplingParams(s.temperature, seed=s.seed, prompt_logprobs=s.prompt_logprobs, logprobs=s.logprobs) for s in sp]
    ra = a.forward_with_logprobs(prompts, sids, [], sampling_params_list=plain)
    rb = b.forward_with_logprobs(prompts, sids, [], sampling_params_list=sp, token_masks_list=[_rand_mask(rng, 0.05), None])
    for x, y in zip(ra, rb):
        for f in ("token_ids", "logprobs", "ranks", "top_ids", "top_logprobs"):
            assert np.array_equal(getattr(x.prompt, f), getattr(y.prompt, f))
