"""GPU: the vocabulary-row kernels (csrc/sampling.cu, logprobs.cu, penalties.cu, prompt_logprobs.cu) at every cluster size C,
at the vocabularies where the shared-memory slice changes, with empty CTAs, unaligned rows, shards that split a noise group and
the edge rows of sampling, against the row run alone and against the restatements (tests/sampling_oracle.py,
logprobs_oracle.py, penalties_oracle.py, prompt_logprobs_oracle.py).

Batch sizes come from tests/vocab_geometry.py, the mirror of cluster_geometry that tests/test_vocab_geometry_cpu.py holds to
the sources; every case id names the cluster size the launch runs (C4-V128256: clusters of 4 CTAs, V = 128256).  Each row's
result is a pure function of the row, so a row must be bit-identical at every C, at every batch position and alone.  The CPU
restatements are slow at large V, so only a few rows per case are restated; the rest are held to the row run alone."""
import numpy as np
import pytest
import torch

import logprobs_oracle as LO
import penalties_oracle as PO
import prompt_logprobs_oracle as PLO
import sampling_oracle as SO
import vocab_geometry as VG

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
DT_IDS = ["bf16", "fp16"]
ROW_VS = [1000, 32001, 128256, 151936]
KEY_CASES = [(C, V) for V in ROW_VS for C in (8, 4, 2, 1) if VG.batch_for(C, V, *VG.KEYS)]
SLOT_CASES = [(C, V) for V in ROW_VS for C in (8, 4, 2, 1) if VG.batch_for(C, V, *VG.SLOTS)]
KEY_EDGES = [102400, 102401, 204800, 204801, 409600, 409601, 819200]
SLOT_EDGES = [51200, 51201, 102400, 102401, 204800, 204801, 409600]
TINY_VS = [1, 2, 7, 8, 9, 17, 63, 65, 129]
BIG_BATCH = 67                                   # runs the smallest cluster the slice allows (vocab_geometry.BATCHES)


def _cid(C, V):
    return f"C{C}-V{V}"


def _edge_ids(Vs, entry):
    return [f"C{VG.smallest_cluster(V, *entry)}-V{V}" for V in Vs]


def _dev(a, dt):
    return torch.as_tensor(a, dtype=dt, device="cuda")


def _bits(t):
    return t.detach().contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


# ---------------------------------------------------------------- rows
def _rows(R, V, dtype, seed):
    """R rows of V logits with repeated values, the row maximum tied on both sides of every CTA slice boundary of every
    cluster size (so the (key desc, id asc) order crosses CTAs), and a tied group just below the maximum (top-k / top-N ties)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    lg = (torch.randn((R, V), generator=g, device="cuda") * 2.5).to(dtype)
    if V >= 200:
        lg[:, ::97] = lg[:, 5:6]
    top = lg.float().max(dim=1).values
    for C in (2, 4, 8):
        for b, _ in VG.cta_ranges(V, C, VG.KEYS[1])[1:]:
            if 0 < b < V:
                lg[:, b - 1] = top.to(dtype)
                lg[:, b] = top.to(dtype)
    if V >= 64:
        second = (top - 0.25).to(dtype)
        lg[:, V // 3:V // 3 + 6] = second[:, None]
    return lg


def _fill(B, V, dtype, seed, probe, at):
    """A batch of B rows: the probe rows at positions `at`, random rows elsewhere."""
    out = _rows(B, V, dtype, seed + 7919)
    out[torch.as_tensor(at, device="cuda")] = probe
    return out


def _positions(B, R, seed):
    return sorted(np.random.default_rng(seed).permutation(B)[:R].tolist())


# ---------------------------------------------------------------- sampling
SAMPLE_KINDS = [(0.0, 0, 1.0), (0.8, 0, 1.0), (1.0, 1, 1.0), (0.9, 5, 1.0), (0.7, 0, 0.9), (1.2, 50, 0.95), (1.7, 0, 0.3),
                (0.5, -1, 1.0)]              # top_k -1: V // 3 + 1 (filled in per V)


def _sample_params(R, V, seed):
    rng = np.random.default_rng(seed)
    kinds = [SAMPLE_KINDS[i % len(SAMPLE_KINDS)] for i in range(R)]
    temp = [float(t) for t, _, _ in kinds]
    top_k = [V // 3 + 1 if k < 0 else k for _, k, _ in kinds]
    top_p = [float(np.float32(p)) for _, _, p in kinds]
    seed_ = [int(x) for x in rng.integers(0, 2 ** 63, size=R)]
    pos = [int(x) for x in rng.integers(1, 5000, size=R)]
    return temp, top_k, top_p, seed_, pos


def _sample(logits, temp, top_k, top_p, seed, pos, vocab_offset=0):
    from swiftllm_b200.worker.kernels.sampling import sample_tokens
    B = logits.shape[0]
    pairs = torch.empty((B, 2), dtype=torch.float32, device="cuda")
    tok = sample_tokens(logits, _dev(temp, torch.float32), _dev(top_k, torch.int32), _dev(top_p, torch.float32),
                        _dev(seed, torch.int64), _dev(pos, torch.int32), vocab_offset=vocab_offset, out_pairs=pairs)
    return tok.cpu(), pairs.cpu()


def _pick(p, idx):
    return [[x[i] for i in idx] for x in p]


def _check_sampled(logits, rows, params, got, vocab_offset=0):
    """Tokens of `rows` against the restatement, with the exemptions of tests/test_sampling_gpu.py."""
    temp, top_k, top_p, seed, pos = params
    ref = SO.sample_tokens(logits[rows], *_pick(params, rows), vocab_offset=vocab_offset)
    for r, res in zip(rows, ref):
        t = int(got[r])
        if res.kept is not None and res.boundary_margin <= 1e-4:
            continue
        if t != res.token:
            assert res.gap <= 1e-5 * abs(res.score), (r, t, res.token, res.gap, temp[r], top_k[r], top_p[r])
        if res.kept is not None:
            assert res.kept[t - vocab_offset], (r, "token outside the kept set")
    return ref


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("C,V", KEY_CASES, ids=[_cid(*c) for c in KEY_CASES])
def test_sampling_is_the_same_at_every_cluster_size(C, V, dtype):
    R = 8
    B = VG.batch_for(C, V, *VG.KEYS)
    assert VG.cluster_geometry(B, V, *VG.KEYS)[0] == C and VG.cluster_geometry(1, V, *VG.KEYS)[0] == 8
    probe = _rows(R, V, dtype, V)
    params = _sample_params(R, V, V + 1)
    alone = [_sample(probe[r:r + 1], *_pick(params, [r])) for r in range(R)]
    at = _positions(B, R, B + V)
    batch = _fill(B, V, dtype, V + B, probe, at)
    fparams = _sample_params(B, V, V + B + 1)
    for j, r in enumerate(at):
        for f, p in zip(fparams, params):
            f[r] = p[j]
    tok, pairs = _sample(batch, *fparams)
    tok2, pairs2 = _sample(batch, *fparams)
    assert torch.equal(tok, tok2) and torch.equal(pairs.view(torch.int32), pairs2.view(torch.int32)), "not run to run"
    for j, r in enumerate(at):
        assert int(tok[r]) == int(alone[j][0][0]), (j, r)
        assert torch.equal(pairs[r].view(torch.int32), alone[j][1][0].view(torch.int32)), (j, r)
    assert 0 <= int(tok.min()) and int(tok.max()) < V
    # the probe rows (identical at every C, so restated once per V) and two filler rows of this batch
    fill = [r for r in range(B) if r not in at][:2]
    _check_sampled(batch, at + fill if V <= 32001 or C == 8 else at[:4] + fill[:1], fparams, tok)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("C,V", KEY_CASES, ids=[_cid(*c) for c in KEY_CASES])
def test_token_logprobs_are_the_same_at_every_cluster_size(C, V, dtype):
    from swiftllm_b200.worker.kernels.logprobs import token_logprobs
    R = 6
    B = VG.batch_for(C, V, *VG.KEYS)
    probe = _rows(R, V, dtype, 3 * V)
    probe[0, 3] = -0.0
    rng = np.random.default_rng(V + C)
    at = _positions(B, R, 2 * B + V)
    batch = _fill(B, V, dtype, 5 * V + B, probe, at)
    tokens = rng.integers(0, V, size=B)
    tokens[at[0]] = int(torch.argmax(batch[at[0]]))
    tk = _dev(tokens, torch.int64)
    for n in (1, 5, 20):
        got = [x.cpu() for x in token_logprobs(batch, tk, n)]
        again = [x.cpu() for x in token_logprobs(batch, tk, n)]
        assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(got, again)), "not run to run"
        for r in at:
            one = [x.cpu() for x in token_logprobs(batch[r:r + 1], tk[r:r + 1], n)]
            assert all(torch.equal(_bits(a[r:r + 1]), _bits(b)) for a, b in zip(got, one)), (r, n)
        rows = at[:3] + [r for r in range(B) if r not in at][:1]
        tl, ids, tlp = (x.numpy()[rows] for x in got)
        sub = batch[rows]
        want_tl, want_ids, _ = LO.token_logprobs(sub, tokens[rows], n)
        assert np.array_equal(ids, want_ids), n
        ref64 = LO.log_softmax64(sub)
        assert np.abs(tl - ref64[np.arange(len(rows)), tokens[rows]]).max() <= LO.TOL
        assert np.abs(tlp - np.take_along_axis(ref64, ids.astype(np.int64), axis=1)).max() <= LO.TOL
        assert ids[0, 0] == tokens[at[0]] and tlp[0, 0] == tl[0]


# ---------------------------------------------------------------- penalties
BS = 16


def _word(ids, out):
    return (np.asarray(ids, dtype=np.int64) | (np.asarray(out, dtype=np.int64) << 31)).astype(np.uint32).view(np.int32)


def _pen_case(B, V, dtype, seed, vocab_offset=0, v_full=None, n_pre=None, hist_lens=(0, 1, 17, 600, 3000)):
    """B rows of a penalty launch (the first n_pre are prefill entries), with histories over [0, v_full) + an id past it,
    behind a shuffled block table; any subset of rows (prefill rows first) can be launched on its own with _pen_run."""
    v_full = v_full or V
    rng = np.random.default_rng(seed)
    logits = _rows(B, V, dtype, seed)
    for j, x in enumerate((float("nan"), float("inf"), -float("inf"), -0.0)):
        if 7 + j < V:
            logits[:, 7 + j] = x
    n_pre = B // 3 if n_pre is None else n_pre
    hist = [hist_lens[i % len(hist_lens)] for i in range(B)]
    n_new = [int(rng.integers(1, 40)) if i < n_pre else 1 for i in range(B)]
    pos = [h + n for h, n in zip(hist, n_new)]
    nblk = [(p + BS - 1) // BS for p in pos]
    pool = rng.permutation(sum(nblk) + 5)
    bt = np.full((B + 2, max(nblk)), -1, dtype=np.int32)
    seq_ids = rng.permutation(B + 2)[:B]
    used = 0
    for i in range(B):
        bt[seq_ids[i], :nblk[i]] = pool[used:used + nblk[i]]
        used += nblk[i]
    tc = rng.integers(-2 ** 31, 2 ** 31, size=(len(pool), BS), dtype=np.int64).astype(np.int32)
    histories, new_ids = [], []
    for i in range(B):
        ids = rng.integers(0, v_full, size=hist[i])
        if hist[i] >= 17:
            ids[:4] = [vocab_offset, vocab_offset + V - 1, v_full + 5, max(0, vocab_offset - 1)]
            ids[4:40] = vocab_offset + (i % V)                        # one id many times (prompt and output)
        out = rng.random(hist[i]) < 0.6
        q = np.arange(hist[i])
        tc[bt[seq_ids[i], q // BS], q % BS] = _word(ids, out)
        new = rng.integers(0, v_full, size=n_new[i])
        histories.append((np.concatenate([ids, new]), np.concatenate([out, np.full(n_new[i], i >= n_pre)])))
        new_ids.append(new)
    params = [(1.0, 0.0, 0.0) if i % 5 == 4 else (float(rng.uniform(0.5, 2.0)), float(rng.uniform(-2, 2)) * (i % 4 != 1),
                                                   float(rng.uniform(-2, 2))) for i in range(B)]
    return dict(logits=logits, params=params, histories=histories, tc=tc, bt=bt, seq_ids=seq_ids, pos=pos, n_pre=n_pre,
                n_new=n_new, new_ids=new_ids, vocab_offset=vocab_offset)


def _pen_run(c, rows, logits=None):
    """Penalises rows `rows` of the case (prefill rows first) as one launch; returns the penalised copy [len(rows), V]."""
    from swiftllm_b200.worker.kernels.penalties import apply_penalties
    rows = list(rows)
    pre = [r for r in rows if r < c["n_pre"]]
    assert rows[:len(pre)] == pre
    lg = (c["logits"] if logits is None else logits)[torch.as_tensor(rows, device="cuda")].clone()
    new = [c["new_ids"][r] for r in rows]
    flat = np.concatenate(new).astype(np.int32)
    last = np.cumsum([len(x) for x in new]) - 1
    r_, f_, p_ = (_dev([c["params"][r][k] for r in rows], torch.float32) for k in range(3))
    tok = _dev(c["tc"], torch.int32).clone()
    apply_penalties(lg, r_, f_, p_, _dev([c["pos"][r] for r in rows], torch.int32), _dev([c["seq_ids"][r] for r in rows], torch.int32),
                    _dev(flat, torch.int32), _dev(last, torch.int32), _dev([c["n_new"][r] for r in pre] or [0], torch.int32),
                    len(pre), _dev(c["bt"], torch.int32), tok, vocab_offset=c["vocab_offset"])
    return lg


def _same_bits(a, b):
    a, b = a.cpu(), b.cpu()
    both_nan = torch.isnan(a.float()) & torch.isnan(b.float())
    return bool(((a.view(torch.int16) == b.view(torch.int16)) | both_nan).all())


def _pen_check(c, rows, got, check):
    for j, r in enumerate(rows):
        if r in check:
            want = PO.penalize_row(c["logits"][r], *c["params"][r], c["histories"][r], vocab_offset=c["vocab_offset"])
            assert _same_bits(got[j], want), (r, c["params"][r])


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("C,V", SLOT_CASES, ids=[_cid(*c) for c in SLOT_CASES])
def test_penalties_are_the_same_at_every_cluster_size(C, V, dtype):
    B = VG.batch_for(C, V, *VG.SLOTS)
    assert VG.cluster_geometry(B, V, *VG.SLOTS)[0] == C
    c = _pen_case(VG.BATCHES[-1], V, dtype, seed=V + 11)
    probe = [0, 1, 2, 30, 31, 33, 60]                   # prefill rows 0-2 (n_pre = 22), decode rows, one row left alone (r % 5 == 4)
    others = [r for r in range(VG.BATCHES[-1]) if r not in probe]
    fill = sorted(np.random.default_rng(C).permutation(others)[:B - len(probe)].tolist())
    rows = sorted(probe + fill, key=lambda r: (r >= c["n_pre"], r if C % 2 else -r))    # prefill first; order varies with C
    got = _pen_run(c, rows)
    alone = {r: _pen_run(c, [r]) for r in probe}
    for j, r in enumerate(rows):
        if r in alone:
            assert torch.equal(got[j].view(torch.int16), alone[r][0].view(torch.int16)), r
    _pen_check(c, rows, got, set(probe) | set(fill[:3]))
    for j, r in enumerate(rows):
        if c["params"][r] == (1.0, 0.0, 0.0):                           # penalties off: the row keeps its bits
            assert torch.equal(got[j].view(torch.int16), c["logits"][r].view(torch.int16)), r


# ---------------------------------------------------------------- vocabulary edges
@pytest.mark.parametrize("V", KEY_EDGES, ids=_edge_ids(KEY_EDGES, VG.KEYS))
def test_sampling_and_logprobs_at_the_vocabulary_edges(V):
    from swiftllm_b200.worker.kernels.logprobs import token_logprobs
    dtype = DTYPES[V % 2]
    B = BIG_BATCH
    assert VG.cluster_geometry(B, V, *VG.KEYS)[0] == VG.smallest_cluster(V, *VG.KEYS)
    probe = _rows(2, V, dtype, V)
    at = [0, B - 1]
    batch = _fill(B, V, dtype, V + 1, probe, at)
    params = _sample_params(B, V, V)
    params[0][0], params[1][0], params[2][0] = 0.8, 50, 0.9                  # row 0: top-k + top-p
    params[0][B - 1], params[1][B - 1], params[2][B - 1] = 1.1, 0, 1.0       # row B - 1: temperature only
    tok, pairs = _sample(batch, *params)
    for r in at:
        one, one_pairs = _sample(batch[r:r + 1], *_pick(params, [r]))
        assert int(one[0]) == int(tok[r]) and torch.equal(one_pairs[0].view(torch.int32), pairs[r].view(torch.int32)), r
    assert 0 <= int(tok.min()) and int(tok.max()) < V
    _check_sampled(batch, at[:1] if V > 204800 else at, params, tok)
    tokens = np.random.default_rng(V).integers(0, V, size=B)
    tk = _dev(tokens, torch.int64)
    got = [x.cpu() for x in token_logprobs(batch, tk, 20)]
    for r in at:
        one = [x.cpu() for x in token_logprobs(batch[r:r + 1], tk[r:r + 1], 20)]
        assert all(torch.equal(_bits(a[r:r + 1]), _bits(b)) for a, b in zip(got, one)), r
    tl, ids, tlp = (x.numpy()[at[:1]] for x in got)
    want_tl, want_ids, _ = LO.token_logprobs(batch[at[:1]], tokens[at[:1]], 20)
    assert np.array_equal(ids, want_ids)
    ref64 = LO.log_softmax64(batch[at[:1]])
    assert abs(tl[0] - ref64[0, tokens[0]]) <= LO.TOL
    assert np.abs(tlp - np.take_along_axis(ref64, ids.astype(np.int64), axis=1)).max() <= LO.TOL


@pytest.mark.parametrize("V", SLOT_EDGES, ids=_edge_ids(SLOT_EDGES, VG.SLOTS))
def test_penalties_at_the_vocabulary_edges(V):
    dtype = DTYPES[V % 2]
    c = _pen_case(BIG_BATCH, V, dtype, seed=V, hist_lens=(5, 40, 300))
    assert VG.cluster_geometry(BIG_BATCH, V, *VG.SLOTS)[0] == VG.smallest_cluster(V, *VG.SLOTS)
    rows = list(range(BIG_BATCH))
    got = _pen_run(c, rows)
    for r in (0, c["n_pre"], BIG_BATCH - 1):
        assert torch.equal(_pen_run(c, [r])[0].view(torch.int16), got[r].view(torch.int16)), r
    _pen_check(c, rows, got, {0, c["n_pre"], BIG_BATCH - 1})


def test_vocabularies_past_the_largest_slice_are_refused_before_any_launch():
    from swiftllm_b200.worker.kernels.logprobs import token_logprobs
    from swiftllm_b200.worker.kernels.sampling import sample_tokens
    assert not VG.accepted(819201, *VG.KEYS) and not VG.accepted(409601, *VG.SLOTS)
    lg = torch.zeros((2, 819201), dtype=torch.bfloat16, device="cuda")
    one = lambda v, dt: _dev([v, v], dt)
    with pytest.raises(RuntimeError, match="does not fit the shared memory"):
        sample_tokens(lg, one(1.0, torch.float32), one(0, torch.int32), one(1.0, torch.float32), one(1, torch.int64),
                      one(1, torch.int32))
    with pytest.raises(RuntimeError, match="does not fit the shared memory"):
        token_logprobs(lg, one(0, torch.int64), 5)
    c = _pen_case(2, 409601, torch.float16, seed=1, hist_lens=(30,))
    with pytest.raises(RuntimeError, match="does not fit the shared memory"):
        _pen_run(c, [0, 1])
    torch.cuda.synchronize()


# ---------------------------------------------------------------- tiny vocabularies: whole CTAs of the cluster empty
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("V", TINY_VS, ids=[_cid(8, V) for V in TINY_VS])
def test_tiny_vocabularies_leave_ctas_empty(V, dtype):
    from swiftllm_b200.worker.kernels.logprobs import token_logprobs
    assert VG.cluster_geometry(1, V, *VG.KEYS)[0] == 8 and VG.cluster_geometry(1, V, *VG.SLOTS)[0] == 8
    lg = (torch.randn((4, V), generator=torch.Generator(device="cuda").manual_seed(V), device="cuda") * 2).to(dtype)
    if V >= 4:
        lg[1, V - 2:] = lg[1].max()                                    # tied maxima in the last (partial) CTA
    kinds = [(0.0, 0, 1.0), (0.9, V + 3, 1.0), (1.3, V, 0.6), (0.7, max(1, V - 1), 0.9), (1.0, 1, 1.0), (2.0, 0, 1e-6)]
    for r in range(4):
        for j, (t, k, p) in enumerate(kinds):
            params = ([t], [k], [float(np.float32(p))], [1000 + 17 * j + r], [r + 1])
            tok, pairs = _sample(lg[r:r + 1], *params)
            assert 0 <= int(tok[0]) < V
            res = SO.sample_tokens(lg[r:r + 1], *params)[0]
            if not (res.kept is not None and res.boundary_margin <= 1e-4):
                assert int(tok[0]) == res.token or res.gap <= 1e-5 * abs(res.score), (r, j)
            if res.kept is not None:
                assert res.kept[int(tok[0])]
                if res.kept.sum() == 1:
                    assert int(tok[0]) == res.token
        tokens = [0, V - 1, V, -1][r]
        tl, ids, tlp = (x.cpu().numpy() for x in token_logprobs(lg[r:r + 1], _dev([tokens], torch.int64), 20))
        want_tl, want_ids, _ = LO.token_logprobs(lg[r:r + 1], [tokens], 20)
        assert np.array_equal(ids, want_ids)
        assert (ids[0, min(V, 20):] == -1).all() and np.isnan(tlp[0, min(V, 20):]).all()
        ref64 = LO.log_softmax64(lg[r:r + 1])
        assert np.abs(tlp[0, :min(V, 20)] - ref64[0, ids[0, :min(V, 20)]]).max() <= LO.TOL
        if 0 <= tokens < V:
            assert abs(tl[0] - ref64[0, tokens]) <= LO.TOL
        else:
            assert np.isnan(tl[0])
    # penalties of a tiny shard at offset 1000: most history ids fall outside it
    c = _pen_case(3, V, dtype, seed=V, vocab_offset=1000, v_full=1000 + V + 50, n_pre=1, hist_lens=(40, 300, 2000))
    for r in range(3):
        got = _pen_run(c, [r])
        _pen_check(c, [r], got, {r})


# ---------------------------------------------------------------- unaligned rows
@pytest.mark.parametrize("V", [1001, 32001])
@pytest.mark.parametrize("off", [1, 3, 5, 8])
def test_unaligned_rows_match_the_contiguous_copy(off, V):
    dtype = torch.bfloat16 if off % 2 else torch.float16
    for B in (5, 24):                                                    # C = 8 and C = 4
        wide = _rows(B, V + 16, dtype, V + off + B)
        view = wide[:, off:off + V]
        params = _sample_params(B, V, off)
        a = _sample(view, *params)
        b = _sample(view.contiguous(), *params)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))
        _check_sampled(view, [0, 1, 2, 3, 4] if B == 5 else [6, 7], params, a[0])
        # penalties in place on the view: the same bits as on the contiguous copy, the columns around it untouched
        c = _pen_case(B, V, dtype, seed=off + B, n_pre=2)
        c["logits"] = view.contiguous()
        want = _pen_run(c, list(range(B)))
        before = wide.clone()
        from swiftllm_b200.worker.kernels.penalties import apply_penalties
        rows = list(range(B))
        new = [c["new_ids"][r] for r in rows]
        apply_penalties(view, *(_dev([c["params"][r][k] for r in rows], torch.float32) for k in range(3)),
                        _dev(c["pos"], torch.int32), _dev(c["seq_ids"], torch.int32), _dev(np.concatenate(new), torch.int32),
                        _dev(np.cumsum([len(x) for x in new]) - 1, torch.int32), _dev(c["n_new"][:2], torch.int32), 2,
                        _dev(c["bt"], torch.int32), _dev(c["tc"], torch.int32).clone())
        assert torch.equal(view.contiguous().view(torch.int16), want.view(torch.int16))
        assert torch.equal(wide[:, :off].view(torch.int16), before[:, :off].view(torch.int16))
        assert torch.equal(wide[:, off + V:].view(torch.int16), before[:, off + V:].view(torch.int16))
        _pen_check(c, rows, want, {0, B - 1})


# ---------------------------------------------------------------- shards that split a Philox group of 4 indices
SHARDS = {32001: [0, 5001, 13002, 20003, 32001], 128256: [0, 30001, 64002, 100003, 128256]}


@pytest.mark.parametrize("V", sorted(SHARDS))
def test_shards_at_offsets_that_split_a_noise_group(V):
    from swiftllm_b200.worker.layers.post_layer import merge_sharded_argmax
    cuts = SHARDS[V]
    assert sorted(c % 4 for c in cuts[1:-1]) == [1, 2, 3]
    B = 24
    assert VG.cluster_geometry(B, V, *VG.KEYS)[0] == 4 and VG.cluster_geometry(3, V, *VG.KEYS)[0] == 8
    lg = _rows(B, V, torch.bfloat16, V)
    temp = [0.0 if i % 6 == 0 else [0.6, 0.9, 1.4][i % 3] for i in range(B)]
    rng = np.random.default_rng(V)
    seed = [int(x) for x in rng.integers(0, 2 ** 63, size=B)]
    pos = [int(x) for x in rng.integers(1, 9000, size=B)]
    k0, p1 = [0] * B, [1.0] * B
    full, _ = _sample(lg, temp, k0, p1, seed, pos)
    assert torch.equal(_sample(lg[:3], temp[:3], k0[:3], p1[:3], seed[:3], pos[:3])[0], full[:3])
    pairs, restated = [], []
    check = [0, 1, 2, 3]
    for a, b in zip(cuts[:-1], cuts[1:]):
        shard = lg[:, a:b].contiguous()
        assert VG.cluster_geometry(B, b - a, *VG.KEYS)[0] == 4
        t4, p4 = _sample(shard, temp, k0, p1, seed, pos, vocab_offset=a)
        t8, p8 = _sample(shard[:3], temp[:3], k0[:3], p1[:3], seed[:3], pos[:3], vocab_offset=a)     # C = 8
        assert torch.equal(t8, t4[:3]) and torch.equal(p8.view(torch.int32), p4[:3].view(torch.int32))
        assert ((t4 >= a) & (t4 < b)).all()
        pairs.append(p4)
        restated.append(SO.sample_tokens(shard[check], *_pick((temp, k0, p1, seed, pos), check), vocab_offset=a))
    assert torch.equal(merge_sharded_argmax(torch.stack(pairs)), full)
    merged = SO.merge_pairs(restated)
    whole = SO.sample_tokens(lg[check], *_pick((temp, k0, p1, seed, pos), check))
    for j, r in enumerate(check):
        assert merged[j] == whole[j].token
        assert int(full[r]) == merged[j] or whole[j].gap <= 1e-5 * abs(whole[j].score), (r, int(full[r]), merged[j])
    # penalties of a shard at an offset = 2 (mod 4), at C = 8 and C = 4
    off, Vs = 30002, 16030
    c = _pen_case(24, Vs, torch.float16, seed=off + V, vocab_offset=off, v_full=128256, n_pre=3)
    got = _pen_run(c, list(range(24)))
    for r in range(3):
        assert torch.equal(_pen_run(c, [r])[0].view(torch.int16), got[r].view(torch.int16))
    _pen_check(c, list(range(24)), got, set(range(24)))


# ---------------------------------------------------------------- sampling edge rows
def _edge_batch(V, dtype):
    """Rows a sampler must survive, and their parameters; returns (logits, params, names)."""
    g = torch.Generator(device="cuda").manual_seed(V)
    lg = (torch.randn((16, V), generator=g, device="cuda") * 2).to(dtype)
    rows = []                                          # (name, T, k, p)
    lg[0, 777] = float("nan"); rows.append(("nan", 0.8, 0, 0.9))
    lg.view(torch.int16)[1, 12345 % V] = -512 if dtype == torch.float16 else -64     # 0xfe00 / 0xffc0: a NaN with the sign bit
    rows.append(("-nan", 0.8, 0, 1.0))
    lg[2, V - 3] = float("inf"); lg[2, 5] = float("inf"); rows.append(("inf", 0.8, 0, 0.9))
    lg[3, :] = -float("inf"); lg[3, V // 2] = 1.5; rows.append(("one-finite", 1.0, 0, 0.5))
    lg[4, :] = 0.0; lg[4, ::3] = -0.0; rows.append(("zeros", 1.0, 0, 1.0))
    lg[5, 4321 % V] = lg[5].max() + 1; rows.append(("k1", 0.9, 1, 1.0))
    rows.append(("k=V-1", 1.1, V - 1, 1.0))
    rows.append(("k>=V", 1.1, V + 9, 1.0))
    lg[8, 999] = lg[8].max() + 4; rows.append(("one-survivor-p", 0.7, 0, 0.01))
    lg[9, :] = -30.0; lg[9, [3, V // 3, V // 3 + 1, V - 1]] = 0.0; rows.append(("p-on-a-tie", 1.0, 0, 0.5))
    rows.append(("T=1e-3", 1e-3, 0, 1.0))
    rows.append(("T=100", 100.0, 0, 0.9))
    lg[12, :] = -float("inf"); rows.append(("all-inf", 0.9, 0, 0.9))
    lg[13, :] = float("nan"); rows.append(("all-nan", 1.0, 3, 1.0))
    lg[14, 10] = float("nan"); rows.append(("nan-k1", 1.0, 1, 1.0))
    lg[15, 20] = float("inf"); lg[15, 21] = float("nan"); rows.append(("inf-nan-greedy", 0.0, 0, 1.0))
    names = [r[0] for r in rows]
    T = [r[1] for r in rows]; K = [r[2] for r in rows]; P = [float(np.float32(r[3])) for r in rows]
    seed = [1000 + i for i in range(16)]; pos = [50 + i for i in range(16)]
    return lg, [T, K, P, seed, pos], names


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("V", [32001, 128256], ids=["C4-V32001", "C4-V128256"])
def test_sampling_edge_rows(V, dtype):
    edge, params, names = _edge_batch(V, dtype)
    R = edge.shape[0]
    alone = [_sample(edge[r:r + 1], *_pick(params, [r]))[0] for r in range(R)]
    ref = SO.sample_tokens(edge, *params)
    results = []
    for B in (24, 33, 40, 67):                                          # C = 4, 4, 2 and 1 (or 2) at two positions each
        for shift in (0, B - R):
            at = list(range(shift, shift + R))
            batch = _fill(B, V, dtype, B + shift, edge, at)
            fp = _sample_params(B, V, B)
            for j, r in enumerate(at):
                for f, p in zip(fp, params):
                    f[r] = p[j]
            tok, _ = _sample(batch, *fp)
            results.append(tok[at])
    for t in results[1:]:
        assert torch.equal(t, results[0]), "depends on the cluster size or the batch position"
    got = results[0]
    assert torch.equal(torch.cat(alone), got)
    assert torch.equal(_sample(edge, *params)[0], got)
    assert ((got >= 0) & (got < V)).all(), got
    by = dict(zip(names, range(R)))
    exact = ["nan", "-nan", "inf", "one-finite", "k1", "one-survivor-p", "p-on-a-tie", "all-inf", "all-nan", "nan-k1",
             "inf-nan-greedy"]
    for n in exact:
        assert int(got[by[n]]) == ref[by[n]].token, (n, int(got[by[n]]), ref[by[n]].token)
    # the bad rows are drawn greedily: the first index of the largest key
    assert int(got[by["nan"]]) == 777 and int(got[by["inf"]]) == 5 and int(got[by["all-inf"]]) == 0
    assert int(got[by["all-nan"]]) == 0 and int(got[by["nan-k1"]]) == 10 and int(got[by["inf-nan-greedy"]]) == 21
    assert int(got[by["-nan"]]) == int(torch.argmax(torch.nan_to_num(edge[by["-nan"]].float(), nan=-float("inf"))))
    assert int(got[by["one-finite"]]) == V // 2
    assert int(got[by["k1"]]) == 4321 % V and int(got[by["one-survivor-p"]]) == 999
    tie = ref[by["p-on-a-tie"]]
    assert set(np.nonzero(tie.kept)[0].tolist()) == {3, V // 3, V // 3 + 1, V - 1}      # the whole tied group
    assert int(got[by["p-on-a-tie"]]) in {3, V // 3, V // 3 + 1, V - 1}
    for n in ("zeros", "k=V-1", "k>=V", "T=1e-3", "T=100"):
        res = ref[by[n]]
        t = int(got[by[n]])
        assert t == res.token or res.gap <= 1e-5 * abs(res.score) or res.boundary_margin <= 1e-4, (n, t, res.token)
        assert res.kept[t]


# ---------------------------------------------------------------- prompt logprobs: the staged / streamed boundary
@pytest.mark.parametrize("V", [49151, 49152, 49153, 49159, 98305])
def test_prompt_logprobs_across_the_staging_boundary(V):
    from swiftllm_b200.worker.kernels.logprobs import prompt_logprobs, token_logprobs
    assert VG.STAGE_KEYS in (49152,) and (V <= VG.STAGE_KEYS) == (V <= 49152)
    dtype = torch.float16 if V % 2 else torch.bfloat16
    R = 8
    wide = _rows(R, V + 8, dtype, V)
    if V > VG.STAGE_KEYS:
        wide[3, :] = wide[3].float().clamp(max=1.0).to(dtype)
        wide[3, ::40] = 4.0                                         # > kMaxCand ties at the top, past the staged keys too
        assert int((wide[3] == 4.0).sum()) > VG.MAX_CAND
    rng = np.random.default_rng(V)
    for a in range(8):                                              # every 2-byte alignment of the row start
        view = wide[:, a:a + V]
        tgt = rng.integers(0, V, size=R)
        tgt[0] = int(torch.argmax(view[0]))
        tgt[1] = V - 1
        tgt[2] = VG.STAGE_KEYS if V > VG.STAGE_KEYS else V // 2
        for n in (0, 5, 20):
            lp, rank, ids, tlp = (x.cpu() for x in prompt_logprobs(view, _dev(tgt, torch.int32), n))
            tl, tids, ttlp = (x.cpu() for x in token_logprobs(view, _dev(tgt, torch.int64), n))
            assert torch.equal(_bits(lp), _bits(tl)) and torch.equal(ids, tids) and torch.equal(_bits(tlp), _bits(ttlp)), (a, n)
            if a in (0, 3) or n == 20:
                want_lp, want_rank, want_ids, _ = PLO.prompt_logprobs(view, tgt, n)
                assert np.array_equal(rank.numpy(), want_rank) and np.array_equal(ids.numpy(), want_ids), (a, n)


# ---------------------------------------------------------------- through LlamaModel: 24 sequences at V = 128256 run C = 4
LLAMA3_VOCAB = dict(model_type="llama", num_hidden_layers=1, num_attention_heads=2, num_key_value_heads=1, hidden_size=256,
                    vocab_size=128256, max_position_embeddings=512, intermediate_size=512, rope_theta=500000.0,
                    rms_norm_eps=1e-5, hidden_act="silu")


def _llama3_vocab_model(w, graph):
    import swiftllm_b200
    from swiftllm_b200.worker.weight import dict_getter
    from test_model_gpu import _hf_tensors
    cfg = LLAMA3_VOCAB
    ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=4,
                                    max_seqs_in_block_table=32, max_blocks_per_seq=8, max_batch_size=32,
                                    max_tokens_in_batch=512, dtype="bfloat16", use_cuda_graph=graph)
    m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(cfg))
    m.load_weights(dict_getter(_hf_tensors(w, cfg["intermediate_size"])))
    m.init_kvcache_and_swap(160)
    m.post_layer.keep_logits = True
    return m


def _mixed_params(n, shift):
    from swiftllm_b200 import SamplingParams
    c = [SamplingParams(0.0, logprobs=5), SamplingParams(0.8, seed=41, logprobs=0), SamplingParams(1.3, top_k=9, seed=42, logprobs=20),
         SamplingParams(0.7, top_p=0.85, seed=43), SamplingParams(1.0, top_k=40, top_p=0.9, seed=44, logprobs=3),
         SamplingParams(0.0), SamplingParams(0.9, seed=45, logprobs=1)]
    return [c[(i + shift) % len(c)] for i in range(n)]


def test_model_decodes_24_sequences_at_the_llama3_vocabulary():
    from oracle.model import OracleWeights
    N = 24
    assert VG.cluster_geometry(N, LLAMA3_VOCAB["vocab_size"], *VG.KEYS)[0] == 4
    w = OracleWeights.random(LLAMA3_VOCAB, dtype=torch.bfloat16, seed=9, std=0.05)
    eager, graph = _llama3_vocab_model(w, False), _llama3_vocab_model(w, True)
    rng = np.random.default_rng(6)
    prompts = [rng.integers(0, LLAMA3_VOCAB["vocab_size"], size=int(rng.integers(3, 20))).tolist() for _ in range(N)]
    sids = list(range(N))
    sp = _mixed_params(N, 0)
    a = eager.forward_with_logprobs(prompts, sids, [], sampling_params_list=sp)
    b = graph.forward_with_logprobs(prompts, sids, [], sampling_params_list=sp)
    assert a == b
    lens = [len(p) for p in prompts]
    for step in range(4):
        lens = [l + 1 for l in lens]
        sp = _mixed_params(N, step + 1)
        ids = [[r.token] for r in a]
        a = eager.forward_with_logprobs(ids, sids, lens, sampling_params_list=sp)
        b = graph.forward_with_logprobs(ids, sids, lens, sampling_params_list=sp)
        assert a == b, step
        logits = eager.post_layer.last_logits
        assert torch.equal(logits, graph.post_layer.last_logits)
        assert logits.shape == (N, LLAMA3_VOCAB["vocab_size"])
        ref = SO.sample_tokens(logits, [s.temperature for s in sp], [s.top_k for s in sp], [s.top_p for s in sp],
                               [s.seed for s in sp], lens)
        for r, res, s in zip(a, ref, sp):
            assert r.token == res.token or res.gap <= 1e-5 * abs(res.score) or res.boundary_margin <= 1e-4, (r.token, res.token)
        lp_rows = [i for i, s in enumerate(sp) if s.logprobs is not None]
        tl, tids, tlp = LO.token_logprobs(logits[lp_rows], [a[i].token for i in lp_rows], 20)
        ref64 = LO.log_softmax64(logits[lp_rows])
        for j, i in enumerate(lp_rows):
            n = sp[i].logprobs
            assert abs(a[i].logprob - ref64[j, a[i].token]) <= LO.TOL
            assert [t for t, _ in a[i].top] == tids[j, :n].tolist()
            assert all(abs(lp - ref64[j, t]) <= LO.TOL for t, lp in a[i].top)
    assert any(k for k in graph._graphs)
