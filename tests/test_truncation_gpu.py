"""GPU: min-p, typical-p and XTC in the sampling kernel's truncated instantiation (csrc/sampling.cu,
sllm_sample_tokens_truncated) against the numpy restatement (tests/truncation_oracle.py), and through LlamaModel (eager, CUDA
graph, chunked prefill, speculative verification) against the restatement applied to the model's own logits."""
import numpy as np
import pytest
import torch

import truncation_oracle as TO

pytestmark = pytest.mark.gpu

# (temperature, top_k, top_p, min_p, typical_p, xtc_threshold, xtc_probability)
KINDS = [
    (0.0, 0, 1.0, 0.3, 0.5, 0.1, 1.0),          # greedy: the filters are ignored
    (1.0, 0, 1.0, 0.05, 1.0, 0.1, 0.0),         # min-p
    (0.8, 0, 1.0, 0.0, 0.95, 0.1, 0.0),         # typical-p
    (1.2, 0, 1.0, 0.0, 1.0, 0.1, 1.0),          # XTC, always drawn
    (1.0, 40, 0.95, 0.02, 0.9, 0.05, 0.5),      # everything
    (1.0, 0, 1.0, 0.0, 1.0, 0.1, 0.0),          # every filter off, through the truncated entry
    (0.7, 0, 1.0, 1.0, 1.0, 0.1, 0.0),          # min_p = 1: the ties of the maximum only
    (1.5, 0, 1.0, 0.0, 1e-4, 0.1, 0.0),         # a tiny typical_p
    (1.0, 0, 1.0, 0.0, 1.0, 0.0, 1.0),          # XTC threshold 0: down to the least likely survivor
    (0.9, 0, 0.9, 0.1, 0.7, 0.02, 1.0),         # top-p then all three
]


def _params(B, rng):
    cols = list(zip(*[KINDS[i % len(KINDS)] for i in range(B)]))
    seed = [int(x) for x in rng.integers(0, 2 ** 63, size=B)]
    pos = [int(x) for x in rng.integers(1, 5000, size=B)]
    return [list(c) for c in cols[:3]], [list(c) for c in cols[3:]], seed, pos


def _t(v, dt, d):
    return torch.tensor(v, dtype=dt, device=d)


def _run(logits, base, filt, seed, pos, vocab_offset=0, pairs=False):
    from swiftllm_b200.worker.kernels.sampling import sample_tokens
    d = logits.device
    (temp, top_k, top_p) = base
    out = torch.empty((logits.shape[0], 2), dtype=torch.float32, device=d) if pairs else None
    kw = {} if filt is None else dict(zip(("min_p", "typical_p", "xtc_threshold", "xtc_probability"),
                                          (_t(f, torch.float32, d) for f in filt)))
    tok = sample_tokens(logits, _t(temp, torch.float32, d), _t(top_k, torch.int32, d), _t(top_p, torch.float32, d),
                        _t(seed, torch.int64, d), _t(pos, torch.int32, d), vocab_offset=vocab_offset, out_pairs=out, **kw)
    return (tok, out) if pairs else tok


def _rows(base, filt, seed, pos, r):
    return [c[r:r + 1] for c in base], [c[r:r + 1] for c in filt], seed[r:r + 1], pos[r:r + 1]


def _logits(B, V, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    logits = (torch.randn((B, V), generator=g, device="cuda") * 2.5).to(dtype)
    logits[:, ::97] = logits[:, 5:6]                    # repeated values: ties at every boundary
    logits[:, 3::211] = float("-inf")                   # masked ids
    if B > 2:
        logits[1, 7] = float("nan")                     # a bad row: greedy whatever the filters
    if B > 3 and dtype == torch.bfloat16:
        logits[2, 0::2] = 3e38                          # differences that overflow fp32
        logits[2, 1::2] = -3e38
    return logits


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V,offset", [(1000, 0), (32000, 0), (128256, 0), (16032, 16032 * 3)])
@pytest.mark.parametrize("B", [1, 3, 64, 257])
def test_kernel_matches_the_restatement(B, V, offset, dtype):
    if B == 257 and V == 128256 and dtype == torch.float16:
        pytest.skip("covered by bf16 at this size (CPU restatement time)")
    rng = np.random.default_rng(B * 7 + V)
    logits = _logits(B, V, dtype, B + V)
    base, filt, seed, pos = _params(B, rng)
    tok = _run(logits, base, filt, seed, pos, offset)
    assert torch.equal(tok, _run(logits, base, filt, seed, pos, offset)), "not deterministic run to run"
    for r in range(min(B, 6)):                          # a row alone == the same row inside the batch
        assert int(_run(logits[r:r + 1], *_rows(base, filt, seed, pos, r), offset)) == int(tok[r])
    ref = TO.sample_tokens(logits, *base, seed, pos, *filt, vocab_offset=offset)
    got = tok.tolist()
    # no exemption: a sampled row never draws a -inf (masked) id while it has a finite one
    drawn = logits.float().gather(1, (tok - offset)[:, None]).squeeze(1).cpu()
    assert all(bool(torch.isfinite(drawn[r])) for r, res in enumerate(ref) if res.kept is not None), \
        [(r, got[r]) for r, res in enumerate(ref) if res.kept is not None and not torch.isfinite(drawn[r])]
    exempt = 0
    for r, res in enumerate(ref):
        if res.kept is not None and res.boundary_margin <= 1e-4:
            exempt += 1
            continue
        if got[r] != res.token:
            assert res.gap <= 1e-5 * abs(res.score), (r, got[r], res.token, res.gap, [c[r] for c in base + filt])
            exempt += 1
        if res.kept is not None:
            assert res.kept[got[r] - offset], (r, "token outside the kept set")
    print(f"B={B} V={V} {dtype}: {exempt} of {B} rows exempt")
    assert exempt <= B // 2 + 2


def test_kept_sets_reached_over_seeds_lie_inside_the_restatement():
    V, S = 4000, 256
    logits = _logits(1, V, torch.bfloat16, 9)
    for kind in KINDS[1:]:
        base = [[kind[0]] * S, [kind[1]] * S, [kind[2]] * S]
        filt = [[f] * S for f in kind[3:]]
        seeds, pos = list(range(1, S + 1)), [33] * S
        toks = _run(logits.expand(S, V).contiguous(), base, filt, seeds, pos).tolist()
        for s, t in zip(seeds[:8], toks[:8]):
            res = TO.sample_tokens(logits, *[[c[0]] for c in base], [s], [33], *[[c[0]] for c in filt])[0]
            if res.boundary_margin > 1e-4:
                assert res.kept[t], (kind, s, t)
        res = TO.sample_tokens(logits, *[[c[0]] for c in base], [1], [33], *[[c[0]] for c in filt])[0]
        if res.boundary_margin > 1e-4 and kind[6] in (0.0, 1.0):            # the XTC draw is per seed unless 0 or 1
            kept = set(np.nonzero(res.kept)[0].tolist())
            assert set(toks) <= kept, (kind, sorted(set(toks) - kept)[:5])
            if len(kept) == 1:
                assert set(toks) == kept


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("V", [5, 1000, 128256])
def test_xtc_threshold_zero_stops_at_the_least_likely_finite_id(V, dtype):
    """Masked (-inf) ids are never XTC top choices: with threshold 0 and probability 1 every seed draws the least likely
    finite id, however many -inf ids lie below it, and never a -inf one."""
    S = 64
    row = torch.full((V,), float("-inf"), dtype=torch.float32)
    row[:5] = torch.tensor([3.0, 1.0, float("-inf"), 0.5, float("-inf")])
    if V > 5:
        row[V - 3:] = torch.tensor([2.0, float("-inf"), 2.5])
    rows = row.to(dtype).cuda()[None].expand(S, V).contiguous()
    for base in ([[1.0] * S, [0] * S, [1.0] * S], [[0.5] * S, [0] * S, [1.0] * S]):
        tok = _run(rows, base, [[0.0] * S, [1.0] * S, [0.0] * S, [1.0] * S], list(range(S)), [9] * S)
        assert set(tok.tolist()) == {3}, sorted(set(tok.tolist()))[:5]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_every_filter_off_equals_the_plain_entry(dtype):
    B, V = 40, 32000
    logits = _logits(B, V, dtype, 4)
    rng = np.random.default_rng(1)
    temp = [0.0 if i % 5 == 0 else float(rng.choice([0.5, 1.0, 1.6])) for i in range(B)]
    base = [temp, [0 if i % 3 else 20 for i in range(B)], [1.0 if i % 2 else 0.9 for i in range(B)]]
    seed = [int(x) for x in rng.integers(0, 2 ** 63, size=B)]
    pos = list(range(7, 7 + B))
    off = [[0.0] * B, [1.0] * B, [0.3] * B, [0.0] * B]
    for o in (0, 5 * V):
        a, pa = _run(logits, base, None, seed, pos, o, pairs=True)
        b, pb = _run(logits, base, off, seed, pos, o, pairs=True)
        assert torch.equal(a, b) and torch.equal(pa.view(torch.int32), pb.view(torch.int32))     # bit for bit (NaN pairs too)


def test_sample_tokens_without_filters_calls_the_plain_entry(monkeypatch):
    from swiftllm_b200 import _lib
    real, called = _lib.lib(), []

    class Spy:
        def __getattr__(self, name):
            called.append(name)
            return getattr(real, name)

    monkeypatch.setattr(_lib, "lib", lambda: Spy())
    logits = _logits(2, 1000, torch.bfloat16, 1)
    base, filt, seed, pos = [[1.0, 1.0], [0, 0], [1.0, 1.0]], [[0.1, 0.0], [1.0, 0.5], [0.1, 0.1], [0.0, 1.0]], [1, 2], [3, 4]
    _run(logits, base, None, seed, pos)
    _run(logits, base, filt, seed, pos)
    assert [c for c in called if c.startswith("sllm_sample")] == ["sllm_sample_tokens", "sllm_sample_tokens_truncated"]


def test_distribution_matches_the_filtered_softmax():
    from scipy.stats import chisquare
    V, S, T = 64, 30000, 0.9
    logits = (torch.linspace(-2, 2, V, device="cuda") ** 3).to(torch.bfloat16)
    for filt in ([0.01, 1.0, 0.1, 0.0], [0.0, 0.8, 0.1, 0.0], [0.02, 0.9, 0.1, 0.0]):
        rows = logits[None].expand(S, V).contiguous()
        tok = _run(rows, [[T] * S, [0] * S, [1.0] * S], [[f] * S for f in filt], list(range(S)), [17] * S).cpu().numpy()
        res = TO.sample_tokens(logits[None], [T], [0], [1.0], [0], [17], *[[f] for f in filt])[0]
        kept = res.kept
        assert kept.sum() > 2, filt
        prob = np.where(kept, np.exp((logits.float().cpu().numpy() - logits.float().max().item()) / T), 0)
        prob /= prob.sum()
        assert kept[tok].all(), filt
        cnt = np.bincount(tok, minlength=V)[kept]
        want = prob[kept].astype(np.float64)
        want *= cnt.sum() / want.sum()
        assert chisquare(cnt, want).pvalue > 1e-3, filt


def test_invalid_launch_arguments_raise():
    from swiftllm_b200 import _lib
    l = _lib.lib()
    x = torch.zeros((2, 1000), dtype=torch.bfloat16, device="cuda")
    f = torch.zeros((2,), dtype=torch.float32, device="cuda")
    p = [f.data_ptr()] * 4
    args = [x.data_ptr(), 2, 1000, 1000, 0, f.data_ptr(), f.data_ptr(), f.data_ptr(), f.data_ptr(), f.data_ptr(), f.data_ptr(),
            None]
    for i in range(4):
        q = list(p)
        q[i] = None
        assert l.sllm_sample_tokens_truncated(*args, *q, _lib.dtype_tag(torch.bfloat16), None) != 0
        assert b"null filter array" in l.sllm_last_error()
    assert l.sllm_sample_tokens_truncated(1, 2, 2_000_000, 2_000_000, 0, 1, 1, 1, 1, 1, 1, None, 1, 1, 1, 1, 1, None) != 0
    assert b"shared memory" in l.sllm_last_error()


# ---------------------------------------------------------------- through LlamaModel
def _model(graph=False, w=None, dtype="bfloat16"):
    from test_model_gpu import ENG2, TINY2, _make_model
    m = _make_model(TINY2, ENG2, w, dtype=dtype, graph=graph)
    m._sampling_rng = np.random.default_rng(0)
    return m


def _weights():
    from oracle.model import OracleWeights
    from test_model_gpu import TINY2
    return OracleWeights.random(TINY2, dtype=torch.bfloat16, seed=5, std=0.05)


def _sp(n, shift=0):
    from swiftllm_b200 import SamplingParams
    c = [SamplingParams(0.0, min_p=0.2), SamplingParams(0.8, seed=21, min_p=0.05),
         SamplingParams(1.3, seed=22, typical_p=0.9), SamplingParams(1.0, seed=23, xtc_threshold=0.02, xtc_probability=1.0),
         SamplingParams(1.0, top_k=40, top_p=0.95, seed=24, min_p=0.02, typical_p=0.8, xtc_probability=0.5),
         SamplingParams(0.9, seed=25)]
    return [c[(i + shift) % len(c)] for i in range(n)]


def _check(logits, toks, sp, pos):
    ref = TO.sample_tokens(logits, *[[getattr(s, f) for s in sp] for f in ("temperature", "top_k", "top_p")],
                           [s.seed for s in sp], pos,
                           *[[getattr(s, f) for s in sp] for f in ("min_p", "typical_p", "xtc_threshold", "xtc_probability")])
    for t, r in zip(toks, ref):
        assert t == r.token or r.gap <= 1e-5 * abs(r.score) or r.boundary_margin <= 1e-4, (t, r.token, r.gap)


def test_model_truncation_matches_the_restatement_eager_graph_and_chunked():
    from swiftllm_b200 import SamplingParams
    from test_model_gpu import _script
    w = _weights()
    eager, graph = _model(False, w), _model(True, w)
    rng = np.random.default_rng(2)
    prompts = _script(rng)
    sids = [3, 9, 0]
    sp = _sp(3)
    a = eager.forward(prompts, sids, [], sampling_params_list=sp)
    b = graph.forward(prompts, sids, [], sampling_params_list=sp)
    assert a == b
    _check(eager.post_layer.last_logits, a, sp, [len(p) for p in prompts])
    lens = [len(p) for p in prompts]
    for step in range(10):                              # decode: graph replay vs eager, both against the restatement
        lens = [l + 1 for l in lens]
        sp = _sp(3, step) if step % 3 else [SamplingParams(0.9, top_p=0.9, seed=40 + i) for i in range(3)]
        a = eager.forward([[t] for t in a], sids, lens, sampling_params_list=sp)
        b = graph.forward([[t] for t in b], sids, lens, sampling_params_list=sp)
        assert a == b
        assert torch.equal(eager.post_layer.last_logits, graph.post_layer.last_logits)
        _check(eager.post_layer.last_logits, a, sp, lens)
    tags = {k[2:] for k in graph._graphs}
    assert (True, False) in tags and (True, False, "truncated") in tags, tags
    # log-probabilities stay those of the raw logits
    lens = [l + 1 for l in lens]
    sp = [SamplingParams(1.0, seed=7 + i, min_p=0.1, typical_p=0.9, logprobs=2) for i in range(3)]
    res = eager.forward_with_logprobs([[t] for t in a], sids, lens, sampling_params_list=sp)
    graph.forward([[t] for t in a], sids, lens, sampling_params_list=sp)             # keep the graph model's cache in step
    raw = torch.log_softmax(eager.post_layer.last_logits.float(), dim=1)
    for i, r in enumerate(res):
        assert abs(r.logprob - float(raw[i, r.token])) <= 1e-3
    _check(eager.post_layer.last_logits, [r.token for r in res], sp, lens)
    # an allowed-token mask with XTC at threshold 0: the least likely ALLOWED token, never a masked one (eager and graph)
    from swiftllm_b200 import token_mask
    V = eager.model_config.vocab_size
    allowed = [5, 17, 200, 311]
    sp = [SamplingParams(1.0, seed=70 + i, xtc_threshold=0.0, xtc_probability=1.0) for i in range(3)]
    for m in (eager, graph):
        t = m.forward([[r.token] for r in res], sids, [l + 1 for l in lens], sampling_params_list=sp,
                      token_masks_list=[token_mask(V, allowed)] * 3)
        lg = m.post_layer.last_logits.float()[:, allowed]
        for i in range(3):                                   # the least likely allowed id (any of them if tied)
            assert t[i] in [allowed[j] for j in torch.nonzero(lg[i] == lg[i].min()).flatten().tolist()], (i, t[i], lg[i])
    lens = [l + 1 for l in lens]
    # chunked prefill of a new prompt with the decodes
    p4 = rng.integers(0, 512, size=50).tolist()
    eager.forward([p4[:20]], [5], [], prefill_prefix_lens_list=[0])
    lens = [l + 1 for l in lens]
    sp = _sp(4, 1)
    t = eager.forward([p4[20:50]] + [[r.token] for r in res], [5] + sids, lens, prefill_prefix_lens_list=[20],
                      sampling_params_list=sp)
    _check(eager.post_layer.last_logits, t, sp, [50] + lens)


def test_forward_speculative_returns_the_plain_decode_tokens():
    """Every row of a speculative entry is drawn like a plain decode step at its position, filters included: the returned
    tokens are the restatement's tokens for the verification's own logits, accepted while the drafts agree."""
    from swiftllm_b200 import SamplingParams
    w = _weights()
    m = _model(False, w)
    prompt = list(range(3, 40))
    sp = [SamplingParams(1.0, seed=11, min_p=0.05, typical_p=0.9, xtc_threshold=0.05, xtc_probability=0.5)]
    first = m.forward([prompt], [1], [], sampling_params_list=sp)
    L = len(prompt)
    for k in (3, 5):
        drafts = rng_drafts = [int(x) for x in np.random.default_rng(k).integers(0, 512, size=k)]
        out = m.forward_speculative([[first[-1]] + rng_drafts], [1], [L], sampling_params_list=sp)[0]
        logits = m.post_layer.last_logits
        ref = TO.sample_tokens(logits, [1.0] * (k + 1), [0] * (k + 1), [1.0] * (k + 1), [11] * (k + 1),
                               [L + j + 1 for j in range(k + 1)], [0.05] * (k + 1), [0.9] * (k + 1), [0.05] * (k + 1),
                               [0.5] * (k + 1))
        y = [r.token for r in ref]
        n = 0
        while n < k and drafts[n] == y[n]:
            n += 1
        if all(r.boundary_margin > 1e-4 and r.gap > 1e-5 * abs(r.score) for r in ref[:n + 1]):
            assert out == y[:n + 1], (out, y)
        L += len(out)
        first = out


def _tp_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    import swiftllm_b200
    from swiftllm_b200 import SamplingParams
    from swiftllm_b200.worker.weight import synthetic_getter
    from test_tp_gpu import CFG
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    out = []
    for graph in (False, True):
        ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=2,
                                        max_seqs_in_block_table=8, max_blocks_per_seq=16, max_batch_size=4, max_tokens_in_batch=256,
                                        dtype="bfloat16", tp_size=world, tp_rank=rank, use_cuda_graph=graph, shard_lm_head=True)
        m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(CFG))
        m.load_weights(synthetic_getter(seed=11, std=0.05, device=f"cuda:{rank}"))
        m.init_kvcache_and_swap(40)
        toks = m.forward([[1, 2, 3, 4, 5], [7, 8], [9] * 20], [0, 1, 2], [], sampling_params_list=_sp(3, 1))
        seq = [toks]
        lens = [5, 2, 20]
        for step in range(6):                               # even steps truncate (gathered rows), odd ones exchange pairs
            lens = [l + 1 for l in lens]
            sp = _sp(3, step) if step % 2 == 0 else [SamplingParams(0.9, seed=5 + i) for i in range(3)]
            toks = m.forward([[t] for t in toks], [0, 1, 2], lens, sampling_params_list=sp)
            seq.append(toks)
        out.append(seq)
    got = [None] * world
    dist.all_gather_object(got, out)
    if rank == 0:
        q.put(got)
    dist.destroy_process_group()


def test_tensor_parallel_ranks_return_identical_truncated_tokens():
    """Two GPUs, vocabulary-sharded lm_head: every rank returns the same tokens with min-p / typical-p / XTC rows (which
    gather the full rows) and without them (pair exchange), eager and graph-replayed."""
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_tp_worker, args=(r, 2, 29937, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        got = q.get(timeout=420)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.exitcode is None:
                p.kill()
    assert all(p.exitcode == 0 for p in procs)
    assert got[0] == got[1]
