"""GPU: multi-LoRA kernels (csrc/lora.cu) against the fp64 restatement (tests/lora_oracle.py), their batch invariance, the rows
and slices they must not touch, and the adapted model end to end: merged weights, CUDA-graph replay, speculative verification
and tensor parallelism."""
import os

import numpy as np
import pytest
import torch

import lora_oracle as LO
from test_lora_cpu import make_adapter, merged_weights

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _bits(t):
    return t.view(torch.int16)


def _pool(g, L, Rp, S, K, N, r, dtype, std=0.05):
    """Slot pools A [L, S * Rp, K] and B [L, N, Rp] with rank-r adapters (zero padding past r), scales and masks."""
    A = torch.zeros((L, S * Rp, K), dtype=dtype)
    B = torch.zeros((L, N, Rp), dtype=dtype)
    for a in range(L):
        for s in range(S):
            A[a, s * Rp:s * Rp + r] = (torch.randn((r, K), generator=g) * std).to(dtype)
        B[a, :, :r] = (torch.randn((N, r), generator=g) * std * 4).to(dtype)
    scales = (torch.rand(L, generator=g) * 2 + 0.25).float()
    return A.to(DEV), B.to(DEV), scales.to(DEV)


def _tiles(slots_rows):
    from swiftllm_b200.worker.lora import lora_tiles
    slots, rows = zip(*slots_rows)
    return torch.tensor(lora_tiles(list(slots), list(rows)), dtype=torch.int32, device=DEV).view(-1, 3)


def _row_slots(slots_rows):
    out = []
    for s, n in slots_rows:
        out += [s] * n
    return out


# runs of every length around TM = 64 (and around 16, the single-fragment path), base rows between, many distinct slots
RUNS = [(0, 1), (1, 15), (None, 2), (2, 16), (3, 17), (0, 63), (4, 64), (None, 1), (5, 65), (6, 1), (7, 1), (1, 1), (6, 3),
        (2, 128), (3, 20)]


@pytest.mark.parametrize("K", [4096, 14336])
@pytest.mark.parametrize("r", [8, 16, 32, 64])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_shrink_and_expand_against_fp64(dtype, r, K):
    from swiftllm_b200.worker.kernels.lora import lora_expand, lora_shrink
    g = torch.Generator().manual_seed(r + K)
    Rp, S, L = (r + 15) // 16 * 16, 3, 8
    n1, n2, N = 512, 768, 1024                         # q | k | v column slices
    A, B, scales = _pool(g, L, Rp, S, K, N, r, dtype)
    masks = torch.tensor([7, 7, 0b101, 7, 1, 0b110, 7, 7], dtype=torch.int32, device=DEV)
    T = sum(n for _, n in RUNS)
    wide = (torch.randn((T, K + 64), generator=g)).to(dtype).to(DEV)
    x = wide[:, 32:32 + K]                              # row-strided input, 16-byte aligned
    tiles = _tiles(RUNS)
    slots = _row_slots(RUNS)
    u = torch.full((T + 3, 3 * Rp), 7.0, dtype=dtype, device=DEV)
    y0 = (torch.randn((T, N), generator=g)).to(dtype).to(DEV)
    y0[::7, ::5] = -0.0
    y = y0.clone()
    lora_shrink(x, u, A, tiles, masks)
    lora_expand(y, u, B, (n1, n2), tiles, masks, scales)
    torch.cuda.synchronize()
    xc, uc, yc, y0c, Ac, Bc = x.cpu(), u.cpu(), y.cpu(), y0.cpu(), A.cpu(), B.cpu()
    ordered = {}
    for a in range(L):                                  # the shrink's reference in the kernel's order, all rows of slot a
        rows = [t for t, s in enumerate(slots) if s == a and int(masks[a]) != 0]
        if rows:
            ref, E = LO.shrink_ordered(xc[rows], Ac[a])
            ordered.update({t: (ref[i:i + 1], E[i:i + 1]) for i, t in enumerate(rows)})
    for t, a in enumerate(slots):
        if a is None or int(masks[a]) == 0:
            assert torch.equal(_bits(uc[t]), _bits(torch.full((3 * Rp,), 7.0, dtype=dtype))), t
            assert torch.equal(_bits(yc[t]), _bits(y0c[t])), t
            continue
        ok = LO.shrink_check(uc[t:t + 1, :S * Rp], *ordered[t])
        assert bool(ok.all()), (t, int((~ok).sum()))
        ref = LO.expand_exact(y0c[t:t + 1], uc[t:t + 1], Bc[a], float(scales[a]), (n1, n2), int(masks[a]), Rp)
        d = (yc[t:t + 1].double() - ref.double()).abs()
        bound = LO.expand_bound(y0c[t:t + 1], uc[t:t + 1], Bc[a], float(scales[a]), ref, Rp, (n1, n2), N)
        assert bool((d <= bound).all()), (t, float((d - bound).max()))
        for sl, (lo, hi) in enumerate(((0, n1), (n1, n2), (n2, N))):
            if not (int(masks[a]) >> sl) & 1:
                assert torch.equal(_bits(yc[t, lo:hi]), _bits(y0c[t, lo:hi])), (t, sl)
    assert torch.equal(_bits(uc[T:]), _bits(torch.full((3, 3 * Rp), 7.0, dtype=dtype)))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_a_rows_result_does_not_depend_on_its_batch(dtype):
    """The same x row and y row, alone, in a decode batch of 64 rows with other slots, and at every position of a 64-row and a
    200-row prefill run: u and y bit-identical (the LoRA kernels alone, fed the same x and y)."""
    from swiftllm_b200.worker.kernels.lora import lora_expand, lora_shrink
    g = torch.Generator().manual_seed(5)
    K, N, Rp, L = 4096, 14336 * 2 // 4, 64, 4
    A, B, scales = _pool(g, L, Rp, 2, K, N, 64, dtype)
    masks = torch.full((L,), 3, dtype=torch.int32, device=DEV)
    xr = torch.randn((1, K), generator=g).to(dtype).to(DEV)
    yr = torch.randn((1, N), generator=g).to(dtype).to(DEV)

    def run(T, runs, where):
        x = torch.randn((T, K), generator=g).to(dtype).to(DEV)
        y = torch.randn((T, N), generator=g).to(dtype).to(DEV)
        x[where] = xr[0]; y[where] = yr[0]
        u = torch.zeros((T, 3 * Rp), dtype=dtype, device=DEV)
        tiles = _tiles(runs)
        lora_shrink(x, u, A, tiles, masks)
        lora_expand(y, u, B, (N // 2, N), tiles, masks, scales)
        return u[where].clone(), y[where].clone()

    ref = run(1, [(2, 1)], 0)
    outs = [run(64, [((i % 3) if i != 37 else 2, 1) for i in range(64)], 37)]
    outs += [run(64, [(2, 64)], w) for w in (0, 15, 16, 31, 63)]
    outs += [run(200, [(0, 3), (2, 197)], w) for w in (3, 66, 130, 199)]
    outs += [run(70, [(1, 5), (2, 65)], w) for w in (5, 69)]
    for u, y in outs:
        assert torch.equal(_bits(u), _bits(ref[0])) and torch.equal(_bits(y), _bits(ref[1]))


def test_empty_tiles_and_untargeted_sites_leave_everything_untouched():
    from swiftllm_b200.worker.kernels.lora import lora_expand, lora_shrink
    g = torch.Generator().manual_seed(6)
    A, B, scales = _pool(g, 3, 16, 1, 1024, 1024, 16, torch.bfloat16)
    x = torch.randn((8, 1024), generator=g).to(torch.bfloat16).to(DEV)
    y = torch.randn((8, 1024), generator=g).to(torch.bfloat16).to(DEV)
    y[:, ::3] = -0.0
    y0 = y.clone()
    u = torch.full((8, 48), 3.0, dtype=torch.bfloat16, device=DEV)
    u0 = u.clone()
    tiles = torch.tensor([[0, 0, 0], [0, 8, 1], [2, 3, 2], [0, 0, 0], [5, 70, 0], [7, 2, 0], [0, 1, 9]], dtype=torch.int32,
                         device=DEV)                    # empty, untargeted slot, rows 0, too many rows, past T, bad slot
    masks = torch.tensor([1, 0, 0], dtype=torch.int32, device=DEV)
    lora_shrink(x, u, A, tiles, masks)
    lora_expand(y, u, B, (1024, 1024), tiles, masks, scales)
    assert torch.equal(_bits(u), _bits(u0)) and torch.equal(_bits(y), _bits(y0))


# ---------------------------------------------------------------- end to end on a small model
CFG = dict(model_type="llama", num_hidden_layers=2, num_attention_heads=8, num_key_value_heads=2, hidden_size=1024,
           vocab_size=512, max_position_embeddings=512, intermediate_size=1024, rope_theta=10000.0, rms_norm_eps=1e-5,
           hidden_act="silu")


def _model(w, **kw):
    import swiftllm_b200
    from swiftllm_b200.worker.weight import dict_getter
    from test_model_gpu import _hf_tensors
    ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=2,
                                    max_seqs_in_block_table=8, max_blocks_per_seq=16, max_batch_size=8, max_tokens_in_batch=256,
                                    dtype="float16", **kw)
    m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(CFG))
    m.load_weights(dict_getter({k: v.to(DEV) for k, v in _hf_tensors(w, CFG["intermediate_size"]).items()}))
    m.init_kvcache_and_swap(40)
    m.post_layer.keep_logits = True
    return m


ADAPTERS = {0: dict(r=16, seed=11), 3: dict(r=64, seed=12, modules=("q_proj", "v_proj", "o_proj", "down_proj"))}


def _adapters():
    return {s: make_adapter(CFG, std=0.03, **kw) for s, kw in ADAPTERS.items()}


def test_adapted_model_matches_merged_weights():
    """Two adapters and a base entry in one batch, prefill then decode: each adapted entry's logits against a second model loaded
    with that adapter merged into its weights; the base entry bit-identical to a run without lora_ids_list."""
    from oracle.model import OracleWeights
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=1, std=0.05)
    ads = _adapters()
    m, base = _model(w, max_loras=4, max_lora_rank=64), _model(w)
    for s, a in ads.items():
        m.load_lora(s, a)
    merged = {s: _model(merged_weights(w, CFG, a)) for s, a in ads.items()}
    rng = np.random.default_rng(1)
    prompts = [rng.integers(0, 512, size=n).tolist() for n in (40, 7, 129)]
    slots, sids = [0, None, 3], [5, 0, 2]
    ids, dec, lens = prompts, [], [len(p) for p in prompts]
    for step in range(5):
        toks = m.forward(ids, sids, dec, lora_ids_list=slots)
        base.forward(ids, sids, dec)
        got, b = m.post_layer.last_logits.float(), base.post_layer.last_logits.float()
        assert torch.equal(_bits(m.post_layer.last_logits[1]), _bits(base.post_layer.last_logits[1]))
        for s, mm in merged.items():
            t_ref = mm.forward(ids, sids, dec)
            r = slots.index(s)
            ref = mm.post_layer.last_logits[r].float()
            err, err_base = float((got[r] - ref).abs().max()), float((b[r] - ref).abs().max())
            assert err <= 0.25 * err_base and err <= 2 ** -7 * float(ref.abs().max()), (step, s, err, err_base)
            top2 = ref.topk(2).values
            if float(top2[0] - top2[1]) > 2 * err:
                assert toks[r] == t_ref[r], (step, s)
        lens = [l + 1 for l in lens]
        ids, dec = [[t] for t in toks], lens


def test_graph_replay_equals_the_eager_step_and_speculative_equals_plain_decoding():
    from oracle.model import OracleWeights
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=2, std=0.05)
    ads = _adapters()
    eager, graph, spec = (_model(w, max_loras=4, max_lora_rank=64, use_cuda_graph=g) for g in (False, True, False))
    for m in (eager, graph, spec):
        for s, a in ads.items():
            m.load_lora(s, a)
    rng = np.random.default_rng(2)
    prompts = [rng.integers(0, 512, size=n).tolist() for n in (33, 9, 70, 12)]
    sids = [1, 2, 3, 4]
    mixes = [[0, None, 3, 0], [None, None, None, None], [3, 3, 3, 3], [0, 3, None, 0], None]
    toks = eager.forward(prompts, sids, [], lora_ids_list=mixes[0])
    assert graph.forward(prompts, sids, [], lora_ids_list=mixes[0]) == toks
    lens = [len(p) for p in prompts]
    for step in range(10):
        mix = mixes[step % len(mixes)] if step < 5 else mixes[0]
        lens = [l + 1 for l in lens]
        ids = [[t] for t in toks]
        toks = eager.forward(ids, sids, lens, lora_ids_list=mix)
        tg = graph.forward(ids, sids, lens, lora_ids_list=mix)
        assert tg == toks, step
        assert torch.equal(_bits(graph.post_layer.last_logits), _bits(eager.post_layer.last_logits)), step
    keys = [k for k in graph._graphs]
    assert any(k[-1] == "lora" for k in keys) and any(k[-1] != "lora" for k in keys)
    # a grown u buffer: the adapted graph keeps reading the buffer it was captured with, which lives exactly as long as it
    import gc
    import weakref
    old = weakref.ref(graph.lora.u)
    graph.lora.ensure_rows(graph.lora.u.shape[0] + 64)
    assert graph.lora.u is not old() and any(t is old() for g in graph._graphs.values() for t in g["keep"])
    for step in range(3):
        lens = [l + 1 for l in lens]
        ids = [[t] for t in toks]
        toks = eager.forward(ids, sids, lens, lora_ids_list=mixes[3])
        assert graph.forward(ids, sids, lens, lora_ids_list=mixes[3]) == toks
        assert torch.equal(_bits(graph.post_layer.last_logits), _bits(eager.post_layer.last_logits)), step
    graph._graphs.clear()
    gc.collect()
    assert old() is None
    # speculative: drafts from plain adapted decoding (one replaced), the same tokens back
    p = rng.integers(0, 512, size=21).tolist()
    x = eager.forward([p], [6], [], lora_ids_list=[3])[0]
    assert spec.forward([p], [6], [], lora_ids_list=[3])[0] == x
    ys, inp = [], x
    for j in range(6):
        ys.append(eager.forward([[inp]], [6], [len(p) + j + 1], lora_ids_list=[3])[0])
        inp = ys[-1]
    out = spec.forward_speculative([[x] + ys[:5]], [6], [len(p)], lora_ids_list=[3])[0]
    assert out == ys
    drafts = list(ys[:5])
    drafts[2] = (drafts[2] + 1) % 512
    spec.free_seqs_resources([6])
    assert spec.forward([p], [6], [], lora_ids_list=[3])[0] == x
    assert spec.forward_speculative([[x] + drafts], [6], [len(p)], lora_ids_list=[3])[0] == ys[:3]


# ---------------------------------------------------------------- tensor parallelism (more than one GPU)
def _tp_run(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import swiftllm_b200
    from oracle.model import OracleWeights
    from swiftllm_b200.worker.weight import dict_getter
    from test_model_gpu import _hf_tensors
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=3, std=0.05)
    ads = _adapters()
    worst = 0.0
    for fused in (False, True):
        def make(tp, r):
            ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9,
                                            num_cpu_blocks=2, max_seqs_in_block_table=8, max_blocks_per_seq=16, max_batch_size=8,
                                            max_tokens_in_batch=256, dtype="float16", tp_size=tp, tp_rank=r,
                                            fused_allreduce=None if fused and tp > 1 else False, max_loras=4, max_lora_rank=64)
            m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(CFG))
            m.load_weights(dict_getter({k: v.to(f"cuda:{rank}") for k, v in _hf_tensors(w, CFG["intermediate_size"]).items()}))
            m.init_kvcache_and_swap(40)
            m.post_layer.keep_logits = True
            for s, a in ads.items():
                m.load_lora(s, a)
            return m
        tp = make(world, rank)
        ref = make(1, 0) if rank == 0 else None
        rng = np.random.default_rng(4)
        prompts = [rng.integers(0, 512, size=n).tolist() for n in (40, 7, 30)]
        sids, slots = [1, 2, 3], [0, None, 3]
        ids, dec, lens = prompts, [], [40, 7, 30]
        for step in range(4):
            t = tp.forward(ids, sids, dec, lora_ids_list=slots)
            if ref is not None:
                ref.forward(ids, sids, dec, lora_ids_list=slots)
                a, b = tp.post_layer.last_logits.float(), ref.post_layer.last_logits.float()
                worst = max(worst, float((a - b).abs().max() / b.abs().max()))
            lens = [l + 1 for l in lens]
            ids, dec = [[x] for x in t], lens
        torch.cuda.synchronize(); dist.barrier()
        del tp, ref
    if rank == 0:
        q.put(worst)
    import time
    time.sleep(0.5)
    os._exit(0)


def test_tensor_parallel_adapted_logits_match_single_gpu():
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_tp_run, args=(r, world, 29810, q)) for r in range(world)]
    for p in procs:
        p.start()
    worst = q.get(timeout=600)
    for p in procs:
        p.join(timeout=120)
    assert worst <= 2 ** -7, worst
