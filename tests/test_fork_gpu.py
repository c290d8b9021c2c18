"""GPU: shared KV blocks - the fork, tail-copy and release kernels bit for bit against fork_oracle.py, and LlamaModel.fork_seqs end
to end: a forked sequence decodes exactly (logits and tokens) like a sequence that prefilled the same prompt itself."""
import numpy as np
import pytest
import torch

import fork_oracle as FO
from oracle.model import OracleWeights
from test_host_path_cpu import _hf_tensors
from test_model_gpu import TINY2

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _i32(x):
    return torch.tensor(list(x), dtype=torch.int32, device=DEV)


def _check(bm, ob):
    torch.cuda.synchronize()
    nsab = bm.num_seq_allocated_blocks.cpu().numpy()
    assert np.array_equal(nsab, ob.nsab) and np.array_equal(bm._host_nsab, ob.nsab)
    table = bm.block_table.cpu().numpy()
    for s, n in enumerate(ob.nsab.tolist()):
        assert table[s, :n].tolist() == ob.table[s, :n].tolist(), s
        assert bm._host_shared[s] == ob.shared(s)
    assert np.array_equal(bm.is_block_free.cpu().numpy(), ob.is_free)
    assert np.array_equal(bm.block_extra_refs.cpu().numpy(), ob.extra)
    assert bm.num_free_blocks == int(ob.is_free.sum())
    ob.check_invariants()


def test_fork_and_release_kernels_match_the_restatement():
    """Scattered block ids (allocations interleaved with frees), n-way forks of full and shorter prefixes, aligned and unaligned,
    then releases: plain, gathered, and every owner of a block in one launch; tables, counts, free map and extra owners equal the
    restatement after each call, and gathered ids are the restatement's."""
    from swiftllm_b200.worker.block_manager import BlockManager
    bs, NB, NS, MB = 16, 300, 64, 12
    bm, ob = BlockManager("GPU", NB, NS, MB, bs, device=DEV), FO.BlockState(NB, NS, MB, bs)
    rng = np.random.default_rng(0)
    lens = {s: int(rng.integers(1, MB * bs)) for s in range(12)}
    for s, L in lens.items():                     # interleave with frees so that rows hold scattered ids
        bm.allocate_blocks_for_seqs(_i32([s, 40 + s]), _i32([L, 40]), seq_ids_list=[s, 40 + s], target_lens_list=[L, 40])
        ob.allocate([s, 40 + s], [L, 40])
    filler = list(range(40, 52, 2))
    bm.free_blocks_for_seqs(_i32(filler), seq_ids_list=filler); ob.release(filler)
    _check(bm, ob)
    src, dst, P = [], [], []
    for d in range(12, 40):
        s = int(rng.integers(0, 12))
        src.append(s); dst.append(d)
        P.append(int(rng.choice([lens[s], (lens[s] // bs) * bs or lens[s], int(rng.integers(1, lens[s] + 1))])))
    src[:8] = [3] * 8                             # an 8-way fork in the same launch
    P[:8] = [lens[3]] * 4 + [max(1, lens[3] - 20)] * 4
    bm.fork_blocks_for_seqs(_i32(src), _i32(dst), _i32(P), src_seq_ids_list=src, dst_seq_ids_list=dst, lens_list=P)
    ob.fork(src, dst, P)
    _check(bm, ob)
    # a second generation: forks of forks
    bm.fork_blocks_for_seqs(_i32([12, 13]), _i32([52, 53]), _i32([P[0], 5]), src_seq_ids_list=[12, 13], dst_seq_ids_list=[52, 53],
                            lens_list=[P[0], 5])
    ob.fork([12, 13], [52, 53], [P[0], 5])
    _check(bm, ob)
    # the parent and all of its forks in one launch (concurrent release of every owner), plus a gathered release
    one = [3] + [d for s, d in zip(src, dst) if s == 3] + [52]
    bm.free_blocks_for_seqs(_i32(one), seq_ids_list=one); ob.release(one)
    _check(bm, ob)
    rest = [s for s in range(NS) if ob.nsab[s] > 0]
    order = rng.permutation(rest).tolist()
    got = bm.gather_allocated_blocks_and_free(_i32(order[:10]), seq_ids_list=order[:10])
    assert got.tolist() == ob.release(order[:10])
    _check(bm, ob)
    bm.free_blocks_for_seqs(_i32(order[10:]), seq_ids_list=order[10:]); ob.release(order[10:])
    _check(bm, ob)
    assert bool(bm.is_block_free.all()) and not bool(bm.block_extra_refs.any())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("head_dim", [128, 64])
@pytest.mark.parametrize("bs", [16, 32])
def test_copy_block_tails_bit_for_bit(dtype, head_dim, bs):
    """Random bit patterns in every page (NaN payloads included): the destination tail blocks become bit copies of the sources'
    (K, V and token pages), aligned entries and every other byte are untouched."""
    from swiftllm_b200.worker.kernels.block_mgmt import copy_block_tails
    L, nkv, NB, MB = 3, 2, 50, 6
    gen = torch.Generator().manual_seed(head_dim + bs)
    shape = (NB, L, nkv, bs, head_dim)
    k = torch.randint(-2 ** 15, 2 ** 15, shape, generator=gen, dtype=torch.int16).view(dtype)
    v = torch.randint(-2 ** 15, 2 ** 15, shape, generator=gen, dtype=torch.int16).view(dtype)
    tok = torch.randint(-2 ** 31, 2 ** 31 - 1, (NB, bs), generator=gen, dtype=torch.int32)
    table = torch.randperm(NB, generator=gen)[:8 * MB].reshape(8, MB).to(torch.int32)
    src, dst = [0, 0, 1, 2, 0], [3, 4, 5, 6, 7]
    P = [5 * bs + 3, 2 * bs, 1, bs - 1, 3 * bs + bs // 2]
    ek, ev, et = k.clone(), v.clone(), tok.clone()
    FO.copy_tails(ek, ev, et, table.numpy(), src, dst, P, bs)
    kd, vd, td = k.to(DEV), v.to(DEV), tok.to(DEV)
    copy_block_tails(kd, vd, td, table.to(DEV), _i32(src), _i32(dst), _i32(P), bs)
    torch.cuda.synchronize()
    assert torch.equal(kd.cpu().view(torch.int16), ek.view(torch.int16))
    assert torch.equal(vd.cpu().view(torch.int16), ev.view(torch.int16))
    assert torch.equal(td.cpu(), et)


# ------------------------------------------------------------------------------------------------ end to end
ENG = dict(block_size=16, num_cpu_blocks=16, max_seqs_in_block_table=16, max_blocks_per_seq=16, num_blocks=64)


def _model(w, dtype="bfloat16", graph=False, **ec_kw):
    import swiftllm_b200
    from swiftllm_b200.worker.weight import dict_getter
    ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=ENG["block_size"], gpu_mem_utilization=0.9,
                                    num_cpu_blocks=ENG["num_cpu_blocks"], max_seqs_in_block_table=ENG["max_seqs_in_block_table"],
                                    max_blocks_per_seq=ENG["max_blocks_per_seq"], max_batch_size=8, max_tokens_in_batch=256,
                                    dtype=dtype, use_cuda_graph=graph, **ec_kw)
    m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(TINY2))
    m.load_weights(dict_getter(_hf_tensors(w, TINY2["intermediate_size"])))
    m.init_kvcache_and_swap(ENG["num_blocks"])
    m.post_layer.keep_logits = True
    return m


_W = {}


def _weights():
    if "w" not in _W:
        _W["w"] = OracleWeights.random(TINY2, dtype=torch.bfloat16, seed=3, std=0.05)
    return _W["w"]


def _pair(m, prompt, shared, sp=None, n=1):
    """Sequences 0 .. n hold `prompt`: forked from 0, or each prefilled in a call of the same shape."""
    t = m.forward([prompt], [0], [], sampling_params_list=sp)[0]
    if shared:
        m.fork_seqs([0] * n, list(range(1, n + 1)), [len(prompt)] * n)
    else:
        for s in range(1, n + 1):
            assert m.forward([prompt], [s], [], sampling_params_list=sp)[0] == t
    return t


def _final_free(m):
    bm = m.gpu_block_manager
    m.free_seqs_resources(list(range(ENG["max_seqs_in_block_table"])))
    torch.cuda.synchronize()
    assert bool(bm.is_block_free.all()) and not bool(bm.block_extra_refs.any()) and bm.num_free_blocks == ENG["num_blocks"]


@pytest.mark.parametrize("plen", [48, 53], ids=["aligned", "unaligned"])
@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "seeded"])
@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_fork_decodes_like_an_unshared_prefill(plen, sampled, graph):
    """Prompt X prefilled into seq 0 and forked to seq 1, against X prefilled into seq 0 and seq 1 by calls of the same shape:
    the same decode steps give bit-identical logits and tokens, and the forked run's block state is the restatement's."""
    from swiftllm_b200 import SamplingParams
    w = _weights()
    X = np.random.default_rng(plen).integers(0, 1000, size=plen).tolist()
    sp = lambda: [SamplingParams(0.9, top_k=50, seed=7 + i) for i in range(2)] if sampled else None
    runs = []
    for shared in (True, False):
        m = _model(w, graph=graph)
        t = _pair(m, X, shared, None if not sampled else sp()[:1])
        last, L, toks, logits = [t, t], plen, [], []
        for _ in range(12):
            L += 1
            last = m.forward([[x] for x in last], [0, 1], [L, L], sampling_params_list=sp())
            toks.append(last)
            logits.append(m.post_layer.last_logits.clone())
        runs.append((toks, torch.stack(logits), m))
    (ta, la, ma), (tb, lb, _) = runs
    assert ta == tb
    assert torch.equal(la.view(torch.int16), lb.view(torch.int16))
    ob = FO.BlockState(ENG["num_blocks"], ENG["max_seqs_in_block_table"], ENG["max_blocks_per_seq"], ENG["block_size"])
    ob.allocate([0], [plen]); ob.fork([0], [1], [plen])
    for k in range(12):
        ob.allocate([0, 1], [plen + k + 1] * 2)
    _check(ma.gpu_block_manager, ob)
    _final_free(ma)


def test_speculative_steps_on_a_fork():
    """forward_speculative on a fork, with wrong drafts (rejection and truncation of private blocks): the unshared run's tokens,
    and the fork keeps its shared prefix."""
    w = _weights()
    X = np.random.default_rng(1).integers(0, 1000, size=45).tolist()
    res = []
    for shared in (True, False):
        m = _model(w)
        t = _pair(m, X, shared)
        L, last, out = 45, t, []
        for k in (7, 3, 5):
            drafts = [(last * 7 + j) % 1000 for j in range(k)]
            o = m.forward_speculative([[last] + drafts], [1], [L])[0]
            out.append(o); L += len(o); last = o[-1]
        out.append(m.forward([[last]], [1], [L + 1]))
        res.append(out)
        if shared:
            assert m.gpu_block_manager._host_shared[1] == 2 and m.gpu_block_manager.num_seq_allocated_blocks[1] == (L + 16) // 16
            _final_free(m)
    assert res[0] == res[1]


def test_chunked_prefill_from_a_forked_template():
    """A template (system prompt) forked to three sequences, each continued by two chunks of its own prompt and decode steps, against
    fresh sequences that prefilled the template in the same shape and the same chunks."""
    w = _weights()
    rng = np.random.default_rng(2)
    system = rng.integers(0, 1000, size=37).tolist()
    tails = [rng.integers(0, 1000, size=n).tolist() for n in (20, 9, 31)]
    res = []
    for shared in (True, False):
        m = _model(w)
        _pair(m, system, shared, n=3)
        sids = [1, 2, 3]
        half = [len(t) // 2 for t in tails]
        m.forward([t[:h] for t, h in zip(tails, half)], sids, [], prefill_prefix_lens_list=[37] * 3)
        last = m.forward([t[h:] for t, h in zip(tails, half)], sids, [], prefill_prefix_lens_list=[37 + h for h in half])
        lens = [37 + len(t) for t in tails]
        out = [last]
        for _ in range(6):
            lens = [x + 1 for x in lens]
            last = m.forward([[x] for x in last], sids, lens)
            out.append(last)
        res.append((out, m.post_layer.last_logits.clone()))
    assert res[0][0] == res[1][0] and torch.equal(res[0][1], res[1][1])


def test_penalised_decoding_inherits_the_history():
    """Penalties on a fork count the parent's prompt (the token page of the copied tail included): tokens equal the unshared run's."""
    from swiftllm_b200 import SamplingParams
    w = _weights()
    X = ([5, 6, 7, 8] * 10)[:37]
    sp = lambda n: [SamplingParams(0.0, repetition_penalty=1.3, frequency_penalty=0.4, presence_penalty=0.2)] * n
    res = []
    for shared in (True, False):
        m = _model(w)
        t = _pair(m, X, shared, sp(1))
        last, L, out = [t, t], 37, []
        for _ in range(10):
            L += 1
            last = m.forward([[x] for x in last], [0, 1], [L, L], sampling_params_list=sp(2))
            out.append(last)
        res.append(out)
    assert res[0] == res[1]


@pytest.mark.parametrize("path", ["host", "device", "copy_stream"])
def test_swapping_one_fork_out_and_back_mid_decode(path):
    """One of three forks is swapped out (its partners keep their shared blocks and keep decoding) and back in with private
    blocks: every sequence's tokens equal those of a run without the swap."""
    w = _weights()
    kw = dict(device_swap=path != "host", swap_on_copy_stream=path == "copy_stream")
    X = np.random.default_rng(3).integers(0, 1000, size=40).tolist()
    res = []
    for swap in (True, False):
        m = _model(w, **kw)
        t = _pair(m, X, True, n=2)
        last, L, out = [t] * 3, 40, []
        for k in range(8):
            L += 1
            if k == 3:                  # both runs split this step the same way: [0, 2], then [1]
                if swap:
                    m.swap_out_seqs([1])
                t02 = m.forward([[last[0]], [last[2]]], [0, 2], [L, L])
                if swap:
                    m.swap_in_seqs([1])
                    assert m.gpu_block_manager._host_shared[1] == 0 and m.gpu_block_manager._host_shared[0] == 2
                t1 = m.forward([[last[1]]], [1], [L])
                last = [t02[0], t1[0], t02[1]]
            else:
                last = m.forward([[x] for x in last], [0, 1, 2], [L] * 3)
            out.append(list(last))
        res.append(out)
        _final_free(m)
    assert res[0] == res[1]


def test_parallel_sampling_with_fresh_and_shared_seeds():
    """n = 8 forks of one prompt: seed None gives 8 different samples, one fixed seed gives 8 identical ones."""
    from swiftllm_b200 import SamplingParams
    w = _weights()
    X = np.random.default_rng(4).integers(0, 1000, size=29).tolist()
    for seed, distinct in ((None, 8), (12345, 1)):
        m = _model(w)
        m.forward([X], [0], [])
        m.fork_seqs([0] * 8, list(range(1, 9)), [28] * 8)          # each sample draws its own first token
        sids, L = list(range(1, 9)), 29
        sp = [SamplingParams(1.0, seed=seed)] * 8
        last = m.forward([[X[-1]]] * 8, sids, [], prefill_prefix_lens_list=[28] * 8, sampling_params_list=sp)
        out = [[x] for x in last]
        for _ in range(9):
            L += 1
            last = m.forward([[x] for x in last], sids, [L] * 8, sampling_params_list=sp)
            for o, x in zip(out, last):
                o.append(x)
        assert len({tuple(o) for o in out}) == distinct
        _final_free(m)


def test_penalised_samples_start_from_the_prompt_history():
    """The n > 1 recipe with penalties: forks at len - 1 continued by a one-token prefill chunk of the last prompt token.  Their
    token pages hold the prompt with no output flag, and their penalised tokens and raw logits equal, bit for bit, those of a
    sequence that prefilled the whole prompt itself and then took the same chunk."""
    from swiftllm_b200 import SamplingParams
    w = _weights()
    X = ([11, 23, 11, 57, 23, 11, 90] * 6)[:41]
    sp = lambda n: [SamplingParams(0.0, repetition_penalty=1.2, frequency_penalty=1.5, presence_penalty=1.0)] * n   # noqa: E731
    res = []
    for shared in (True, False):
        m = _model(w)
        m.forward([X], [0], [], sampling_params_list=sp(1))
        if shared:
            m.fork_seqs([0, 0], [1, 2], [40, 40])
        else:
            for s in (1, 2):
                m.forward([X], [s], [], sampling_params_list=sp(1))
        last = m.forward([X[-1:]] * 2, [1, 2], [], prefill_prefix_lens_list=[40, 40], sampling_params_list=sp(2))
        logits = [m.post_layer.last_logits.clone()]
        bt, tok = m.gpu_block_manager.block_table.cpu(), m.token_cache.cpu()
        for s in (1, 2):
            assert [int(tok[int(bt[s, q // 16]), q % 16]) for q in range(41)] == X
        out, L = [last], 41
        for _ in range(6):
            L += 1
            last = m.forward([[x] for x in last], [1, 2], [L, L], sampling_params_list=sp(2))
            out.append(last)
            logits.append(m.post_layer.last_logits.clone())
        res.append((out, torch.stack(logits)))
    assert res[0][0] == res[1][0]
    assert torch.equal(res[0][1].view(torch.int16), res[1][1].view(torch.int16))
