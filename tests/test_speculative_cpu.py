"""CPU: speculative decoding (LlamaModel.forward_speculative) through the product's host path with oracle-backed kernels.

The verify attention computes chunked-prefill attention for entries of 1..8 rows, so its stand-in is the chunked-prefill
restatement (oracle/kernels.py: prefix_prefill_attention_exact); block truncation has its restatement below.  The reference for
every row is the oracle fed the same rows one at a time as 1-token chunks: row j's logits are those of a plain decode step at
position prefix + j."""
import multiprocessing as mp
import os

import numpy as np
import pytest
import torch

import sampling_oracle as SO
from cpu_shim import _prefill_attention_paged, product_on_cpu
from oracle.model import OracleWeights
from test_host_path_cpu import CFG, ENG, _oracle, _product
from test_sampling_cpu import PATCH as SAMPLE_PATCH

BS = ENG["block_size"]


def _truncate(nsab, block_table, is_free, seq_ids, target_lens, block_size):
    """Restatement of sllm_truncate_blocks_for_seqs: entries [ceil(target / bs), allocated) of each row become free."""
    for sid, tl in zip(seq_ids.tolist(), target_lens.tolist()):
        n = int(nsab[sid])
        keep = min(n, (tl + block_size - 1) // block_size)
        is_free[block_table[sid, keep:n].long()] = True
        nsab[sid] = keep


SPEC = [("swiftllm_b200.worker.layers.transformer_layer", "paged_attention_verify", _prefill_attention_paged),
        ("swiftllm_b200.worker.block_manager", "_truncate_kernel", _truncate)]


def _oracle_rows(o, ids, sid, prefix):
    """Logits of every row of a speculative entry: the rows fed to the oracle one at a time."""
    out = []
    for j, t in enumerate(ids):
        o.forward([[t]], [sid], [], prefill_prefix_lens_list=[prefix + j])
        out.append(o.last_logits[0])
    return torch.stack(out)


def _accept(ids, y):
    n = 0
    while n < len(ids) - 1 and ids[n + 1] == y[n]:
        n += 1
    return y[:n + 1]


def _check_blocks(m, lens):
    """Each sequence holds ceil(len / bs) blocks (device and host mirror); the free map is exactly the complement of the tables."""
    bm = m.gpu_block_manager
    nsab = bm.num_seq_allocated_blocks.numpy()
    used = set()
    for sid, L in lens.items():
        want = (L + BS - 1) // BS
        assert nsab[sid] == want and bm._host_nsab[sid] == want, (sid, L, nsab[sid], bm._host_nsab[sid])
        used |= set(bm.block_table.numpy()[sid, :want].tolist())
    free = set(np.nonzero(bm.is_block_free.numpy())[0].tolist())
    assert free.isdisjoint(used) and len(free) + len(used) == bm.num_blocks
    assert bm.num_free_blocks == len(free)


def _greedy_plain(w, prompt, sid, n):
    """All-plain oracle run: the prompt's first token and n greedy decode tokens after it."""
    o = _oracle(w)
    toks = o.forward([prompt], [sid], [])
    for j in range(n):
        toks.append(o.forward([[toks[-1]]], [sid], [len(prompt) + j + 1])[0])
    return toks


@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "seeded-sampling"])
def test_speculative_rows_match_the_oracle_ragged_batch(sampled):
    """Eight entries of 1..8 rows in one call, prefixes on both sides of block boundaries (1, 3, 9, 12, 15, 16, 17, 30):
    per-row logits within the host-path tolerance of the oracle, each y_j the oracle's token for that row, the returned tokens
    the accepted prefix, and every sequence left with ceil(len / bs) blocks."""
    from swiftllm_b200 import SamplingParams
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=7, std=0.08)
    rng = np.random.default_rng(17)
    plens = [15, 16, 17, 1, 9, 30, 3, 12]
    sids = list(range(8))
    prompts = [rng.integers(0, 300, size=n).tolist() for n in plens]
    rows = [1, 2, 3, 4, 5, 6, 7, 8]
    with product_on_cpu(SPEC + SAMPLE_PATCH):
        m, o = _product(w), _oracle(w)
        first = m.forward(prompts, sids, [])
        assert first == o.forward(prompts, sids, [])
        entries = []
        for i, (p, x) in enumerate(zip(prompts, first)):
            if i % 2 == 0 and not sampled:        # the greedy continuation: every draft is accepted
                cont = _greedy_plain(w, p, sids[i], rows[i])
                assert cont[0] == x
                entries.append(cont[:rows[i]])
            else:
                entries.append([x] + rng.integers(0, 300, size=rows[i] - 1).tolist())
        params = [SamplingParams(0.9 if i % 3 else 0.0, top_k=(0, 20)[i % 2], seed=100 + i) for i in range(8)] if sampled else None
        out = m.forward_speculative(entries, sids, plens, params)
        ref = torch.cat([_oracle_rows(o, e, s, p) for e, s, p in zip(entries, sids, plens)])
        got = m.post_layer.last_logits
        assert got.shape == ref.shape
        # the oracle's one-row GEMMs round differently from the batched ones: the chunked-vs-whole-prompt tolerance
        assert float((got - ref).abs().max()) <= 2e-3 * float(ref.abs().max())
        top2 = ref.float().topk(2, dim=1).values
        clear = (top2[:, 0] - top2[:, 1]) > 8e-3 * float(ref.abs().max())
        assert bool(clear.float().mean() > 0.8)
        assert torch.equal(torch.argmax(got, dim=1)[clear], torch.argmax(ref, dim=1)[clear])
        if sampled:
            rep = np.repeat(np.arange(8), rows)
            pos = [p + j + 1 for p, n in zip(plens, rows) for j in range(n)]
            res = SO.sample_tokens(got, [params[i].temperature for i in rep], [params[i].top_k for i in rep],
                                   [params[i].top_p for i in rep], [params[i].seed for i in rep], pos)
            y = [r.token for r in res]
        else:
            y = torch.argmax(got, dim=1).tolist()
        s = 0
        for e, r, got_i in zip(entries, rows, out):
            assert got_i == _accept(e, y[s:s + r])
            s += r
        if not sampled:                           # all k drafts accepted: k + 1 tokens, those of the plain run
            for i in (0, 2, 4, 6):
                assert out[i] == _greedy_plain(w, prompts[i], sids[i], rows[i])[1:]
        _check_blocks(m, {sid: p + len(t) for sid, p, t in zip(sids, plens, out)})


def test_draft_wrong_at_index_m_accepts_exactly_m_and_plain_decoding_continues():
    """Drafts taken from the all-plain greedy run, with draft m + 1 replaced: exactly m drafts are accepted, every returned token
    is the plain run's, and alternating speculative and plain steps reproduce the plain run's tokens to the end."""
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=5, std=0.08)
    rng = np.random.default_rng(3)
    prompt = rng.integers(0, 300, size=14).tolist()
    sid = 3
    N = 40
    plain = _greedy_plain(w, prompt, sid, N)            # plain[0] after the prompt, plain[k] after k decode steps
    with product_on_cpu(SPEC):
        m = _product(w)
        got = m.forward([prompt], [sid], [])
        L = len(prompt)                                 # cached tokens; got[-1] is the next input
        schedule = [(7, 3), (7, 7), (2, 0), (5, 1), (0, 0), (3, None), (6, 6), (4, 2)]
        for k, wrong in schedule:
            x = got[-1]
            drafts = plain[len(got):len(got) + k]
            if wrong is not None and wrong < k:
                drafts[wrong] = (drafts[wrong] + 1) % 300
            out = m.forward_speculative([[x] + drafts], [sid], [L])[0]
            m_acc = min(wrong, k) if wrong is not None else k
            assert len(out) == m_acc + 1, (k, wrong, out)
            assert out == plain[len(got):len(got) + len(out)]
            got += out
            L += len(out)
            _check_blocks(m, {sid: L})
            t = m.forward([[got[-1]]], [sid], [L + 1])     # one plain step in between
            got += t
            L += 1
            _check_blocks(m, {sid: L})
        assert got == plain[:len(got)]


def test_rejected_inputs_raise_before_anything_changes():
    from swiftllm_b200 import SamplingParams
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=3, std=0.08)
    with product_on_cpu(SPEC):
        m = _product(w)
        t = m.forward([[1, 2, 3, 4, 5]], [2], [])
        bm = m.gpu_block_manager
        before = (bm.num_seq_allocated_blocks.clone(), bm.is_block_free.clone(), bm.num_free_blocks, bm._host_nsab.copy())
        max_pos = m._cos_cached.shape[0]
        bad = [
            dict(input_ids_list=[[]], seq_ids_list=[2], prefix_lens_list=[5]),
            dict(input_ids_list=[[t[0]] + [1] * 8], seq_ids_list=[2], prefix_lens_list=[5]),
            dict(input_ids_list=[[t[0], 1]], seq_ids_list=[2], prefix_lens_list=[-1]),
            dict(input_ids_list=[[t[0], 1, 2]], seq_ids_list=[2], prefix_lens_list=[max_pos - 2]),
            dict(input_ids_list=[[t[0]]], seq_ids_list=[2], prefix_lens_list=[5], ignore_kvcache=True),
            dict(input_ids_list=[[t[0], 1]], seq_ids_list=[2], prefix_lens_list=[5],
                 sampling_params_list=[SamplingParams(0.7, repetition_penalty=1.2)]),
            dict(input_ids_list=[[t[0], 1]], seq_ids_list=[2], prefix_lens_list=[5],
                 sampling_params_list=[SamplingParams(0.0, presence_penalty=0.5)]),
            dict(input_ids_list=[[t[0], 1]], seq_ids_list=[2], prefix_lens_list=[5], sampling_params_list=[SamplingParams(-1.0)]),
            dict(input_ids_list=[[t[0], 1]], seq_ids_list=[2, 3], prefix_lens_list=[5]),
        ]
        for kw in bad:
            with pytest.raises(ValueError):
                m.forward_speculative(**kw)
            assert torch.equal(bm.num_seq_allocated_blocks, before[0]) and torch.equal(bm.is_block_free, before[1])
            assert bm.num_free_blocks == before[2] and np.array_equal(bm._host_nsab, before[3])


def test_block_manager_truncation_frees_the_tail_lowest_first_reuse():
    from swiftllm_b200.worker.block_manager import BlockManager
    with product_on_cpu(SPEC):
        bm = BlockManager("GPU", 12, 4, 6, 16, device="cpu")
        sids = torch.tensor([0, 2], dtype=torch.int32)
        bm.allocate_blocks_for_seqs(sids, torch.tensor([70, 40], dtype=torch.int32), seq_ids_list=[0, 2], target_lens_list=[70, 40])
        assert bm.block_table[0, :5].tolist() == [0, 1, 2, 3, 4] and bm.block_table[2, :3].tolist() == [5, 6, 7]
        bm.truncate_blocks_for_seqs(sids, torch.tensor([33, 40], dtype=torch.int32), seq_ids_list=[0, 2], target_lens_list=[33, 40])
        assert bm.num_seq_allocated_blocks[[0, 2]].tolist() == [3, 3] and bm._host_nsab[[0, 2]].tolist() == [3, 3]
        assert bm.num_free_blocks == 6 and bm.is_block_free.tolist() == [False] * 3 + [True] * 2 + [False] * 3 + [True] * 4
        with pytest.raises(AssertionError, match="Logic error"):
            bm.truncate_blocks_for_seqs(sids[:1], torch.tensor([49], dtype=torch.int32), seq_ids_list=[0], target_lens_list=[49])
        new = bm.allocate_blocks_for_seqs(sids[1:], torch.tensor([64], dtype=torch.int32), seq_ids_list=[2], target_lens_list=[64])
        assert new.tolist() == [3]                     # freed ids come back lowest first


def test_offline_example_speculation_returns_the_plain_tokens():
    """examples/offline.py: generate() with --speculate (prompt-lookup drafts) returns the tokens of plain greedy decoding; the
    repetitive prompts make some drafts right."""
    import importlib.util
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("offline_example", os.path.join(root, "examples", "offline.py"))
    ex = importlib.util.module_from_spec(spec); spec.loader.exec_module(ex)
    assert ex.prompt_lookup([1, 2, 3, 9, 1, 2, 3], 3) == [9, 1, 2] and ex.prompt_lookup([5, 6, 7], 2) == []
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=5, std=0.08)
    prompts = [[7, 8, 9, 10] * 4, [3] * 9, [1, 2, 3, 4, 5]]
    with product_on_cpu(SPEC):
        a, _, _ = ex.generate(_product(w), prompts, 12)
        b, _, _ = ex.generate(_product(w), prompts, 12, speculate=4)
    assert a == b and all(len(o) == 12 for o in b)


def _worker_tp(rank, world, port, ret):
    """forward_speculative with tp_size=world on CPU (gloo collectives, vocabulary-sharded lm_head): the same tokens and block
    counts as the unsharded model."""
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import warnings
    import swiftllm_b200
    from swiftllm_b200.worker.weight import dict_getter
    from test_host_path_cpu import _hf_tensors
    cfg = dict(CFG, vocab_size=96)
    w = OracleWeights.random(cfg, dtype=torch.float16, seed=14, std=0.08)
    rng = np.random.default_rng(8)
    prompts = [rng.integers(0, 96, size=n).tolist() for n in (21, 3)]
    drafts = [rng.integers(0, 96, size=n).tolist() for n in (3, 7)]

    def run(tp):
        with product_on_cpu(SPEC), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=2,
                                            max_seqs_in_block_table=8, max_blocks_per_seq=8, max_batch_size=8,
                                            max_tokens_in_batch=128, dtype="float16", tp_size=tp, tp_rank=rank if tp > 1 else 0,
                                            shard_lm_head=tp > 1)
            m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(cfg))
            m.load_weights(dict_getter(_hf_tensors(w, cfg["intermediate_size"])))
            m.init_kvcache_and_swap(20)
            t = m.forward(prompts, [4, 1], [])
            res, lens, last = [t], [21, 3], t
            for _ in range(3):
                out = m.forward_speculative([[x] + d for x, d in zip(last, drafts)], [4, 1], lens)
                res.append(out)
                lens = [L + len(o) for L, o in zip(lens, out)]
                last = [o[-1] for o in out]
            return res, m.gpu_block_manager.get_num_allocated_blocks_host([4, 1])

    sharded = run(world)
    gathered = [None] * world
    dist.all_gather_object(gathered, sharded)
    dist.destroy_process_group()
    if rank == 0:
        single = run(1)
        ret.put([g == single for g in gathered])


def test_speculative_under_tensor_parallelism_on_cpu():
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_worker_tp, args=(r, 2, 29781, ret)) for r in range(2)]
    for p in procs:
        p.start()
    oks = ret.get(timeout=240)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(oks), oks
