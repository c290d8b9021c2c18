"""CPU: shared KV blocks (LlamaModel.fork_seqs) through the product's host path, with the fork, tail-copy and release kernels
replaced by their restatements in fork_oracle.py.

Block state is held to the restatement after every operation of random schedules; a forked sequence decodes exactly like a
sequence that prefilled the same prompt itself; invalid calls and writes into shared blocks raise before anything changes."""
import multiprocessing as mp
import os

import numpy as np
import pytest
import torch

import fork_oracle as FO
from cpu_shim import product_on_cpu
from oracle.model import OracleWeights
from test_host_path_cpu import CFG, _hf_tensors
from test_sampling_cpu import PATCH as SAMPLE_PATCH
from test_speculative_cpu import SPEC

CALLS = []


def _fork_stand_in(nsab, block_table, extra, src, dst, lens, block_size):
    CALLS.append("fork")
    FO.fork_rows(nsab.numpy(), block_table.numpy(), extra.numpy(), src.tolist(), dst.tolist(), lens.tolist(), block_size)


def _release_stand_in(nsab, block_table, is_free, extra, seq_ids, total_blocks=None):
    CALLS.append("release")
    ids = FO.release(nsab.numpy(), block_table.numpy(), is_free.numpy(), extra.numpy(), seq_ids.tolist())
    return None if total_blocks is None else torch.tensor(ids, dtype=torch.int32)


def _copy_tails_stand_in(k_cache, v_cache, token_cache, block_table, src, dst, lens, block_size):
    CALLS.append("copy_tails")
    FO.copy_tails(k_cache, v_cache, token_cache, block_table.numpy(), src.tolist(), dst.tolist(), lens.tolist(), block_size)


FORK = [("swiftllm_b200.worker.block_manager", "_fork_kernel", _fork_stand_in),
        ("swiftllm_b200.worker.block_manager", "_release_kernel", _release_stand_in),
        ("swiftllm_b200.worker.model", "copy_block_tails", _copy_tails_stand_in)]
PATCH = FORK + SPEC + SAMPLE_PATCH

BS = 16


def _model(w, num_blocks=40, num_cpu_blocks=16, max_seqs=12, mbps=8, **ec_kw):
    import swiftllm_b200
    from swiftllm_b200.worker.weight import dict_getter
    ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=BS, gpu_mem_utilization=0.9,
                                    num_cpu_blocks=num_cpu_blocks, max_seqs_in_block_table=max_seqs, max_blocks_per_seq=mbps,
                                    max_batch_size=8, max_tokens_in_batch=256, dtype="float16", **ec_kw)
    m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(CFG))
    m.load_weights(dict_getter(_hf_tensors(w, CFG["intermediate_size"])))
    m.init_kvcache_and_swap(num_blocks)
    m.post_layer.keep_logits = True
    return m


def _state(bm):
    return (bm.num_seq_allocated_blocks.clone(), bm.block_table.clone(), bm.is_block_free.clone(), bm.block_extra_refs.clone(),
            bm.num_free_blocks, bm._host_nsab.copy(), bm._host_shared.copy())


def _same_state(a, b):
    return all(np.array_equal(np.asarray(x), np.asarray(y)) if not isinstance(x, int) else x == y for x, y in zip(a, b))


def _check(bm, ob: FO.BlockState):
    """Device state, host mirror and the restatement agree (tables compared where they are defined)."""
    nsab = bm.num_seq_allocated_blocks.numpy()
    assert np.array_equal(nsab, ob.nsab) and np.array_equal(bm._host_nsab, ob.nsab)
    table = bm.block_table.numpy()
    for s, n in enumerate(ob.nsab.tolist()):
        assert table[s, :n].tolist() == ob.table[s, :n].tolist(), s
        assert bm._host_shared[s] == ob.shared(s), (s, bm._host_shared[s], ob.shared(s))
    assert np.array_equal(bm.is_block_free.numpy(), ob.is_free)
    assert np.array_equal(bm.block_extra_refs.numpy(), ob.extra)
    assert bm.num_free_blocks == int(bm.is_block_free.sum()) == int(ob.is_free.sum())
    ob.check_invariants()


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_random_schedules_match_the_restatement(seed):
    """Prefill, n-way forks (prefixes shorter than the parent, aligned and unaligned), decode steps, speculative steps with
    truncation, frees of several owners of one block in one call, swap out of one fork while its partners keep running, swap in:
    block state held to the restatement after every operation, on both managers."""
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=11, std=0.08)
    rng = np.random.default_rng(seed)
    with product_on_cpu(PATCH):
        m = _model(w)
        gpu, cpu = FO.BlockState(40, 12, 8, BS), FO.BlockState(16, 12, 8, BS)
        lens, last, where = {}, {}, {}          # cached tokens, next input, "gpu" / "cpu"
        forks = 0
        for i in range(50):
            free_rows = [s for s in range(12) if s not in lens]
            on_gpu = [s for s in lens if where[s] == "gpu"]
            op = ["prefill", "fork"][i] if i < 2 else rng.choice(["prefill", "fork", "fork", "decode", "spec", "free", "swap_out",
                                                                  "swap_in"])
            if op == "prefill" and free_rows and gpu.is_free.sum() >= 4:
                s = int(rng.choice(free_rows)); n = int(rng.integers(1, 50))
                last[s] = m.forward([rng.integers(0, 300, size=n).tolist()], [s], [])[0]
                gpu.allocate([s], [n]); lens[s] = n; where[s] = "gpu"
            elif op == "fork" and on_gpu and free_rows:
                srcs, dsts, ps = [], [], []
                k = int(rng.integers(1, min(4, len(free_rows)) + 1))
                for d in rng.choice(free_rows, size=k, replace=False).tolist():
                    s = int(rng.choice(on_gpu))
                    p = int(rng.choice([lens[s], max(1, lens[s] - int(rng.integers(0, 20))), (lens[s] // BS) * BS or lens[s]]))
                    srcs.append(s); dsts.append(d); ps.append(p)
                if sum(p % BS > 0 for p in ps) > gpu.is_free.sum():
                    continue
                m.fork_seqs(srcs, dsts, ps)
                gpu.fork(srcs, dsts, ps)
                forks += 1
                for s, d, p in zip(srcs, dsts, ps):
                    lens[d] = p; where[d] = "gpu"; last[d] = int(rng.integers(0, 300))
            elif op == "decode" and on_gpu:
                sids = rng.choice(on_gpu, size=int(rng.integers(1, len(on_gpu) + 1)), replace=False).tolist()
                if sum((lens[s] + 1 + BS - 1) // BS - (lens[s] + BS - 1) // BS for s in sids) > gpu.is_free.sum():
                    continue
                out = m.forward([[last[s]] for s in sids], sids, [lens[s] + 1 for s in sids])
                gpu.allocate(sids, [lens[s] + 1 for s in sids])
                for s, t in zip(sids, out):
                    lens[s] += 1; last[s] = t
            elif op == "spec" and on_gpu:
                s = int(rng.choice(on_gpu)); r = int(rng.integers(1, 9))
                if lens[s] + r > 8 * BS or gpu.is_free.sum() < 1:
                    continue
                out = m.forward_speculative([[last[s]] + rng.integers(0, 300, size=r - 1).tolist()], [s], [lens[s]])[0]
                gpu.allocate([s], [lens[s] + r]); gpu.truncate([s], [lens[s] + len(out)])
                lens[s] += len(out); last[s] = out[-1]
            elif op == "free" and lens:
                sids = rng.choice(list(lens), size=int(rng.integers(1, len(lens) + 1)), replace=False).tolist()
                m.free_seqs_resources(sids)
                gpu.release(sids); cpu.release(sids)
                for s in sids:
                    del lens[s], where[s], last[s]
            elif op == "swap_out" and on_gpu:
                s = int(rng.choice(on_gpu)); n = int(gpu.nsab[s])
                if n > cpu.is_free.sum():
                    continue
                m.swap_out_seqs([s])
                gpu.release([s]); cpu.allocate([s], [n * BS]); where[s] = "cpu"
            elif op == "swap_in":
                out_ = [s for s in lens if where[s] == "cpu"]
                if not out_ or cpu.nsab[out_[0]] > gpu.is_free.sum():
                    continue
                s = out_[0]; n = int(cpu.nsab[s])
                m.swap_in_seqs([s])
                cpu.release([s]); gpu.allocate([s], [n * BS]); where[s] = "gpu"
            _check(m.gpu_block_manager, gpu)
            _check(m.cpu_block_manager, cpu)
        assert forks > 0
        m.free_seqs_resources(list(lens))
        gpu.release(list(lens)); cpu.release(list(lens))
        _check(m.gpu_block_manager, gpu)
        assert m.gpu_block_manager.num_free_blocks == 40 and not m.gpu_block_manager.block_extra_refs.any()


def test_n_way_fork_and_release_of_every_owner_in_one_call():
    """Five forks of one parent at an unaligned length: the full blocks gain five owners, each fork gets its own tail (lowest free
    ids, batch order) with the parent's tail pages; freeing all six in one call frees every block exactly once."""
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=2, std=0.08)
    with product_on_cpu(PATCH):
        m = _model(w)
        m.forward([list(range(1, 41))], [0], [])                  # 40 tokens: blocks 0, 1, 2 (tail of 8)
        with torch.inference_mode():
            m.token_cache[m.gpu_block_manager.block_table[0, 2]] = torch.arange(BS, dtype=torch.int32) + 7
        m.fork_seqs([0] * 5, [1, 2, 3, 4, 5], [40] * 5)
        bm = m.gpu_block_manager
        assert bm.block_extra_refs[:2].tolist() == [5, 5] and bm.block_extra_refs[2:].sum() == 0
        assert [bm.block_table[d, :3].tolist() for d in range(1, 6)] == [[0, 1, 3 + i] for i in range(5)]
        for d in range(1, 6):
            t = int(bm.block_table[d, 2])
            assert torch.equal(m.k_cache[t], m.k_cache[2]) and torch.equal(m.v_cache[t], m.v_cache[2])
            assert torch.equal(m.token_cache[t], m.token_cache[2])
        assert bm._host_shared[:6].tolist() == [2] * 6 and bm.num_free_blocks == 32
        m.free_seqs_resources([3, 0, 5, 1, 2, 4])
        assert bool(bm.is_block_free.all()) and not bm.block_extra_refs.any() and bm.num_free_blocks == 40
        assert not bm._rows and not bm._holders


def _prefill_pair(m, prompt, shared, sampled):
    """Seq 0 and seq 1 both hold `prompt`: forked (shared) or prefilled twice in calls of the same shape."""
    from swiftllm_b200 import SamplingParams
    sp = [SamplingParams(0.8, top_k=40, seed=5)] if sampled else None
    t0 = m.forward([prompt], [0], [], sampling_params_list=sp)[0]
    if shared:
        m.fork_seqs([0], [1], [len(prompt)])
        t1 = t0
    else:
        t1 = m.forward([prompt], [1], [], sampling_params_list=sp)[0]
    return [t0, t1]


@pytest.mark.parametrize("plen", [32, 37], ids=["aligned", "unaligned"])
@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "seeded"])
def test_forked_run_matches_an_unshared_run(plen, sampled):
    """The same decode steps after a fork and after prefilling the prompt twice: identical logits and tokens (distinct seeds per
    sequence), and identical block tables, up to the blocks the fork shares."""
    from swiftllm_b200 import SamplingParams
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=4, std=0.08)
    prompt = np.random.default_rng(1).integers(0, 300, size=plen).tolist()
    runs = []
    with product_on_cpu(PATCH):
        for shared in (True, False):
            m = _model(w)
            last = _prefill_pair(m, prompt, shared, sampled)
            L, toks, logits = plen, [], []
            for _ in range(20):
                L += 1
                sp = [SamplingParams(0.8, top_k=40, seed=10 + i) for i in range(2)] if sampled else None
                last = m.forward([[t] for t in last], [0, 1], [L, L], sampling_params_list=sp)
                toks.append(last); logits.append(m.post_layer.last_logits.clone())
            runs.append((toks, torch.stack(logits), m.gpu_block_manager))
    (ta, la, bma), (tb, lb, bmb) = runs
    assert ta == tb and torch.equal(la, lb)
    nb = (plen + 20 + BS - 1) // BS
    assert bma.num_free_blocks == bmb.num_free_blocks + plen // BS
    assert bma.block_table[0, :nb].tolist()[:plen // BS] == bma.block_table[1, :nb].tolist()[:plen // BS]


def test_chunked_prefill_and_speculative_steps_continue_a_fork():
    """A template holding a system prompt is forked; each fork continues by chunked prefill from the template's length and by
    speculative steps; tokens equal those of sequences that prefilled template + suffix themselves."""
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=6, std=0.08)
    rng = np.random.default_rng(4)
    system = rng.integers(0, 300, size=21).tolist()
    suffixes = [rng.integers(0, 300, size=n).tolist() for n in (5, 17)]
    drafts = [rng.integers(0, 300, size=3).tolist() for _ in suffixes]
    res = []
    with product_on_cpu(PATCH):
        for shared in (True, False):
            m = _model(w)
            m.forward([system], [0], [])
            if shared:
                m.fork_seqs([0, 0], [1, 2], [21, 21])
            else:                                # calls of the template's shape: the same K/V bits
                m.forward([system], [1], []); m.forward([system], [2], [])
            first = m.forward(suffixes, [1, 2], [], prefill_prefix_lens_list=[21, 21])
            out = m.forward_speculative([[t] + d for t, d in zip(first, drafts)], [1, 2], [21 + len(s) for s in suffixes])
            res.append((first, out))
    assert res[0] == res[1]


def test_invalid_forks_raise_before_anything_changes():
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=3, std=0.08)
    with product_on_cpu(PATCH):
        m = _model(w, num_blocks=6, num_cpu_blocks=4)
        m.forward([list(range(20)), list(range(40))], [0, 1], [])       # 2 + 3 blocks, 1 free
        m.forward([list(range(5))], [2], [])                            # the last free block
        m.swap_out_seqs([2])
        m.forward([list(range(5))], [4], [])                            # the block seq 2 gave back
        gpu, cpu = m.gpu_block_manager, m.cpu_block_manager
        before = (_state(gpu), _state(cpu))
        bad = [
            ([0], [3, 4], [5]),                  # list lengths differ
            ([0], [3], [0]),                     # P < 1
            ([0], [3], [33]),                    # P > blocks(src) * bs
            ([5], [3], [4]),                     # src holds no blocks
            ([2], [3], [4]),                     # src swapped out
            ([0], [1], [4]),                     # dst holds GPU blocks
            ([0], [2], [4]),                     # dst holds CPU blocks
            ([0, 1], [3, 3], [4, 4]),            # dst repeats
            ([0, 3], [3, 6], [4, 4]),            # dst is also a src
            ([0], [12], [4]),                    # dst out of the table
            ([-1], [3], [4]),                    # src out of the table
        ]
        for args in bad:
            with pytest.raises(ValueError):
                m.fork_seqs(*args)
            assert _same_state(_state(gpu), before[0]) and _same_state(_state(cpu), before[1])
        with pytest.raises(RuntimeError, match="No enough free blocks available on GPU"):
            m.fork_seqs([0], [3], [17])          # a tail block, none free
        assert _same_state(_state(gpu), before[0]) and _same_state(_state(cpu), before[1])
        assert not gpu.forked
        m.fork_seqs([0], [3], [16])              # aligned: no tail needed
        assert gpu.block_table[3, 0] == gpu.block_table[0, 0] and gpu.num_free_blocks == 0


def test_writes_into_shared_blocks_are_rejected_on_every_step_path():
    """Eager steps (prefill over a shared prefix, chunked prefill into it, decode at a shared position), the graph-replayed decode
    path and speculative steps raise ValueError before anything changes; continuing past the shared prefix is allowed."""
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=3, std=0.08)
    with product_on_cpu(PATCH):
        for graph in (False, True):
            m = _model(w, use_cuda_graph=graph)
            m.forward([list(range(40))], [0], [])
            m.fork_seqs([0, 0], [1, 2], [40, 32])
            bm = m.gpu_block_manager
            before = _state(bm)
            for call in [lambda: m.forward([[1]], [0], [32]),                       # position 31: block 1, shared
                         lambda: m.forward([[1]], [2], [32]),
                         lambda: m.forward([[1, 2]], [1], [], prefill_prefix_lens_list=[30]),
                         lambda: m.forward([list(range(8))], [1], []),
                         lambda: m.forward_speculative([[1, 2]], [2], [31])]:
                with pytest.raises(ValueError, match="shares with a fork"):
                    call()
                assert _same_state(_state(bm), before)
            if not graph:                        # the graph path itself needs a device; its check runs before the capture
                m.forward([[1], [2]], [1, 2], [41, 33])
                m.forward_speculative([[1, 2, 3]], [0], [40])


def test_a_run_without_fork_stages_and_launches_what_it_did_before():
    """No fork: the release and gather of the parent's kernels run (the new wrappers never), nothing is checked per step, and
    the staged metadata of each step is the parent's (the per-step check adds no words)."""
    import swiftllm_b200.worker.model as model_mod
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=3, std=0.08)
    staged = []
    with product_on_cpu(PATCH):
        m = _model(w)
        orig = m._stage_metadata
        m._stage_metadata = lambda *parts: (staged.append([list(p) for p in parts]), orig(*parts))[1]
        CALLS.clear()
        t0 = m.forward([list(range(20)), list(range(7))], [0, 1], [])
        t1 = m.forward([[x] for x in t0], [0, 1], [21, 8])
        m.forward_speculative([[t1[0], 3]], [0], [21])
        m.swap_out_seqs([1]); m.swap_in_seqs([1])
        m.free_seqs_resources([0, 1])
        assert CALLS == [] and not m.gpu_block_manager.forked and model_mod.copy_block_tails is _copy_tails_stand_in
        assert [len(s) for s in staged] == [8, 8, 9]
        assert staged[1] == [t0, [0, 1], [21, 8], [], [], [20, 7], [0, 1], []]
        assert bool(m.gpu_block_manager.is_block_free.all()) and not m.gpu_block_manager.block_extra_refs.any()


def test_offline_example_parallel_sampling():
    """examples/offline.py --n 3: each prompt prefilled once and forked twice; with a fixed seed the three samples use seeds s,
    s + 1, s + 2 and differ; greedy samples are identical; --n 1 output is unchanged."""
    import importlib.util
    from swiftllm_b200 import SamplingParams
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("offline_example", os.path.join(root, "examples", "offline.py"))
    ex = importlib.util.module_from_spec(spec); spec.loader.exec_module(ex)
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=5, std=0.08)
    prompts = [[7, 8, 9, 10] * 5, [3, 1, 4, 1, 5, 9, 2, 6]]
    with product_on_cpu(PATCH):
        g1, _, _ = ex.generate(_model(w), prompts, 8)
        g3, _, _ = ex.generate(_model(w), prompts, 8, n=3)
        assert g3[:2] == g1 and g3[2] == g3[3] == g1[0] and g3[4] == g3[5] == g1[1]
        sp = SamplingParams(1.0, seed=3)
        s3, _, _ = ex.generate(_model(w), prompts, 8, params=sp, n=3)
        s1, _, _ = ex.generate(_model(w), prompts, 8, params=sp)
        assert s3[:2] == s1 and len({tuple(s3[0]), tuple(s3[2]), tuple(s3[3])}) == 3
        m = _model(w)
        ex.generate(m, prompts, 8, params=sp, n=3)
        assert m.gpu_block_manager.forked


def test_parallel_samples_count_the_last_prompt_token_as_prompt():
    """Penalised n > 1 (examples/offline.py --n 3 with frequency and presence penalties): each fork draws its first token after
    a one-token prefill chunk of the last prompt token, so its history is the parent's bit for bit (every prompt token without
    the output flag: frequency / presence penalties see no output yet), and its penalised first-step logits are the prompt's own
    prefill row, penalised with the same history, to the chunked-vs-whole-prompt tolerance."""
    import importlib.util
    import penalties_oracle as PO
    from swiftllm_b200 import SamplingParams
    from test_penalties_cpu import PATCH as PEN_PATCH
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("offline_example", os.path.join(root, "examples", "offline.py"))
    ex = importlib.util.module_from_spec(spec); spec.loader.exec_module(ex)
    w = OracleWeights.random(CFG, dtype=torch.float16, seed=8, std=0.08)
    prompt = [5, 9, 5, 17, 9, 5, 40] * 3                                  # 21 tokens: the forks copy a partial tail
    sp = SamplingParams(0.0, repetition_penalty=1.2, frequency_penalty=1.5, presence_penalty=1.0)
    hist = [(t, False) for t in prompt]
    with product_on_cpu(FORK + SPEC + PEN_PATCH):
        m = _model(w)
        ex.generate(m, [prompt], 1, params=sp, n=3)                       # rows 1 and 2 fork row 0
        bt, tok = m.gpu_block_manager.block_table, m.token_cache
        pages = lambda s: [int(tok[int(bt[s, q // BS]), q % BS]) for q in range(len(prompt))]    # noqa: E731
        assert pages(0) == prompt and pages(1) == prompt and pages(2) == prompt

        m = _model(w)
        t0 = m.forward([prompt], [0], [], sampling_params_list=[sp])[0]
        want = PO.penalize_row(m.post_layer.last_logits[0], 1.2, 1.5, 1.0, hist)
        m.fork_seqs([0], [1], [len(prompt) - 1])
        t1 = m.forward([prompt[-1:]], [1], [], prefill_prefix_lens_list=[len(prompt) - 1], sampling_params_list=[sp])[0]
        got = PO.penalize_row(m.post_layer.last_logits[0], 1.2, 1.5, 1.0, hist)
        assert float((got - want).abs().max()) <= 2e-3 * float(want.abs().max())
        assert t1 == int(torch.argmax(got)) and t0 == int(torch.argmax(want))
        assert pages(1) == prompt


def _worker_tp(rank, world, port, ret):
    """fork + decode with tp_size=world on CPU (gloo collectives): the same tokens and block tables as tp 1."""
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import warnings
    import swiftllm_b200
    from swiftllm_b200.worker.weight import dict_getter
    cfg = dict(CFG, vocab_size=96)
    w = OracleWeights.random(cfg, dtype=torch.float16, seed=14, std=0.08)
    prompt = np.random.default_rng(8).integers(0, 96, size=37).tolist()

    def run(tp):
        with product_on_cpu(PATCH), warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=16, gpu_mem_utilization=0.9, num_cpu_blocks=4,
                                            max_seqs_in_block_table=8, max_blocks_per_seq=8, max_batch_size=8,
                                            max_tokens_in_batch=128, dtype="float16", tp_size=tp, tp_rank=rank if tp > 1 else 0,
                                            shard_lm_head=tp > 1)
            m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(cfg))
            m.load_weights(dict_getter(_hf_tensors(w, cfg["intermediate_size"])))
            m.init_kvcache_and_swap(20)
            t = m.forward([prompt], [0], [])
            m.fork_seqs([0, 0], [3, 5], [37, 30])
            last, lens, res = [t[0], t[0], 11], [37, 37, 30], [t]
            for _ in range(4):
                lens = [L + 1 for L in lens]
                last = m.forward([[x] for x in last], [0, 3, 5], lens)
                res.append(last)
            bm = m.gpu_block_manager
            return res, bm.block_table[[0, 3, 5], :3].tolist(), bm.block_extra_refs.tolist()

    sharded = run(world)
    gathered = [None] * world
    dist.all_gather_object(gathered, sharded)
    dist.destroy_process_group()
    if rank == 0:
        single = run(1)
        ret.put([g == single for g in gathered])


def test_fork_under_tensor_parallelism_on_cpu():
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_worker_tp, args=(r, 2, 29961, ret)) for r in range(2)]
    for p in procs:
        p.start()
    oks = ret.get(timeout=240)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(oks), oks
