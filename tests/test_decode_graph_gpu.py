"""GPU: pure-decode steps replayed from CUDA graphs (LlamaModel._forward_decode_graph) at long, ragged lengths, against the
fp64 definition of attention and against the eager path.

A decode graph plans attention for a length bucket, not for the batch: it is captured with max_decoding_len =
ceil(max_len / 1024) * 1024 and kept under the key (B, bucket if the launch splits else 0), at most max_cuda_graphs of them.
So a replay can run a different split length than the eager step would (csrc/paged_attn.cu, choose_split_tokens), extra
splits that are empty for every row, or a graph captured at a few hundred tokens at thousands of tokens.

Each scenario runs an eager model and a graph model with the same weights (Llama-3 heads: 32 q / 8 kv heads of 128, two
layers) and the same N(0, 1) cache, feeds both the eager model's tokens and asserts after every step:
  * equal block tables and allocation counts;
  * every (sequence, head) of every layer's attention output inside the graph (copied out by captured copies) within
    tests/attention_check.py's tolerance of fp64, on the sequence's pages read back from the cache;
  * where the eager and the graph launch use the same split length (restated below and held to the library's workspace
    size): logits, attention outputs and caches bit-identical.  Where they do not: the same greedy token wherever eager's
    top-1 margin exceeds twice the observed logit difference, and the eager attention output also within tolerance of fp64."""
import collections

import numpy as np
import pytest
import torch

from attention_check import check_attention
from oracle import kernels as K
from oracle.model import OracleWeights
from test_kernels_gpu import paged_gen  # noqa: F401 (fixture)
from test_model_gpu import _hf_tensors

pytestmark = pytest.mark.gpu
DEV = "cuda"
BS, D, NQ, NKV, LAYERS = 16, 128, 32, 8, 2
CFG = dict(model_type="llama", num_hidden_layers=LAYERS, num_attention_heads=NQ, num_key_value_heads=NKV, hidden_size=NQ * D,
           vocab_size=1024, max_position_embeddings=10240, intermediate_size=1024, rope_theta=500000.0, rms_norm_eps=1e-5,
           hidden_act="silu")
PA_MAX_SPLIT_TOKENS = 16384


def split_tokens(B, max_len):
    """choose_split_tokens (csrc/paged_attn.cu) for 8 kv heads and a library-chosen split length."""
    pairs = B * NKV
    want = -(-6 * torch.cuda.get_device_properties(0).multi_processor_count // pairs)      # >= 6 work items per SM
    if want <= 1:
        return PA_MAX_SPLIT_TOKENS
    st = -(-max_len // want)
    return min(max(-(-st // 128) * 128, 256), PA_MAX_SPLIT_TOKENS)


def bucket(max_len):
    """max_decoding_len a decode graph is captured with (LlamaModel._forward_decode_graph)."""
    return -(-max_len // 1024) * 1024


def plans(B, max_len):
    """Split lengths of the eager launch (max_len) and of the graph launch (its bucket).  The restatement must ask for the
    workspace the library asks for at both lengths, so it cannot drift from choose_split_tokens."""
    from swiftllm_b200 import _lib
    out = []
    for n in (max_len, bucket(max_len)):
        st = split_tokens(B, n)
        ns = -(-n // st)
        ws = 0 if ns <= 1 else B * NQ * ns * (D + 1) * 4
        assert _lib.lib().sllm_paged_attention_workspace_bytes(B, NQ, D, n, 0, NKV) == ws, f"planner restatement at B={B}, {n}"
        out.append(st)
    return tuple(out)


@pytest.fixture(scope="module")
def weights():
    return OracleWeights.random(CFG, dtype=torch.bfloat16, seed=11, std=0.02)


def _make_model(w, graph, max_seqs, max_len, num_blocks, max_graphs):
    import swiftllm_b200
    from swiftllm_b200.worker.weight import dict_getter
    ec = swiftllm_b200.EngineConfig(model_path="", use_dummy=False, block_size=BS, gpu_mem_utilization=0.9, num_cpu_blocks=0,
                                    max_seqs_in_block_table=max_seqs, max_blocks_per_seq=-(-max_len // BS) + 8,
                                    max_batch_size=max_seqs, max_tokens_in_batch=max(max_seqs, 64), dtype="bfloat16",
                                    use_cuda_graph=graph, max_cuda_graphs=max_graphs)
    m = swiftllm_b200.LlamaModel(ec, swiftllm_b200.LlamaModelConfig(CFG))
    m.load_weights(dict_getter(_hf_tensors(w, CFG["intermediate_size"])))
    m.init_kvcache_and_swap(num_blocks)
    m.post_layer.keep_logits = True
    return m


class Pair:
    """An eager and a graph model over identical weights and caches.  paged_attention is wrapped so that, inside the graph
    model's captures, q and o of every layer are copied into static buffers (one set per batch size, allocated before any
    capture): every replay refreshes them.  The wrapper is keyed on the graph model's cache, so the warm-up against the
    scratch cache writes nothing; the eager model's q and o are cloned per call."""

    def __init__(self, w, monkeypatch, batch_sizes, seqs, max_len, max_graphs=16):
        from swiftllm_b200.worker.layers import transformer_layer as TL
        nblk = sum(-(-n // BS) for n in seqs) + 64
        self.eager = _make_model(w, False, len(seqs), max_len, nblk, max_graphs)
        self.graph = _make_model(w, True, len(seqs), max_len, nblk, max_graphs)
        g = torch.Generator(device=DEV).manual_seed(1234)
        chunk = max(1, nblk // 64)
        with torch.inference_mode():                         # the caches are inference tensors
            for s in range(0, nblk, chunk):                  # N(0, 1), as bench.py fills its cache
                self.eager.k_cache[s:s + chunk].normal_(generator=g)
                self.eager.v_cache[s:s + chunk].normal_(generator=g)
            self.graph.k_cache.copy_(self.eager.k_cache)
            self.graph.v_cache.copy_(self.eager.v_cache)
        self.bufs = {B: [(torch.empty(B, NQ, D, dtype=torch.bfloat16, device=DEV),
                          torch.empty(B, NQ * D, dtype=torch.bfloat16, device=DEV)) for _ in range(LAYERS)] for B in batch_sizes}
        self.eager_qo = {}
        graph_k, eager_k = self.graph.k_cache.data_ptr(), self.eager.k_cache.data_ptr()
        orig = TL.paged_attention

        def hooked(q, k_cache, v_cache, block_table, mcfg, ecfg, st, cur_layer, o):
            orig(q, k_cache, v_cache, block_table, mcfg, ecfg, st, cur_layer, o)
            if k_cache.data_ptr() == graph_k:
                qb, ob = self.bufs[q.shape[0]][cur_layer]
                qb.copy_(q); ob.copy_(o)
            elif k_cache.data_ptr() == eager_k:
                self.eager_qo[cur_layer] = (q.clone(), o.clone())
        monkeypatch.setattr(TL, "paged_attention", hooked)
        self.captures = []                                   # batch size of every capture, in order
        capture = self.graph._capture_decode_graph

        def counted(B, *a, **kw):
            self.captures.append(B)
            return capture(B, *a, **kw)
        self.graph._capture_decode_graph = counted

    def close(self):
        self.graph._graphs.clear()
        del self.eager, self.graph, self.bufs, self.eager_qo
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

    def step(self, ids, sids, lens, fp64=True, label=""):
        """One decode step of both models; returns whether the two attention plans coincided."""
        B = len(sids)
        a = self.eager.forward([[t] for t in ids], sids, lens)
        le = self.eager.post_layer.last_logits.clone()
        b = self.graph.forward([[t] for t in ids], sids, lens)
        lg = self.graph.post_layer.last_logits.clone()
        torch.cuda.synchronize()
        be, bg = self.eager.gpu_block_manager, self.graph.gpu_block_manager
        n = be.num_seq_allocated_blocks.cpu()
        assert torch.equal(n, bg.num_seq_allocated_blocks.cpu()), "allocation counts differ"
        assert be.num_free_blocks == bg.num_free_blocks
        bte, btg = be.block_table.cpu(), bg.block_table.cpu()
        for s in sids:
            assert torch.equal(bte[s, :n[s]], btg[s, :n[s]]), f"block table row {s} differs"
        st_e, st_g = plans(B, max(lens))
        what = f"decode graph B={B} bucket {bucket(max(lens))} split {st_g}{label}"
        if fp64:
            self.check_fp64(self.graph, [self.bufs[B][l] for l in range(LAYERS)], sids, lens, what)
        if st_e == st_g:
            assert a == b, "graph and eager tokens differ under the same plan"
            assert torch.equal(le, lg), "graph and eager logits differ under the same plan"
            for l in range(LAYERS):
                assert torch.equal(self.eager_qo[l][1], self.bufs[B][l][1]), f"layer {l}: attention output differs"
            self.assert_caches_equal()
        else:
            le, lg = le.float(), lg.float()
            diff = float((le - lg).abs().max())
            top2 = le.topk(2, dim=1).values
            clear = ((top2[:, 0] - top2[:, 1]) > 2 * diff).tolist()
            assert sum(clear) > 0
            for i, (x, y, c) in enumerate(zip(a, b, clear)):
                assert not c or x == y, f"row {i}: eager token {x}, graph token {y} (margin clear of 2 x {diff:.3g})"
            if fp64:
                self.check_fp64(self.eager, [self.eager_qo[l] for l in range(LAYERS)], sids, lens,
                                f"decode eager B={B} split {st_e}{label}")
        return st_e == st_g, a

    def assert_caches_equal(self):
        n = self.eager.k_cache.shape[0]
        c = max(1, n // 16)
        for s in range(0, n, c):
            assert torch.equal(self.eager.k_cache[s:s + c], self.graph.k_cache[s:s + c]), "K caches differ"
            assert torch.equal(self.eager.v_cache[s:s + c], self.graph.v_cache[s:s + c]), "V caches differ"

    @staticmethod
    def check_fp64(model, qo, sids, lens, what):
        """Every (sequence, head) of each layer's o against paged_attention_exact on that sequence's pages, gathered from the
        model's cache after the step into a compact cache with its own block table."""
        bt = model.gpu_block_manager.block_table
        npg = [-(-n // BS) for n in lens]
        ids = torch.cat([bt[s, :k] for s, k in zip(sids, npg)]).long()
        table = torch.full((len(sids), max(npg)), -1, dtype=torch.int32)
        off = 0
        for i, k in enumerate(npg):
            table[i, :k] = torch.arange(off, off + k, dtype=torch.int32); off += k
        for l, (q, o) in enumerate(qo):
            kc, vc = model.k_cache[ids, l:l + 1].cpu(), model.v_cache[ids, l:l + 1].cpu()
            o64 = K.paged_attention_exact(q.cpu(), kc, vc, table, range(len(sids)), lens, D ** -0.5, BS, 0)
            check_attention(o.cpu(), o64, NQ, lens, what=f"{what}, layer {l}")


@pytest.fixture
def make_pair(weights, monkeypatch):
    made = []

    def make(*a, **kw):
        made.append(Pair(weights, monkeypatch, *a, **kw))
        return made[-1]
    yield make
    for p in made:
        p.close()


def test_bench_regime_bucket_transition(make_pair):
    """bench.py's regime (B = 64, 8 kv heads: two items per (sequence, kv head)).  The longest row goes 4094 -> 4097: at
    4094-4096 the graph of bucket 4096 runs the eager plan (two splits of 2048); at 4097 a new graph is captured for bucket
    5120 (two splits of 2560) while eager runs two of 2176."""
    B, steps = 64, 4
    rng = np.random.default_rng(4094)
    lens0 = rng.integers(1, 4001, size=B)
    lens0[:8] = [4094, 1, 16, 17, 2047, 2048, 2049, 3071]
    lens0 = [int(x) for x in lens0]
    pair = make_pair([B], [n + steps for n in lens0], 4094 + steps)
    sids = list(range(B))
    ids = rng.integers(0, CFG["vocab_size"], size=B).tolist()
    same, ngraphs = [], []
    for k in range(steps):
        lens = [n + k for n in lens0]
        eq, ids = pair.step(ids, sids, lens, fp64=k in (0, steps - 2, steps - 1))
        same.append(eq)
        ngraphs.append(len(pair.graph._graphs))
    assert same == [True, True, True, False], same
    assert plans(B, 4097) == (2176, 2560) and plans(B, 4096) == (2048, 2048)
    assert ngraphs == [1, 1, 1, 2] and pair.captures == [B, B], (ngraphs, pair.captures)


def test_small_batch_empty_trailing_splits(make_pair, paged_gen):
    """B = 4: 256-token splits, so the graph of bucket 4096 runs 16 split items per (sequence, kv head), most of them empty
    for every row, and the merge must read only each row's own ceil(len / 256) partials.  The plans coincide at every step
    (the 256-token floor), across the longest row's 3072 -> 3073 bucket change and other rows' 1024 and 2048 edges, so every
    step is bit-identical to eager, caches included."""
    B, steps = 4, 6
    lens0 = [1021, 3069, 1800, 2046]
    pair = make_pair([B], [n + steps for n in lens0], 3069 + steps)
    sids = [2, 0, 3, 1]
    ids = [5, 600, 77, 1000]
    for k in range(steps):
        lens = [n + k for n in lens0]
        assert plans(B, max(lens)) == (256, 256)
        eq, ids = pair.step(ids, sids, lens)
        assert eq
    assert pair.captures == [B, B] and len(pair.graph._graphs) == 2      # buckets 3072 and 4096
    pair.assert_caches_equal()


def test_single_pass_key_reuse(make_pair):
    """Batch x kv heads >= 6 x SMs: the launch never splits, so the graph key is (B, 0) whatever the length.  A graph captured
    at a few hundred tokens is replayed unchanged for a batch whose longest row holds about 9000 tokens."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = -(-6 * sms // NKV) + 1
    rng = np.random.default_rng(B)
    short = rng.integers(100, 500, size=B).tolist()
    long_ = rng.integers(1, 400, size=B).tolist()
    long_[:6] = [9000, 1, 16, 17, 2049, 4097]
    steps = 2
    pair = make_pair([B], [n + steps for n in short + long_], 9000 + steps)
    ids = rng.integers(0, CFG["vocab_size"], size=B).tolist()
    for sids, lens0, tag in ((list(range(B)), short, "short"), (list(range(B, 2 * B)), long_, "long")):
        for k in range(steps):
            lens = [n + k for n in lens0]
            assert plans(B, max(lens)) == (PA_MAX_SPLIT_TOKENS, PA_MAX_SPLIT_TOKENS)
            eq, ids = pair.step(ids, sids, lens, label=f" ({tag} rows)")
            assert eq
            assert len(pair.graph._graphs) == 1 and pair.captures == [B], "the (B, 0) graph must be reused"
    assert list(pair.graph._graphs) == [(B, 0)]


def test_graph_eviction(make_pair):
    """max_cuda_graphs = 2 with batch sizes 3, 5 and 7 in turn: each step evicts the least recently used graph and captures
    its own again into the shared memory pool.  Every replay equals eager bit for bit (same plans: 256-token splits)."""
    sizes, rounds = (3, 5, 7), 3
    rng = np.random.default_rng(357)
    sids = {}
    for B in sizes:
        sids[B] = list(range(sum(len(v) for v in sids.values()), sum(len(v) for v in sids.values()) + B))
    lens0 = {B: rng.integers(200, 1000, size=B).tolist() for B in sizes}
    ids = {B: rng.integers(0, CFG["vocab_size"], size=B).tolist() for B in sizes}
    pair = make_pair(list(sizes), [n + rounds for B in sizes for n in lens0[B]], 1000 + rounds, max_graphs=2)
    for r in range(rounds):
        for B in sizes:
            lens = [n + r for n in lens0[B]]
            eq, ids[B] = pair.step(ids[B], sids[B], lens)
            assert eq
            assert len(pair.graph._graphs) <= 2
    counts = collections.Counter(pair.captures)
    assert all(counts[B] >= 2 for B in sizes), counts                   # every graph evicted and captured again
