"""GPU: prefill attention, packed and chunked, at the lengths the project times and in the regimes where the kernels can
go wrong, every row of every (sequence, head) against the fp64 definition (tests/attention_check.py, the fp64 reference
evaluated on the device by tests/prefill64.py), both kernel generations wherever a shape is served by both:
  * packed prompts at the timed shapes (4 x 4096 in bench.py; 8 x 4096, 2 x 16384 and 32 x 1024 in
    scripts/prefill_bench.py), Llama-3-8B heads (32 q / 8 kv of 128);
  * one ragged batch: a 16384-token prompt, lengths at the 64- and 128-token step and block edges, and about 500 short
    prompts (grid.z in the hundreds, almost every CTA returns at once); bit-exact against each prompt run alone and
    against a second launch;
  * chunked prefill over a long prefix: every 2048-token chunk of a 16384-token prompt (and every 512-token chunk of a
    4096-token prompt, the SARATHI schedule) in one launch, bit-exact with the whole prompt's packed output; chunks of
    1 to 513 tokens after prefixes at page and step edges up to 16383;
  * rows dominated by one "sink" key and rows whose maximum ramps up by just under the wgmma kernel's lazy-rescale
    threshold per 64-key step, packed and chunked;
  * batch isolation: Inf or NaN in one prompt's Q, K or V (and in rows past the last prompt) leaves every other
    prompt's output bit-identical."""
import numpy as np
import pytest
import torch

import prefill64
from attention_check import check_attention
from oracle import kernels as K
from test_chunked_prefill_gpu import i32
from test_kernels_gpu import NS, prefill_gen  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda"
NQ, NKV, D, BS = 32, 8, 128, 16
G = NQ // NKV
SCALE = D ** -0.5
C = SCALE * K.LOG2E                      # raw score -> log2 units
ROWS_PER_CHECK = 16384                   # check_attention copies its arguments to the host in fp64


def _u(dtype):
    """Unit roundoff of the storage dtype."""
    return 2.0 ** -11 if dtype == torch.float16 else 2.0 ** -8


def _starts(lens):
    return [int(x) for x in np.cumsum([0] + list(lens[:-1]))]


def _randn(g, *shape):
    return torch.randn(*shape, generator=g, device=DEV)


def _packed(q, k, v, starts, lens):
    """sllm_prefill_attention on device tensors into a zeroed output."""
    from swiftllm_b200.worker.kernels.prefill_attn import prefill_attention
    st = NS(num_prefill_seqs=len(lens), prefill_seq_start_locs=i32(starts), prefill_seq_lens=i32(lens),
            max_prefill_len=int(max(lens)), softmax_scale=SCALE)
    o = torch.zeros(q.shape, dtype=q.dtype, device=DEV)
    prefill_attention(q, k, v, o, None, None, st)
    torch.cuda.synchronize()
    return o


def _chunked(q, kc, vc, bt, starts, chunk, prefix):
    """sllm_prefill_attention_paged (chunk i in block-table row i, layer 0) into a zeroed output."""
    from swiftllm_b200.worker.kernels.prefill_attn import prefill_attention_paged
    st = NS(num_prefill_seqs=len(chunk), seq_ids=i32(range(len(chunk))), prefill_seq_start_locs=i32(starts),
            prefill_seq_lens=i32(chunk), prefill_prefix_lens=i32(prefix), max_prefill_len=int(max(chunk)),
            softmax_scale=SCALE)
    o = torch.zeros(q.shape, dtype=q.dtype, device=DEV)
    prefill_attention_paged(q, kc, vc, bt, o, None, None, st, 0)
    torch.cuda.synchronize()
    return o


def _check(o, o64, starts, lens, prefix=None, what="prefill"):
    """check_attention over consecutive sequences, at most ROWS_PER_CHECK rows per call (a longer sequence alone)."""
    i = 0
    while i < len(lens):
        j, rows = i + 1, lens[i]
        while j < len(lens) and rows + lens[j] <= ROWS_PER_CHECK:
            rows += lens[j]; j += 1
        a = starts[i]
        assert starts[j - 1] + lens[j - 1] == a + rows, "sequences must be packed back to back"
        check_attention(o[a:a + rows], o64[a:a + rows], NQ, lens[i:j], starts=[s - a for s in starts[i:j]],
                        prefix=None if prefix is None else prefix[i:j], what=what)
        i = j


def _same_bits(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def _paged_cache(k, v, starts, lens, seed):
    """The sequences' K / V in paged caches [blocks, 1, NKV, BS, D] over randomly permuted blocks (sequence i in
    block-table row i, slots past each end zero); returns the caches and the device block table."""
    g = torch.Generator().manual_seed(seed)
    need = [-(-n // BS) for n in lens]
    perm = torch.randperm(sum(need), generator=g)
    bt = torch.full((len(lens), max(need) + 1), -1, dtype=torch.int32)
    kc = torch.zeros(sum(need), 1, NKV, BS, D, dtype=k.dtype, device=DEV)
    vc = torch.zeros_like(kc)
    p = 0
    for i, (s0, n) in enumerate(zip(starts, lens)):
        ids = perm[p:p + need[i]]; p += need[i]
        bt[i, :need[i]] = ids.to(torch.int32)
        for src, dst in ((k, kc), (v, vc)):
            pad = torch.zeros(need[i] * BS, NKV, D, dtype=k.dtype, device=DEV)
            pad[:n] = src[s0:s0 + n]
            dst[ids.to(DEV), 0] = pad.view(need[i], BS, NKV, D).transpose(1, 2)
    return kc, vc, bt.to(DEV)


# ----------------------------------------------------------------------------- long packed prompts
def _timed_case(B, L, dtype):
    g = torch.Generator(device=DEV).manual_seed(B * L)
    T = B * L
    q, k, v = (_randn(g, T, n, D).to(dtype) for n in (NQ, NKV, NKV))
    starts, lens = [s * L for s in range(B)], [L] * B
    return q, k, v, starts, lens, prefill64.prefill_attention(q, k, v, starts, lens, SCALE)


@pytest.mark.parametrize("dtype,B,L", [(torch.bfloat16, 4, 4096), (torch.bfloat16, 8, 4096), (torch.bfloat16, 2, 16384),
                                       (torch.float16, 2, 16384), (torch.bfloat16, 32, 1024)],
                         ids=["bf16-4x4096", "bf16-8x4096", "bf16-2x16384", "fp16-2x16384", "bf16-32x1024"])
def test_packed_timed_shapes(dtype, B, L, prefill_gen):
    """The prefill shapes the project times, every row: at 16384 tokens a CTA streams 256 K/V steps through its rings
    and its running max gets 256 chances to take or skip a rescale."""
    q, k, v, starts, lens, o64 = _timed_case(B, L, dtype)
    o = _packed(q, k, v, starts, lens)
    _check(o, o64, starts, lens)


def test_packed_ragged_batch(prefill_gen):
    """One 16384-token prompt, lengths at the 64-token step and 128-row block edges, and 500 prompts of 1-40 tokens
    (grid.z = 510 with 128 row blocks each: nearly every CTA returns at once).  Every row against fp64; a second launch
    gives the same bits, and so does each of several prompts run alone at row 0."""
    rng = np.random.default_rng(510)
    lens = [16384, 1, 63, 64, 65, 127, 128, 129, 4095, 4097] + rng.integers(1, 41, size=500).tolist()
    order = rng.permutation(len(lens))                          # the long prompts land at arbitrary start offsets
    lens = [37] + [int(lens[i]) for i in order]
    starts = _starts(lens)
    T = sum(lens)
    g = torch.Generator(device=DEV).manual_seed(T)
    q, k, v = (_randn(g, T, n, D).to(torch.bfloat16) for n in (NQ, NKV, NKV))
    o = _packed(q, k, v, starts, lens)
    _check(o, prefill64.prefill_attention(q, k, v, starts, lens, SCALE), starts, lens)
    assert _same_bits(o, _packed(q, k, v, starts, lens)), "two launches differ"
    for n in (16384, 4097, 129, 65, 1, lens[-1]):
        i = len(lens) - 1 if n == lens[-1] else lens.index(n)
        s0 = starts[i]
        alone = _packed(q[s0:s0 + n].contiguous(), k[s0:s0 + n].contiguous(), v[s0:s0 + n].contiguous(), [0], [n])
        assert _same_bits(alone, o[s0:s0 + n]), f"prompt {i} ({n} tokens at row {s0}) differs from the same prompt alone"


# ----------------------------------------------------------------------------- chunked prefill over long prefixes
@pytest.mark.parametrize("L,chunk", [(16384, 2048), (4096, 512)], ids=["16384-in-2048", "sarathi-4096-in-512"])
def test_chunked_every_chunk_of_a_long_prompt(L, chunk, prefill_gen):
    """A prompt stored with store_kvcache_chunked, then all its chunks in one launch as sequences whose block-table rows
    point at the same pages (chunk i at prefix chunk * i).  Every row against fp64, and bit-exact with the whole prompt
    through the packed kernel: with prefixes on 128-row boundaries both see the same keys in the same 64-key steps."""
    from swiftllm_b200.worker.kernels.kvcache_mgmt import store_kvcache
    n = L // chunk
    g = torch.Generator(device=DEV).manual_seed(L + chunk)
    q, k, v = (_randn(g, L, h, D).to(torch.bfloat16) for h in (NQ, NKV, NKV))
    npg = L // BS
    perm = torch.randperm(npg + 5, generator=torch.Generator().manual_seed(L))
    bt = torch.full((n, npg + 1), -1, dtype=torch.int32)
    bt[:, :npg] = perm[:npg].to(torch.int32)
    bt = bt.to(DEV)
    kc = torch.zeros(npg + 5, 1, NKV, BS, D, dtype=torch.bfloat16, device=DEV)
    vc = torch.zeros_like(kc)
    starts, chunks, prefix = [chunk * i for i in range(n)], [chunk] * n, [chunk * i for i in range(n)]
    st = NS(seq_ids=i32(range(n)), prefill_seq_start_locs=i32(starts), prefill_seq_lens=i32(chunks),
            decoding_seq_lens=i32([]), num_prefill_seqs=n, num_decoding_seqs=0, num_prefill_tokens=L, max_prefill_len=chunk,
            prefill_prefix_lens=i32(prefix))
    store_kvcache(k, v, kc, vc, bt, None, None, st, 0)
    o = _chunked(q, kc, vc, bt, starts, chunks, prefix)
    o64 = prefill64.prefix_prefill_attention(q, kc, vc, bt, range(n), starts, chunks, prefix, SCALE, BS, 0)
    _check(o, o64, starts, chunks, prefix, what="paged_prefill")
    assert _same_bits(o, _packed(q, k, v, [0], [L])), "chunked output differs from the whole prompt's"


def test_chunked_prefix_edges(prefill_gen):
    """Chunks of 1, 63, 64, 65 and 513 tokens after prefixes of 8191, 8192, 8193 and 16383 (page and 64-key step edges),
    all in one launch over one 16896-token cache whose pages every sequence shares."""
    prefixes, sizes = [8191, 8192, 8193, 16383], [1, 63, 64, 65, 513]
    prefix = [p for p in prefixes for _ in sizes]
    chunk = [c for _ in prefixes for c in sizes]
    L = max(p + c for p, c in zip(prefix, chunk))
    g = torch.Generator(device=DEV).manual_seed(L)
    k, v = (_randn(g, L, NKV, D).to(torch.bfloat16) for _ in range(2))
    kc, vc, bt1 = _paged_cache(k, v, [0], [L], seed=L)
    bt = bt1.expand(len(chunk), -1).contiguous()
    starts = _starts(chunk)
    q = _randn(g, sum(chunk), NQ, D).to(torch.bfloat16)
    o = _chunked(q, kc, vc, bt, starts, chunk, prefix)
    o64 = prefill64.prefix_prefill_attention(q, kc, vc, bt, range(len(chunk)), starts, chunk, prefix, SCALE, BS, 0)
    _check(o, o64, starts, chunk, prefix, what="paged_prefill")


# ----------------------------------------------------------------------------- sink keys and the lazy rescale
SINK_LENS = [300, 300, 300, 300, 300, 300, 300, 1000, 4097]
SINK_POS = [0, 63, 64, 127, 128, 233, 299, 970, 4096]     # key steps' edges, inside a diagonal step, last token, last step


def _chunks_of(lens, size):
    """The last `size` tokens of each sequence as a chunk after the rest: (prefix, chunk) lists."""
    chunk = [min(n, size) for n in lens]
    return [n - c for n, c in zip(lens, chunk)], chunk


def _run_mode(mode, q, k, v, lens, chunk_size, seed):
    """Run the packed kernel over the sequences, or the chunked kernel over their last chunk_size tokens (the earlier
    ones as the prefix in a paged cache).  Returns (o, o64, row -> (sequence, position) map as tensors, starts, lens,
    prefix) of the rows computed."""
    starts = _starts(lens)
    if mode == "packed":
        o = _packed(q, k, v, starts, lens)
        o64 = prefill64.prefill_attention(q, k, v, starts, lens, SCALE)
        return o, o64, starts, lens, None, list(range(sum(lens)))
    prefix, chunk = _chunks_of(lens, chunk_size)
    kc, vc, bt = _paged_cache(k, v, starts, lens, seed)
    rows = [s0 + p + t for s0, p, c in zip(starts, prefix, chunk) for t in range(c)]
    qc = q[torch.tensor(rows, device=DEV)].contiguous()
    cst = _starts(chunk)
    o = _chunked(qc, kc, vc, bt, cst, chunk, prefix)
    o64 = prefill64.prefix_prefill_attention(qc, kc, vc, bt, range(len(lens)), cst, chunk, prefix, SCALE, BS, 0)
    return o, o64, cst, chunk, prefix, rows


@pytest.mark.parametrize("mode", ["packed", "chunked"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_sink_keys(mode, dtype, prefill_gen):
    """Per (sequence, kv head) one key whose logit exceeds every other key's of the sequence by more than 150 (log2
    units) for every row that sees it: every other p is exactly 0 and those rows return the sink's V up to the output
    rounding.  Rows before the sink are ordinary.  Chunked: the last 160 tokens of each sequence after the rest."""
    B, T = len(SINK_LENS), sum(SINK_LENS)
    starts = _starts(SINK_LENS)
    g = torch.Generator(device=DEV).manual_seed(150)
    u = torch.randint(0, 2, (B, NKV, D), generator=g, device=DEV).float() * 2 - 1       # one +-1 direction per kv head
    k, v = _randn(g, T, NKV, D), _randn(g, T, NKV, D)
    per_row = torch.repeat_interleave(torch.arange(B, device=DEV), torch.tensor(SINK_LENS, device=DEV))
    q = 0.3 * _randn(g, T, NQ, D) + u.repeat_interleave(G, dim=1)[per_row]
    for s, j in enumerate(SINK_POS):
        k[starts[s] + j] = 16 * u[s]
    q, k, v = q.to(dtype), k.to(dtype), v.to(dtype)
    for s, (n, j) in enumerate(zip(SINK_LENS, SINK_POS)):          # the premise, against every key of the sequence
        s0 = starts[s]
        sc = torch.einsum("rhgd,nhd->hgrn", q[s0 + j:s0 + n].double().view(-1, NKV, G, D), k[s0:s0 + n].double()) * C
        others = torch.cat([sc[..., :j], sc[..., j + 1:]], dim=-1)
        assert float((sc[..., j] - others.amax(-1)).min()) > 150
    o, o64, cst, clens, prefix, rows = _run_mode(mode, q, k, v, SINK_LENS, 160, seed=151)
    _check(o, o64, cst, clens, prefix, what="prefill" if mode == "packed" else "paged_prefill")
    rows = torch.tensor(rows, device=DEV)                           # row of o -> row of the packed sequences
    seq = per_row[rows]
    first = torch.tensor(starts, device=DEV)[seq]
    sink_row = first + torch.tensor(SINK_POS, device=DEV)[seq]
    sees = rows >= sink_row
    assert int(sees.sum()) > 0
    vs = v[sink_row].float().repeat_interleave(G, dim=1)[sees]                              # [rows seeing it, NQ, D]
    got = o[sees].float()
    bad = (got - vs).abs() > _u(dtype) * vs.abs()
    assert not bad.any(), f"{int(bad.any(-1).any(-1).sum())} rows that see the sink do not return its V"


def _ramp_logits(n, offset, g):
    """Target logits (log2 units) of the keys of one sequence: a level that rises by 7.5 per 64 keys for 40 steps, then
    jumps by 9 and stays; within a step each key sits up to 2 below its level."""
    t = (torch.arange(n, device=DEV) + offset) // 64
    level = torch.where(t <= 40, 7.5 * t, 7.5 * 40 + 9.0)
    return level - 2 * torch.rand(n, generator=g, device=DEV)


@pytest.mark.parametrize("mode", ["packed", "chunked"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_lazy_rescale_ramp(mode, dtype, prefill_gen):
    """Rows whose maximum rises by about 7.5 (log2 units) per 64-key step for 40 steps, just under the wgmma kernel's
    rescale threshold of 8, then jumps by 9: its reference point trails the maximum by up to 8 at alternate steps (p
    up to 2^8, the largest weights rounded) and the jump forces a rescale after a skipped one.  Logits are exact by
    construction: q and k lie along one +-1 direction per kv head with small orthogonal noise.  One sequence has its
    ramp steps on the kernel's 64-key steps, one half a step off; chunked: the last 700 tokens after the rest."""
    lens = [64 * 44, 64 * 44 - 37]
    offsets = [0, 32]
    T = sum(lens)
    g = torch.Generator(device=DEV).manual_seed(75)
    qs, ks = [], []
    for n, off in zip(lens, offsets):
        u = torch.randint(0, 2, (NKV, D), generator=g, device=DEV).float() * 2 - 1
        uh = u.repeat_interleave(G, dim=0)

        def perp(x, uu):                                      # remove the component along the direction
            return x - (x * uu).sum(-1, keepdim=True) / D * uu
        a = torch.stack([_ramp_logits(n, off, g) for _ in range(NKV)], dim=1) / (C * D)        # [n, NKV]
        ks.append(a[..., None] * u + 0.1 * perp(_randn(g, n, NKV, D), u))
        qs.append(uh + 0.1 * perp(_randn(g, n, NQ, D), uh))
    q, k = torch.cat(qs).to(dtype), torch.cat(ks).to(dtype)
    v = _randn(g, T, NKV, D).to(dtype)
    # the premise: the last row's step maxima rise by 7-8 per step, then jump by 8.5-9.5 (aligned sequence)
    sc = torch.einsum("hgd,nhd->hgn", q[lens[0] - 1].double().view(NKV, G, D), k[:lens[0]].double()) * C
    rise = sc.view(NKV, G, 44, 64).amax(-1).diff(dim=-1)
    assert float(rise[..., :40].min()) > 7 and float(rise[..., :40].max()) < 8, rise[..., :40]
    assert float(rise[..., 40].min()) > 8.5 and float(rise[..., 40].max()) < 9.5, rise[..., 40]
    o, o64, cst, clens, prefix, _ = _run_mode(mode, q, k, v, lens, 700, seed=76)
    _check(o, o64, cst, clens, prefix, what="prefill" if mode == "packed" else "paged_prefill")


# ----------------------------------------------------------------------------- batch isolation
@pytest.mark.parametrize("value", [float("inf"), float("-inf"), float("nan")], ids=["+inf", "-inf", "nan"])
@pytest.mark.parametrize("tensor", ["q", "k", "v"])
def test_packed_batch_isolation(tensor, value, prefill_gen):
    """Three prompts, the middle one (and the rows past the last prompt) holding a non-finite value in its Q, K or V (an
    fp16 overflow in another user's request): the other prompts' outputs are bit-identical to a run where every value is
    finite.  The first and last prompts end inside a 64-key step, so the wgmma kernel's last K / V boxes reach into the
    poisoned rows: K there is masked, V there must not reach the P . V product."""
    lens = [300, 257, 130]
    starts = _starts(lens)
    T = sum(lens) + 70
    g = torch.Generator(device=DEV).manual_seed(3)
    q, k, v = (_randn(g, T, n, D).to(torch.bfloat16) for n in (NQ, NKV, NKV))
    o_ref = _packed(q, k, v, starts, lens)
    check_attention(o_ref, prefill64.prefill_attention(q, k, v, starts, lens, SCALE), NQ, lens, starts=starts)
    t = {"q": q, "k": k, "v": v}[tensor].clone()
    t[starts[1]:starts[1] + lens[1]] = value
    t[sum(lens):] = value
    args = {"q": q, "k": k, "v": v, tensor: t}
    o = _packed(args["q"], args["k"], args["v"], starts, lens)
    for i in (0, 2):
        rows = slice(starts[i], starts[i] + lens[i])
        bad = (o[rows].view(torch.int16) != o_ref[rows].view(torch.int16)).any(-1).any(-1)
        assert not bad.any(), (f"prompt {i}: {int(bad.sum())} of {lens[i]} rows changed (first at token "
                               f"{int(bad.nonzero()[0])}; {int((~torch.isfinite(o[rows].float())).any(-1).any(-1).sum())} "
                               f"non-finite) when prompt 1 holds {value} in {tensor.upper()}")
    assert (o[sum(lens):] == 0).all(), "rows past the last prompt were written"
