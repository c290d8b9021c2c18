"""tests/attention_check.py has power: at the shapes and lengths of the GPU attention tests, in fp16 and bf16, a CPU model
of the kernels' rounding (fp32 scores and softmax, P rounded to the storage dtype before P.V, l in fp32, o rounded once)
passes the check, and each fault model a kernel could plausibly commit fails it:
  * a 2 % weight slip on one split (the second half of every sequence's keys), e.g. a wrong split merge or rescale;
  * the last 128-token tile of a row's keys dropped;
  * the last partial page (block_size 16 or 32) dropped;
  * an off-by-one causal mask, in both directions (prefill);
  * a wrong kv head: h // 8 or h // 16 (the padded group width of the wgmma decode kernel) instead of h // g;
  * one head's output written over its neighbour's;
and, for speculative verification (entries of 1-8 rows after a cached prefix, tests/test_speculative_gpu.py):
  * every row of an entry sees the whole entry (masked by the entry's length instead of the row's position);
  * row j's output written to row j + 1 of its entry (a wrong (row, head) column decode)."""
import functools

import numpy as np
import pytest
import torch

from attention_check import TOL, check_attention
from oracle import kernels as K
from verify_shapes import LAYOUTS, VERIFY_GEOMS, verify_layout

DTYPES = [torch.float16, torch.bfloat16]
LOG2E = 1.4426950408889634

# (nq, nkv, D) of the GPU tests, the new GQA groups (3, 5, 6, 7, 12) included
DECODE_GEOMS = [(4, 4, 64), (8, 2, 128), (32, 8, 128), (8, 1, 128), (16, 1, 128), (4, 4, 128), (12, 4, 64),
                (24, 8, 128), (40, 8, 128), (12, 2, 128), (28, 4, 128), (24, 2, 128)]
DECODE_LENS = [1, 15, 16, 17, 63, 64, 65, 128, 200, 333, 777]
FULL_LENS = [4096, 4096, 4095, 2049]                                     # test_paged_attention_full_length_properties
PREFILL_GEOMS = [(4, 2, 64), (8, 2, 128), (4, 4, 128), (12, 4, 64), (24, 8, 128), (40, 8, 128), (12, 2, 128),
                 (28, 4, 128), (24, 2, 128)]
PREFILL_LENS = [1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 300, 513, 700]
PAGED_PREFIX = [0, 13, 64, 500, 100, 3, 255, 0]                          # test_prefill_attention_paged_vs_exact_oracle
PAGED_CHUNK = [37, 200, 64, 1, 513, 2, 257, 300]
def _padded_group(g):
    return 8 if g <= 8 else 16


def _attend(q, Kc, V, pos, scale, dtype=None, kv_of_head=None, visible=None, weight=None, lag=None):
    """Attention of queries q [n, nq, D] at positions pos [n] of a sequence with keys / values [nkv, L, D].
    dtype None: the fp64 definition.  Otherwise the kernels' rounding: fp32 scores and softmax, p = exp2(s - m_ref)
    rounded to `dtype` before P.V, l = sum p in fp32 (unrounded), o rounded to `dtype`.  m_ref is the row max, or with
    `lag` [nq, n] (log2 units, in [0, 8)) that much below it, as in the lazy rescale of the wgmma prefill kernel: p is then
    up to 2^8 and even the largest key's weight is rounded.  kv_of_head / visible [n, L] / weight [n, L] (a multiplier
    of p) describe a faulty kernel."""
    n, nq, D = q.shape
    nkv, L, _ = Kc.shape
    if kv_of_head is None:
        kv_of_head = torch.arange(nq) // (nq // nkv)
    if visible is None:
        visible = torch.arange(L)[None, :] <= pos[:, None]
    cd = torch.float64 if dtype is None else torch.float32
    Kh, Vh = Kc[kv_of_head].to(cd), V[kv_of_head].to(cd)                    # [nq, L, D]
    s = torch.matmul(q.transpose(0, 1).to(cd), Kh.transpose(1, 2))          # [nq, n, L]
    s = s.masked_fill(~visible[None], float("-inf"))
    if dtype is None:
        return torch.matmul(torch.softmax(s * scale, dim=-1), Vh).transpose(0, 1)
    s = s * (scale * LOG2E)
    m_ref = s.amax(-1, keepdim=True)
    if lag is not None:
        m_ref = m_ref - lag[..., None]
    p = torch.exp2(s - m_ref)
    if weight is not None:
        p = p * weight[None].float()
    l = p.sum(-1, keepdim=True)
    o = torch.matmul(p.to(dtype).float(), Vh) / l
    return o.to(dtype).transpose(0, 1)


class Case:
    """Random inputs of one GPU test shape: per sequence, queries at positions prefix .. prefix + n - 1 (decode: the
    last position) and the sequence's keys / values."""

    def __init__(self, kind, nq, nkv, D, dtype, lens, prefix=None, bs=16, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.kind, self.nq, self.nkv, self.D, self.dtype, self.bs = kind, nq, nkv, D, dtype, bs
        self.scale = D ** -0.5
        self.seqs = []
        for i, n in enumerate(lens):
            pre = 0 if prefix is None else prefix[i]
            L = pre + n if kind != "decode" else n
            nqr = 1 if kind == "decode" else n
            q = torch.randn(nqr, nq, D, generator=g).to(dtype)
            kc = torch.randn(nkv, L, D, generator=g).to(dtype)
            v = torch.randn(nkv, L, D, generator=g).to(dtype)
            pos = torch.tensor([L - 1]) if kind == "decode" else pre + torch.arange(n)
            self.seqs.append((q, kc, v, pos))
        self.lens = lens
        self.prefix = prefix
        self.starts = None if kind == "decode" else list(np.cumsum([0] + list(lens[:-1])))
        self.o64 = self.run(None)

    def run(self, dtype, fault=None, lazy=False):
        outs = []
        g = torch.Generator().manual_seed(8)
        for q, kc, v, pos in self.seqs:
            kw = {} if fault is None else fault(self, kc.shape[1], pos)
            if lazy:
                kw["lag"] = 8 * torch.rand(self.nq, len(pos), generator=g)
            outs.append(_attend(q, kc, v, pos, self.scale, dtype, **kw))
        return torch.cat(outs, 0)                                            # [rows, nq, D]

    def check(self, o):
        return check_attention(o, self.o64, self.nq, self.lens, starts=self.starts, prefix=self.prefix, what=self.kind)


# ----------------------------------------------------------------------------- fault models (kwargs of _attend)
def _causal(pos, L):
    return torch.arange(L)[None, :] <= pos[:, None]


def slip_one_split(c, L, pos):
    """The second half of the sequence's keys (one of two splits) weighted by 1.02."""
    w = torch.ones(len(pos), L, dtype=torch.float64)
    w[:, L // 2:] = 1.02
    return dict(weight=w)


def drop_last_tile(c, L, pos):
    """Each row loses the last 128-token tile of its keys (rows with one tile keep it)."""
    vis = _causal(pos, L)
    for i, p in enumerate(pos.tolist()):
        if p >= 128:
            vis[i, (p // 128) * 128:] = False
    return dict(visible=vis)


def drop_last_partial_page(c, L, pos):
    """The sequence's last page, when partly filled and not the only one, is never read."""
    vis = _causal(pos, L)
    if L % c.bs and L > c.bs:
        vis[:, (L // c.bs) * c.bs:] = False
    return dict(visible=vis)


def causal_one_short(c, L, pos):
    """Query at position p sees keys < p (position 0 keeps its key, so the fault is not a NaN)."""
    vis = torch.arange(L)[None, :] < pos[:, None]
    vis[:, 0] = True
    return dict(visible=vis)


def causal_one_long(c, L, pos):
    """Query at position p also sees key p + 1."""
    return dict(visible=torch.arange(L)[None, :] <= pos[:, None] + 1)


def wrong_kv_head(c, L, pos):
    """Head h reads kv head h // NP (the padded group width) instead of h // g."""
    return dict(kv_of_head=torch.arange(c.nq) // _padded_group(c.nq // c.nkv))


def whole_entry(c, L, pos):
    """Every row sees all L keys of its entry: the causal mask taken from the entry's length, not the row's position."""
    return dict(visible=torch.ones(len(pos), L, dtype=torch.bool))


FAULTS = {"slip_one_split": slip_one_split, "drop_last_tile": drop_last_tile, "drop_last_partial_page": drop_last_partial_page,
          "causal_one_short": causal_one_short, "causal_one_long": causal_one_long, "wrong_kv_head": wrong_kv_head,
          "head_to_neighbour": None, "whole_entry": whole_entry, "row_to_next_row": None}
APPLIES = {"decode": ["slip_one_split", "drop_last_tile", "drop_last_partial_page", "wrong_kv_head", "head_to_neighbour"],
           "prefill": ["slip_one_split", "drop_last_tile", "causal_one_short", "causal_one_long", "wrong_kv_head",
                       "head_to_neighbour"],
           "paged_prefill": ["slip_one_split", "drop_last_tile", "drop_last_partial_page", "causal_one_short", "causal_one_long",
                             "wrong_kv_head", "head_to_neighbour"],
           "verify": list(FAULTS)}


def _faulty(case, name):
    if name == "head_to_neighbour":
        o = case.run(case.dtype).clone()
        h = case.nq // 2 - 1
        o[:, h + 1] = o[:, h]
        return o
    if name == "row_to_next_row":          # row j of each entry lands on row j + 1 (row 0 keeps its own output)
        o = case.run(case.dtype).clone()
        for s0, n in zip(case.starts, case.lens):
            o[s0 + 1:s0 + n] = o[s0:s0 + n - 1].clone()
        return o
    return case.run(case.dtype, FAULTS[name])


# ----------------------------------------------------------------------------- shapes
SHAPES = ([("decode", g, None) for g in DECODE_GEOMS] + [("decode", (32, 8, 128), "full")] +
          [("prefill", g, None) for g in PREFILL_GEOMS] +
          [("paged_prefill", g, 16) for g in PREFILL_GEOMS] + [("paged_prefill", (8, 2, 128), 32)] +
          [("verify", (g * nkv, nkv, 128), (r, lay)) for g, nkv, r, _ in VERIFY_GEOMS for lay in LAYOUTS])


@functools.lru_cache(maxsize=None)
def _case(kind, geom, extra, dtype):
    nq, nkv, D = geom
    seed = nq * 1000 + nkv * 10 + D
    if kind == "decode":
        return Case(kind, nq, nkv, D, dtype, FULL_LENS if extra == "full" else DECODE_LENS, seed=seed)
    if kind == "prefill":
        return Case(kind, nq, nkv, D, dtype, PREFILL_LENS, seed=seed)
    if kind == "verify":
        rows, prefix = verify_layout(extra[1], nq // nkv, extra[0])
        return Case(kind, nq, nkv, D, dtype, rows, prefix=prefix, seed=seed + extra[0])
    return Case(kind, nq, nkv, D, dtype, PAGED_CHUNK, prefix=PAGED_PREFIX, bs=extra, seed=seed)


def _id(s):
    kind, (nq, nkv, D), extra = s
    if kind == "verify":
        extra = f"{extra[0]}rows-{extra[1]}"
    return f"{kind}-{nq}q{nkv}kv-d{D}" + (f"-{extra}" if extra is not None else "")


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("shape", SHAPES, ids=_id)
@pytest.mark.parametrize("m_ref", ["row_max", "lazy"])
def test_kernel_rounding_passes(shape, dtype, m_ref):
    """The rounding the kernels legitimately do stays inside the tolerance."""
    c = _case(*shape, dtype)
    c.check(c.run(dtype, lazy=m_ref == "lazy"))


def _applies(shape, fault):
    kind, (nq, nkv, D), extra = shape
    if kind == "verify" and extra[0] == 1 and fault in ("causal_one_long", "whole_entry", "row_to_next_row"):
        return False                      # 1-row entries: the row is the last position, there is no later row or key
    if fault == "wrong_kv_head":          # only where h // NP differs from h // g for some head
        return not torch.equal(torch.arange(nq) // _padded_group(nq // nkv), torch.arange(nq) // (nq // nkv))
    return fault in APPLIES[kind]


@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("shape,fault", [pytest.param(s, f, id=f"{f}-{_id(s)}") for s in SHAPES for f in FAULTS if _applies(s, f)])
def test_fault_is_rejected(shape, fault, dtype):
    c = _case(*shape, dtype)
    with pytest.raises(AssertionError):
        c.check(_faulty(c, fault))


def test_batch_max_normalisation_misses_a_split_slip():
    """Why the check normalises per (row, head): at the decode test's lengths in bf16, a 2 % slip on one split stays
    under the tolerance when measured against the batch's largest output."""
    c = _case("decode", (32, 8, 128), None, torch.bfloat16)
    o = _faulty(c, "slip_one_split")
    assert float((o.double() - c.o64).abs().max()) <= TOL[torch.bfloat16] * float(c.o64.abs().max())
    with pytest.raises(AssertionError):
        c.check(o)


def test_model_matches_the_oracle_definition():
    """The fp64 arm of the model is the definition in oracle/kernels.py (decode and chunked prefill)."""
    nq, nkv, D, bs = 12, 4, 64, 16
    c = Case("paged_prefill", nq, nkv, D, torch.bfloat16, [5, 20], prefix=[17, 0], seed=1)
    need = [(p + n + bs - 1) // bs for p, n in zip(c.prefix, c.lens)]
    kc = torch.zeros(sum(need), 1, nkv, bs, D, dtype=torch.bfloat16); vc = torch.zeros_like(kc)
    bt = torch.zeros(2, max(need), dtype=torch.int32)
    b0 = 0
    for s, (q, k, v, pos) in enumerate(c.seqs):
        L = k.shape[1]
        for j in range(need[s]):
            bt[s, j] = b0 + j
            t = k[:, j * bs:(j + 1) * bs]
            kc[b0 + j, 0, :, :t.shape[1]] = t; vc[b0 + j, 0, :, :t.shape[1]] = v[:, j * bs:(j + 1) * bs]
        b0 += need[s]
    q = torch.cat([s[0] for s in c.seqs])
    o = K.prefix_prefill_attention_exact(q, kc, vc, bt, [0, 1], c.starts, c.lens, c.prefix, c.scale, bs, 0)
    assert torch.allclose(o, c.o64, atol=1e-12)
    last = torch.stack([q[c.starts[s] + c.lens[s] - 1] for s in range(2)])
    od = K.paged_attention_exact(last, kc, vc, bt, [0, 1], [17 + 5, 20], c.scale, bs, 0).reshape(2, nq, D)
    assert torch.allclose(od, torch.stack([c.o64[c.starts[s] + c.lens[s] - 1] for s in range(2)]), atol=1e-12)
