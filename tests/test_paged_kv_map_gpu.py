"""GPU: the two KV page maps of the sm_90a decode and verification kernels (csrc/paged_attn_tc.cu, kv_maps_and_layout).

The kernels load K / V pages either through the permuted-stride 4-D tensor map (one box per 16-token page) or, where the
driver rejects that map, through the cache viewed as [rows, 128] (two boxes per page, other shared-memory strides).  The
H100 driver accepts the 4-D map, so the 2-D layout only runs under SLLM_PAGED_ATTN_KV_MAP=2d.  Every case here runs the same
inputs under both maps and asserts:
  * sllm_paged_attention_kv_map_rank() is 2 under the switch and 4 without it (where the driver rejects the 4-D map the case
    says so and checks the 2-D layout alone);
  * the 2-D output is bit-identical to the 4-D output: only the placement of bytes in shared memory differs;
  * the 2-D output is within tests/attention_check.py's tolerance of fp64.
Decode: GQA groups 1, 3, 4, 8 (wgmma N = 8) and 12, 16 (N = 16) in the bench regime (two splits), the single-pass regime and
a small batch with many splits, lengths at page, tile and split edges, and poisoned pages.  Verification: N = 8, 16 and 32,
rows 1-8 straddling split boundaries."""
import warnings

import numpy as np
import pytest
import torch

from attention_check import check_attention
from oracle import kernels as K
from test_attention_regimes_gpu import (BS, D, DTYPES, _check_verify, _decode_case, _dev, _paged_run, _single_pass_lens, _table,
                                        _verify_case, _verify_exact, _verify_raw, num_splits, verify_split_tokens)
from verify_shapes import VERIFY_GEOMS, geom_id, verify_np

pytestmark = pytest.mark.gpu
ENV = "SLLM_PAGED_ATTN_KV_MAP"
EDGES = (1, 15, 16, 17, 127, 128, 129, 2047, 2048, 2049)        # page (16), tile (128) and split (2048 = 8 x 256) edges
GROUPS = [1, 3, 4, 8, 12, 16]                                    # 8 kv heads each


def kv_map_rank():
    from swiftllm_b200 import _lib
    return _lib.lib().sllm_paged_attention_kv_map_rank()


@pytest.fixture
def wgmma_only(monkeypatch):
    """Both decode and verification must run the sm_90a kernels (a shape they do not serve is an error), under the driver's
    own map choice unless a test sets the switch."""
    monkeypatch.setenv("SLLM_PAGED_ATTN_GEN", "2")
    monkeypatch.delenv(ENV, raising=False)
    return monkeypatch


def both_maps(mp, run):
    """run() under the driver's map, then under SLLM_PAGED_ATTN_KV_MAP=2d, checking the rank each time; the two outputs must
    be equal bit for bit when the first one used the 4-D map.  Returns the 2-D output."""
    mp.delenv(ENV, raising=False)
    o_drv = run()
    rank = kv_map_rank()
    assert rank in (2, 4), f"kv_map_rank() = {rank} after a launch"
    mp.setenv(ENV, "2d")
    assert kv_map_rank() == 2, "the switch must select the 2-D map"
    o_2d = run()
    assert kv_map_rank() == 2
    mp.delenv(ENV)
    assert kv_map_rank() == rank, "the switch must leave the driver probe as it was"
    if rank == 4:
        assert torch.equal(o_drv.view(torch.int16), o_2d.view(torch.int16)), "the 2-D page map changed the output bits"
    else:
        warnings.warn("the driver rejects the 4-D KV map: only the 2-D layout was checked")
    return o_2d


# ----------------------------------------------------------------------------- decode
def _decode_lens(regime, nq, nkv):
    """Lengths of a decode batch in `regime`, with the regime asserted through the planner's workspace."""
    if regime == "bench":                                        # bench.py's batch: two splits of 2048 tokens at 4096
        rng = np.random.default_rng(64)
        lens = rng.integers(1, 4097, size=64)
        lens[:12] = [4096, 4096, 4095, 2049, 2048, 2047, 1, 17, 128, 129, 2176, 3968]
        lens = tuple(int(x) for x in lens)
        assert num_splits(len(lens), nq, nkv, max(lens)) == 2
    elif regime == "single_pass":                                # batch x kv heads >= 6 x SMs: one item per (sequence, kv head)
        lens = _single_pass_lens(nkv, 2049)
        assert num_splits(len(lens), nq, nkv, max(lens)) == 1
    else:                                                        # 10 sequences: 256-token splits, most items empty
        lens = EDGES
        assert num_splits(len(lens), nq, nkv, max(lens)) >= 8
    return lens


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("group", GROUPS, ids=lambda g: f"g{g}")
@pytest.mark.parametrize("regime", ["bench", "single_pass", "many_splits"])
def test_decode_2d_map(dtype, group, regime, wgmma_only):
    nkv = 8
    nq = group * nkv
    lens = _decode_lens(regime, nq, nkv)
    q, kc, vc, bt, o64 = _decode_case(lens, nq, nkv, dtype, seed=group)
    qd, kd, vd, btd = _dev(q, kc, vc, bt)
    o = both_maps(wgmma_only, lambda: _paged_run(qd, kd, vd, btd, list(range(len(lens))), list(lens), D ** -0.5, BS, 0))
    check_attention(o, o64, nq, lens, what=f"decode(wgmma, 2d map, np{8 if group <= 8 else 16})")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("group", [3, 12], ids=lambda g: f"g{g}")
def test_decode_2d_map_poisoned_pages(dtype, group, wgmma_only):
    """NaN in every block (and layer) the batch does not own; slots of a sequence's last page past its end hold NaN K and
    V = 3e4.  The 2-D map loads whole pages in two boxes, so the tail must be masked exactly as with the 4-D map."""
    nkv, L, layer = 8, 2, 1
    nq = group * nkv
    lens = list(EDGES) + [777, 4091]
    g = torch.Generator().manual_seed(92 + group)
    bt, nblk = _table(g, lens, extra_blocks=7)
    kc = torch.randn(nblk, L, nkv, BS, D, generator=g).to(dtype); vc = torch.randn(nblk, L, nkv, BS, D, generator=g).to(dtype)
    q = torch.randn(len(lens), nq, D, generator=g).to(dtype)
    sids = list(range(len(lens)))
    o64 = K.paged_attention_exact(q, kc, vc, bt, sids, lens, D ** -0.5, BS, layer)
    owned = set()
    for s, n in enumerate(lens):
        npg = (n + BS - 1) // BS
        owned |= set(bt[s, :npg].tolist())
        last = int(bt[s, npg - 1])
        kc[last, layer, :, n - (npg - 1) * BS:] = float("nan"); vc[last, layer, :, n - (npg - 1) * BS:] = 3.0e4
    kc[:, 1 - layer] = float("nan"); vc[:, 1 - layer] = float("nan")
    for b in range(nblk):
        if b not in owned:
            kc[b] = float("nan"); vc[b] = float("nan")
    qd, kd, vd, btd = _dev(q, kc, vc, bt)
    o = both_maps(wgmma_only, lambda: _paged_run(qd, kd, vd, btd, sids, lens, D ** -0.5, BS, layer))
    assert torch.isfinite(o.float()).all()
    check_attention(o, o64, nq, lens, what=f"decode(wgmma, 2d map, np{8 if group <= 8 else 16})")


# ----------------------------------------------------------------------------- verification
VERIFY_WGMMA = [gm for gm in VERIFY_GEOMS if gm[3] is not None]


def _straddle_layout(g_, nkv, max_rows):
    """Rows 8, 7, ..., 1 (capped at max_rows) at prefixes that put the middle of each entry on a split boundary (split length
    read back from the workspace size), plus a one-row entry that fixes the longest length at 4000."""
    rows = [min(r, max_rows) for r in (8, 7, 6, 5, 4, 3, 2, 1)] + [1]
    B, T = len(rows), sum(rows)
    st = verify_split_tokens(B, T, g_ * nkv, nkv, 4000)
    prefix = [(i + 1) * st - r // 2 for i, r in enumerate(rows[:-1])] + [3999]
    assert max(p + r for p, r in zip(prefix, rows)) == 4000
    for p, r in zip(prefix, rows[:-1]):                          # the premise: every entry of 2+ rows sees two splits
        if r >= 2:
            assert len({-(-(p + j + 1) // st) for j in range(r)}) == 2
    return rows, prefix


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("geom", VERIFY_WGMMA, ids=geom_id)
def test_verify_2d_map(dtype, geom, wgmma_only):
    g_, nkv, max_rows, npad = geom
    nq = g_ * nkv
    rows, prefix = _straddle_layout(g_, nkv, max_rows)
    assert verify_np(g_, max(rows)) == npad
    g = torch.Generator().manual_seed(g_ * 100 + max_rows)
    q, kc, vc, bt = _verify_case(g, rows, prefix, nq, nkv, dtype)
    o64 = _verify_exact(q, kc, vc, bt, rows, prefix)
    dev = _dev(q, kc, vc, bt)
    o = both_maps(wgmma_only, lambda: _verify_raw(*dev, rows, prefix).cpu())
    _check_verify(o, o64, nq, rows, prefix, f"paged_attention_verify(wgmma, 2d map, np{npad})")


# ----------------------------------------------------------------------------- one process, both layouts
def test_switch_alternates_within_one_process(wgmma_only):
    """4-D, 2-D, 4-D again on the same caches: the switch acts per launch and the tensor-map cache keeps the two layouts of
    one cache apart (a 2-D launch that reused a cached 4-D map, or the reverse, would read the pages at the wrong strides)."""
    mp = wgmma_only
    nq, nkv = 32, 8
    lens = _decode_lens("bench", nq, nkv)
    q, kc, vc, bt, o64 = _decode_case(lens, nq, nkv, torch.bfloat16, seed=4)
    qd, kd, vd, btd = _dev(q, kc, vc, bt)
    rows, prefix = _straddle_layout(4, nkv, 8)
    g = torch.Generator().manual_seed(48)
    vq, vkc, vvc, vbt = _verify_case(g, rows, prefix, nq, nkv, torch.bfloat16)
    v64 = _verify_exact(vq, vkc, vvc, vbt, rows, prefix)
    vdev = _dev(vq, vkc, vvc, vbt)
    outs = []
    for env in (None, "2d", None):
        if env is None:
            mp.delenv(ENV, raising=False)
        else:
            mp.setenv(ENV, env)
        od = _paged_run(qd, kd, vd, btd, list(range(len(lens))), list(lens), D ** -0.5, BS, 0)
        ov = _verify_raw(*vdev, rows, prefix).cpu()
        rank = kv_map_rank()
        if env == "2d":
            assert rank == 2
        elif rank != 4:
            warnings.warn("the driver rejects the 4-D KV map: only the 2-D layout was checked")
        outs.append((rank, od, ov))
        check_attention(od, o64, nq, lens, what=f"decode(wgmma, rank {rank} map)")
        _check_verify(ov, v64, nq, rows, prefix, f"paged_attention_verify(wgmma, rank {rank} map, np32)")
    assert outs[0][0] == outs[2][0]
    for r, od, ov in outs[1:]:
        assert torch.equal(od.view(torch.int16), outs[0][1].view(torch.int16)), f"decode bits differ under the rank-{r} map"
        assert torch.equal(ov.view(torch.int16), outs[0][2].view(torch.int16)), f"verify bits differ under the rank-{r} map"
