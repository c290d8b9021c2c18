"""GPU parity tests: every CUDA kernel (through the reference-named wrappers -> C ABI) against
 (1) the golden vectors produced by the unmodified reference (tests/golden), and
 (2) the CPU oracle on seeded random inputs (fp16 and bf16), including ragged / empty / maximum-ish cases,
 (3) size-independent properties at larger sizes.
Tolerances are stated per test; integer / copy work is bit-exact."""
import json
import types

import numpy as np
import pytest
import torch

from attention_check import check_attention
from oracle import kernels as K

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.float16, torch.bfloat16]


def T(a):
    return torch.from_numpy(np.ascontiguousarray(a))


def ulp_diff(a: torch.Tensor, b: torch.Tensor) -> int:
    """max distance in units of representable values of the 16-bit dtype (sign-magnitude aware)."""
    def key(t):
        i = t.contiguous().view(torch.int16).to(torch.int32)
        return torch.where(i < 0, -(i & 0x7FFF), i)
    return int((key(a.cpu()) - key(b.cpu())).abs().max())


def NS(**kw):
    return types.SimpleNamespace(**kw)


# ----------------------------------------------------------------------------- elementwise
def test_rmsnorm_golden(golden):
    from swiftllm_b200.worker.kernels.rmsnorm import rmsnorm_inplace, fused_add_rmsnorm_inplace
    z = golden("elementwise")
    x = T(z["rms_x"]).to(DEV); w = T(z["rms_w"]).to(DEV)
    rmsnorm_inplace(x, w, float(z["rms_eps"]))
    assert ulp_diff(x, T(z["rms_out"])) <= 1           # fp32 reduction order differs from numpy's
    x = T(z["rms_x"]).to(DEV); r = T(z["rms_r"]).to(DEV)
    fused_add_rmsnorm_inplace(x, r, w, float(z["rms_eps"]))
    assert ulp_diff(r, T(z["farms_r_out"])) == 0       # the storage-dtype add is exact
    assert ulp_diff(x, T(z["farms_x_out"])) <= 1


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", [(1, 64), (7, 256), (256, 4096), (33, 8192), (3, 1000 * 8)])
def test_rmsnorm_vs_oracle(dtype, shape):
    from swiftllm_b200.worker.kernels.rmsnorm import rmsnorm_inplace, fused_add_rmsnorm_inplace
    g = torch.Generator().manual_seed(shape[0] * 131 + shape[1])
    x = (torch.randn(shape, generator=g) * 2).to(dtype); r = torch.randn(shape, generator=g).to(dtype)
    w = (1 + 0.1 * torch.randn(shape[1], generator=g)).to(dtype)
    xo = K.rmsnorm(x, w, 1e-5)
    xd = x.to(DEV); rmsnorm_inplace(xd, w.to(DEV), 1e-5)
    assert ulp_diff(xd, xo) <= 1
    xo, ro = K.fused_add_rmsnorm(x, r, w, 1e-5)
    xd, rd = x.to(DEV), r.to(DEV); fused_add_rmsnorm_inplace(xd, rd, w.to(DEV), 1e-5)
    assert ulp_diff(rd, ro) == 0 and ulp_diff(xd, xo) <= 1


def test_rotary_golden_bit_exact(golden):
    from swiftllm_b200.worker.kernels.rotary_emb import rotary_embedding_inplace
    z = golden("elementwise")
    for tag in "ab":
        q, k = T(z[f"rot{tag}_q"]).to(DEV), T(z[f"rot{tag}_k"]).to(DEV)
        st = NS(position_cos=T(z[f"rot{tag}_cos"]).to(DEV), position_sin=T(z[f"rot{tag}_sin"]).to(DEV))
        rotary_embedding_inplace(q, k, st)
        assert ulp_diff(q, T(z[f"rot{tag}_q_out"])) == 0 and ulp_diff(k, T(z[f"rot{tag}_k_out"])) == 0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", [(1, 1, 1, 16), (5, 32, 8, 128), (300, 8, 1, 64), (257, 64, 8, 128)])
def test_rotary_vs_oracle_bit_exact(dtype, shape):
    from swiftllm_b200.worker.kernels.rotary_emb import rotary_embedding_inplace
    Tn, nq, nkv, D = shape
    g = torch.Generator().manual_seed(sum(shape))
    q = torch.randn(Tn, nq, D, generator=g).to(dtype); k = torch.randn(Tn, nkv, D, generator=g).to(dtype)
    ang = torch.rand(Tn, D // 2, generator=g) * 6.28
    cos, sin = torch.cos(ang).to(dtype), torch.sin(ang).to(dtype)
    qo, ko = K.rotary_embedding(q, k, cos, sin)
    qd, kd = q.to(DEV), k.to(DEV)
    rotary_embedding_inplace(qd, kd, NS(position_cos=cos.to(DEV), position_sin=sin.to(DEV)))
    assert ulp_diff(qd, qo) == 0 and ulp_diff(kd, ko) == 0


def test_silu_golden(golden):
    from swiftllm_b200.worker.kernels.silu_and_mul import silu_and_mul_inplace
    z = golden("elementwise")
    x = T(z["silu_x"]).to(DEV); silu_and_mul_inplace(x)
    ref = T(z["silu_out"])
    F = ref.shape[1] // 2
    assert ulp_diff(x[:, F:], ref[:, F:]) == 0             # gate half untouched
    assert ulp_diff(x[:, :F], ref[:, :F]) <= 1             # expf/division rounding (1 fp32 ulp) may flip an fp16 rounding


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", [(1, 8), (256, 14336), (9, 1792), (1025, 512)])
def test_silu_vs_oracle(dtype, shape):
    from swiftllm_b200.worker.kernels.silu_and_mul import silu_and_mul_inplace
    Tn, F = shape
    g = torch.Generator().manual_seed(Tn + F)
    x = (torch.randn(Tn, 2 * F, generator=g) * 3).to(dtype)
    ref = K.silu_and_mul(x)
    xd = x.to(DEV); silu_and_mul_inplace(xd)
    assert ulp_diff(xd[:, F:], ref[:, F:]) == 0
    # g is rounded to the dtype before the product: a 1-ulp flip of g moves the product by <= 1 ulp (+1 for its own rounding)
    assert ulp_diff(xd[:, :F], ref[:, :F]) <= 2
    frac = ((xd[:, :F].cpu().view(torch.int16) != ref[:, :F].contiguous().view(torch.int16)).float().mean())
    assert frac < 2e-3


# ----------------------------------------------------------------------------- KV store / block tables / swap
def _store_state(z_or_dict):
    d = z_or_dict
    return NS(seq_ids=d["seq_ids"], num_prefill_seqs=d["nps"], num_decoding_seqs=d["nds"], num_prefill_tokens=d["npt"],
              prefill_seq_start_locs=d["starts"], prefill_seq_lens=d["plens"], max_prefill_len=d["maxp"],
              decoding_seq_lens=d["dlens"])


def test_store_kvcache_golden_exact(golden):
    from swiftllm_b200.worker.kernels.kvcache_mgmt import store_kvcache
    z = golden("store_kvcache")
    i32 = lambda n: T(z[n]).to(torch.int32).to(DEV)
    st = _store_state(dict(seq_ids=i32("seq_ids"), nps=2, nds=1, npt=25, starts=i32("prefill_seq_start_locs"),
                           plens=i32("prefill_seq_lens"), maxp=20, dlens=i32("decoding_seq_lens")))
    kc = torch.zeros(z["k_cache_out"].shape, dtype=torch.float16, device=DEV); vc = torch.zeros_like(kc)
    store_kvcache(T(z["k"]).to(DEV), T(z["v"]).to(DEV), kc, vc, i32("block_table"), None, None, st, int(z["cur_layer"]))
    assert torch.equal(kc.cpu(), T(z["k_cache_out"])) and torch.equal(vc.cpu(), T(z["v_cache_out"]))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("cfg", [dict(plens=[], dlens=[5, 16, 17, 1]), dict(plens=[1, 16, 33, 100], dlens=[]),
                                 dict(plens=[40, 3], dlens=[64, 2, 31]), dict(plens=[257], dlens=[129] * 9)])
def test_store_kvcache_vs_oracle_exact(dtype, cfg):
    from swiftllm_b200.worker.kernels.kvcache_mgmt import store_kvcache
    L, nkv, bs, D, mbps = 3, 4, 16, 128, 20
    plens, dlens = cfg["plens"], cfg["dlens"]
    nseq = len(plens) + len(dlens)
    g = torch.Generator().manual_seed(nseq * 7 + sum(plens) + sum(dlens))
    need = [(n + bs - 1) // bs for n in plens + dlens]
    nblk = sum(need) + 3
    perm = torch.randperm(nblk, generator=g).tolist()
    sids = torch.randperm(nseq + 2, generator=g)[:nseq].tolist()
    bt = torch.full((nseq + 2, mbps), -1, dtype=torch.int32)
    p = 0
    for s, n in zip(sids, need):
        bt[s, :n] = torch.tensor(perm[p:p + n], dtype=torch.int32); p += n
    Tn = sum(plens) + len(dlens)
    k = torch.randn(Tn, nkv, D, generator=g).to(dtype); v = torch.randn(Tn, nkv, D, generator=g).to(dtype)
    starts = list(np.cumsum([0] + plens[:-1])) if plens else []
    kc = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype); vc = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype)
    kco, vco = kc.clone(), vc.clone()
    K.store_kvcache_inplace(k, v, kco, vco, bt, sids, starts, plens, dlens, len(plens), sum(plens), bs, 2)
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=DEV)
    st = _store_state(dict(seq_ids=i32(sids), nps=len(plens), nds=len(dlens), npt=sum(plens), starts=i32(starts),
                           plens=i32(plens), maxp=max(plens) if plens else 0, dlens=i32(dlens)))
    kcd, vcd = kc.to(DEV), vc.to(DEV)
    store_kvcache(k.to(DEV), v.to(DEV), kcd, vcd, bt.to(DEV), None, None, st, 2)
    assert torch.equal(kcd.cpu().view(torch.int16), kco.view(torch.int16))
    assert torch.equal(vcd.cpu().view(torch.int16), vco.view(torch.int16))


def _check_bm(bm, ref_bt, ref_n, ref_free, ref_nfree):
    n = bm.num_seq_allocated_blocks.cpu().numpy()
    assert np.array_equal(n, ref_n)
    assert np.array_equal(bm.is_block_free.cpu().numpy(), ref_free)
    assert bm.num_free_blocks == int(ref_nfree)
    bt = bm.block_table.cpu().numpy()
    for s in range(len(n)):
        assert np.array_equal(bt[s, : n[s]], ref_bt[s, : n[s]])
    assert np.array_equal(bm._host_nsab, n)               # host mirror in sync with the device


def test_block_manager_golden_trace_exact(golden):
    """KV-block indices bit-exact with the reference BlockManager on its recorded trace."""
    from swiftllm_b200.worker.block_manager import BlockManager
    z = golden("block_mgmt")
    ops = json.loads(str(z["ops"]))
    bm = BlockManager("GPU", 24, 8, 6, 16)
    t = lambda x: torch.tensor(x, dtype=torch.int32, device=DEV)
    for i, op in enumerate(ops):
        ret = None
        if op[0] == "alloc":
            ret = bm.allocate_blocks_for_seqs(t(op[1]), t(op[2]))          # tensor-only call (reference signature)
            bm.check_device_status()
        elif op[0] == "free":
            bm.free_blocks_for_seqs(t(op[1]))
        else:
            ret = bm.gather_allocated_blocks_and_free(t(op[1]))
        _check_bm(bm, z[f"s{i}_block_table"], z[f"s{i}_num_seq_allocated_blocks"], z[f"s{i}_is_block_free"], z[f"s{i}_num_free_blocks"])
        if ret is not None:
            assert np.array_equal(ret.cpu().numpy().astype(np.int64), z[f"s{i}_ret"].astype(np.int64))


def test_block_mgmt_wrappers_match_reference_kernels(golden):
    """The three block_mgmt.py wrappers (reference signatures) on their own."""
    from swiftllm_b200.worker.kernels import block_mgmt as B
    nsab = torch.zeros(6, dtype=torch.int32, device=DEV); bt = torch.full((6, 8), -1, dtype=torch.int32, device=DEV)
    free = torch.ones(32, dtype=torch.bool, device=DEV)
    o_nsab = np.zeros(6, dtype=np.int32); o_bt = np.full((6, 8), -1, dtype=np.int32); o_free = np.ones(32, dtype=bool)
    cand = torch.tensor([9, 3, 30, 7, 1, 0, 12], dtype=torch.int64)
    sids = torch.tensor([4, 1, 5], dtype=torch.int32); need = torch.tensor([3, 0, 4], dtype=torch.int32)
    B.set_block_table_and_num_seq_alloc_blocks(nsab, bt, cand.to(DEV), sids.to(DEV), need.to(DEV))
    K.set_block_table_and_num_seq_alloc_blocks(o_nsab, o_bt, cand.numpy(), sids.numpy(), need.numpy())
    assert np.array_equal(nsab.cpu().numpy(), o_nsab) and np.array_equal(bt.cpu().numpy(), o_bt)
    free[cand.to(DEV)] = False; o_free[cand.numpy()] = False
    g = B.gather_allocated_blocks_and_unset(nsab, bt, torch.tensor([5, 4], dtype=torch.int32, device=DEV), free)
    og = K.gather_allocated_blocks_and_unset(o_nsab, o_bt, [5, 4], o_free)
    assert np.array_equal(g.cpu().numpy(), og) and np.array_equal(free.cpu().numpy(), o_free) and np.array_equal(nsab.cpu().numpy(), o_nsab)
    B.set_block_table_and_num_seq_alloc_blocks(nsab, bt, cand.to(DEV), sids.to(DEV), need.to(DEV))
    K.set_block_table_and_num_seq_alloc_blocks(o_nsab, o_bt, cand.numpy(), sids.numpy(), need.numpy())
    B.unset_block_table_and_num_seq_alloc_blocks(nsab, bt, torch.tensor([4], dtype=torch.int32, device=DEV), free)
    K.unset_block_table_and_num_seq_alloc_blocks(o_nsab, o_bt, [4], o_free)
    assert np.array_equal(free.cpu().numpy(), o_free) and np.array_equal(nsab.cpu().numpy(), o_nsab)


@pytest.mark.parametrize("num_blocks", [7, 64, 1000, 70001])
def test_block_manager_random_ops_vs_oracle(num_blocks):
    """State machine: random alloc / grow / free / gather sequences, device allocator vs the oracle BlockManager."""
    from swiftllm_b200.worker.block_manager import BlockManager
    rng = np.random.default_rng(num_blocks)
    max_seqs, mbps, bs = 40, 64, 16
    bm = BlockManager("GPU", num_blocks, max_seqs, mbps, bs)
    ob = K.BlockManagerOracle(num_blocks, max_seqs, mbps, bs)
    lens = np.zeros(max_seqs, dtype=np.int64)
    t = lambda x: torch.tensor(np.asarray(x), dtype=torch.int32, device=DEV)
    for step in range(60):
        op = rng.choice(["alloc", "alloc", "free", "gather"])
        k = int(rng.integers(1, 12))
        sids = rng.choice(max_seqs, size=k, replace=False)
        if op == "alloc":
            tgt = np.minimum(lens[sids] + rng.integers(0, 200, size=k), mbps * bs)
            need = int(((tgt + bs - 1) // bs - ob.num_seq_allocated_blocks[sids]).sum())
            if need > ob.num_free_blocks:
                with pytest.raises(RuntimeError):
                    bm.allocate_blocks_for_seqs(t(sids), t(tgt), seq_ids_list=sids.tolist(), target_lens_list=tgt.tolist())
                continue
            r = bm.allocate_blocks_for_seqs(t(sids), t(tgt), seq_ids_list=sids.tolist(), target_lens_list=tgt.tolist())
            ro = ob.allocate_blocks_for_seqs(sids, tgt)
            if len(ro):
                assert bm.check_device_status() == len(ro)
            assert np.array_equal(r.cpu().numpy(), ro)
            lens[sids] = tgt
        elif op == "free":
            bm.free_blocks_for_seqs(t(sids), seq_ids_list=sids.tolist()); ob.free_blocks_for_seqs(sids); lens[sids] = 0
        else:
            r = bm.gather_allocated_blocks_and_free(t(sids), seq_ids_list=sids.tolist())
            ro = ob.gather_allocated_blocks_and_free(sids); lens[sids] = 0
            assert np.array_equal(r.cpu().numpy(), ro)
        _check_bm(bm, ob.block_table, ob.num_seq_allocated_blocks, ob.is_block_free, ob.num_free_blocks)


@pytest.mark.parametrize("pinned", [True, False])
def test_swap_blocks_exact(pinned):
    from swiftllm_b200 import swiftllm_c
    g = torch.Generator().manual_seed(3)
    shape = (12, 2, 2, 16, 64)
    kc = torch.randn(shape, generator=g).half(); vc = torch.randn(shape, generator=g).half()
    ks = torch.randn((9,) + shape[1:], generator=g).half(); vs = torch.randn((9,) + shape[1:], generator=g).half()
    src, dst = [3, 4, 5, 9, 10, 2], [0, 1, 2, 3, 7, 8]
    kco, vco, kso, vso = kc.clone(), vc.clone(), ks.clone(), vs.clone()
    K.swap_blocks_inplace(src, dst, False, kco, vco, kso, vso)
    kcd, vcd = kc.to(DEV), vc.to(DEV)
    ksd = ks.clone().pin_memory() if pinned else ks.clone(); vsd = vs.clone().pin_memory() if pinned else vs.clone()
    swiftllm_c.swap_blocks(src, dst, False, kcd, vcd, ksd, vsd); torch.cuda.synchronize()
    assert torch.equal(ksd, kso) and torch.equal(vsd, vso)
    K.swap_blocks_inplace(dst, src, True, kco, vco, kso, vso)
    swiftllm_c.swap_blocks(dst, src, True, kcd, vcd, ksd, vsd); torch.cuda.synchronize()
    assert torch.equal(kcd.cpu(), kco) and torch.equal(vcd.cpu(), vco)
    swiftllm_c.swap_blocks([], [], True, kcd, vcd, ksd, vsd)       # empty is a no-op


# ----------------------------------------------------------------------------- paged (decode) attention
def _paged_run(q, kc, vc, bt, sids, lens, scale, bs, layer, sbs=0):
    from swiftllm_b200.worker.kernels.paged_attn import paged_attention
    Bd, nq, D = q.shape
    i32 = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.int32).to(DEV)
    st = NS(num_decoding_seqs=Bd, num_prefill_seqs=0, seq_ids=i32(sids), decoding_seq_lens=i32(lens), softmax_scale=scale,
            max_decoding_len=int(max(lens)), paged_attn_seq_block_size=sbs)
    o = torch.zeros(Bd, nq * D, dtype=q.dtype, device=DEV)
    paged_attention(q.to(DEV), kc.to(DEV) if not kc.is_cuda else kc, vc.to(DEV) if not vc.is_cuda else vc, bt.to(DEV),
                    None, NS(block_size=bs), st, layer, o)
    return o.cpu()


def _gz(z, c):
    return (T(z[f"{c}_q"]), T(z[f"{c}_k_cache"]), T(z[f"{c}_v_cache"]), T(z[f"{c}_block_table"]), z[f"{c}_seq_ids"], z[f"{c}_seq_lens"],
            float(z[f"{c}_scale"]), int(z[f"{c}_block_size"]), int(z[f"{c}_cur_layer"]))


@pytest.mark.parametrize("case", ["c1", "c2"])
@pytest.mark.parametrize("sbs", [0, "ref"])
def test_paged_attention_golden(golden, case, sbs, paged_gen):
    """vs the reference's own outputs.  The reference accumulates q.k in fp16 (its own error vs fp64 is 1-3e-3 of
    max|o|, SURVEY.md §7); this kernel accumulates in fp32, so the tolerance is 3e-3 * max|o| against the reference
    and 1e-3 * max|o| against the fp64 definition (plus the per-(sequence, head) check of tests/attention_check.py)."""
    z = golden("paged_attention")
    args = _gz(z, case)
    s = int(z[f"{case}_seq_block_size"]) if sbs == "ref" else 0
    o = _paged_run(*args, sbs=s)
    o_ref = T(z[f"{case}_o"])
    o64 = K.paged_attention_exact(*args)
    assert (o.double() - o_ref.double()).abs().max() <= 3e-3 * o64.abs().max()
    assert (o.double() - o64).abs().max() <= 1e-3 * o64.abs().max()
    check_attention(o, o64, args[0].shape[1], args[5], what="decode")


@pytest.fixture(params=["gen2-tcgen05", "gen1-mma.sync"])
def paged_gen(request, monkeypatch):
    """Both kernel generations are exercised on every head_dim-128 shape (gen 2 is the default product path; shapes it
    does not cover - head_dim 64 - always run gen 1)."""
    monkeypatch.setenv("SLLM_PAGED_ATTN_GEN", "1" if request.param.startswith("gen1") else "0")
    return request.param


@pytest.mark.parametrize("dtype", DTYPES)
# GQA groups 1, 4, 8, 16 and the groups of real models that are not powers of two: 3 (24/8 heads, and head_dim 64),
# 5 (40/8), 6 (12/2), 7 (28/4), 12 (24/2); the wgmma kernel pads them to 8 or 16 heads
@pytest.mark.parametrize("geom", [dict(nq=4, nkv=4, D=64), dict(nq=8, nkv=2, D=128), dict(nq=32, nkv=8, D=128),
                                  dict(nq=8, nkv=1, D=128), dict(nq=16, nkv=1, D=128), dict(nq=4, nkv=4, D=128),
                                  dict(nq=12, nkv=4, D=64), dict(nq=24, nkv=8, D=128), dict(nq=40, nkv=8, D=128),
                                  dict(nq=12, nkv=2, D=128), dict(nq=28, nkv=4, D=128), dict(nq=24, nkv=2, D=128)])
@pytest.mark.parametrize("sbs", [0, 64, 256])
def test_paged_attention_vs_exact_oracle(dtype, geom, sbs, paged_gen):
    nq, nkv, D = geom["nq"], geom["nkv"], geom["D"]
    if D == 64 and paged_gen.startswith("gen2"):
        pytest.skip("head_dim 64 is served by gen 1 only")
    L, bs = 2, 16
    lens = [1, 15, 16, 17, 63, 64, 65, 128, 200, 333, 777]
    g = torch.Generator().manual_seed(nq * 1000 + D + sbs)
    need = [(n + bs - 1) // bs for n in lens]
    nblk = sum(need) + 5
    perm = torch.randperm(nblk, generator=g).tolist()
    sids = torch.randperm(len(lens) + 3, generator=g)[: len(lens)].tolist()
    mbps = max(need) + 2
    bt = torch.full((len(lens) + 3, mbps), -1, dtype=torch.int32)
    p = 0
    for s, n in zip(sids, need):
        bt[s, :n] = torch.tensor(perm[p:p + n], dtype=torch.int32); p += n
    kc = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype); vc = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype)
    q = torch.randn(len(lens), nq, D, generator=g).to(dtype)
    scale = D ** -0.5
    o64 = K.paged_attention_exact(q, kc, vc, bt, sids, lens, scale, bs, 1)
    o = _paged_run(q, kc, vc, bt, sids, lens, scale, bs, 1, sbs=sbs)
    check_attention(o, o64, nq, lens, what="decode")


def test_paged_attention_full_length_properties(paged_gen):
    """BASELINE config-2 sequence length (4096) at a reduced batch, Llama-3-8B head geometry, bf16:
    (a) vs the fp64 oracle, (b) v1 vs v2 agree, (c) result is invariant under a permutation of the physical blocks,
    (d) linear in V."""
    dtype, nq, nkv, D, bs, L = torch.bfloat16, 32, 8, 128, 16, 2
    lens = [4096, 4096, 4095, 2049]
    g = torch.Generator().manual_seed(11)
    need = [(n + bs - 1) // bs for n in lens]
    nblk = sum(need)
    kc = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype); vc = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype)
    q = torch.randn(len(lens), nq, D, generator=g).to(dtype)
    def table(perm):
        bt = torch.full((len(lens), max(need)), -1, dtype=torch.int32); p = 0
        for s, n in enumerate(need):
            bt[s, :n] = torch.tensor(perm[p:p + n], dtype=torch.int32); p += n
        return bt
    ident = list(range(nblk))
    sids = list(range(len(lens)))
    scale = D ** -0.5
    o1 = _paged_run(q, kc, vc, table(ident), sids, lens, scale, bs, 0)
    o64 = K.paged_attention_exact(q, kc, vc, table(ident), sids, lens, scale, bs, 0)
    check_attention(o1, o64, nq, lens, what="decode")
    o2 = _paged_run(q, kc, vc, table(ident), sids, lens, scale, bs, 0, sbs=512)          # forced flash-decoding split
    assert (o1.float() - o2.float()).abs().max() <= 2 ** -7 * o64.abs().max()           # both round to bf16 once
    perm = torch.randperm(nblk, generator=g).tolist()
    inv = torch.empty(nblk, dtype=torch.long); inv[torch.tensor(perm)] = torch.arange(nblk)
    kc_p = torch.empty_like(kc); vc_p = torch.empty_like(vc)
    kc_p[torch.tensor(perm)] = kc; vc_p[torch.tensor(perm)] = vc
    o3 = _paged_run(q, kc_p, vc_p, table(perm), sids, lens, scale, bs, 0)
    assert torch.equal(o1.view(torch.int16), o3.view(torch.int16))                       # same math, different pages
    vc2 = torch.randn(vc.shape, generator=g).to(dtype)
    oa = _paged_run(q, kc, vc2, table(ident), sids, lens, scale, bs, 0)
    ob = _paged_run(q, kc, (vc.float() + vc2.float()).to(dtype), table(ident), sids, lens, scale, bs, 0)
    assert (ob.float() - (o1.float() + oa.float())).abs().max() <= 3e-2 * o64.abs().max()


# ----------------------------------------------------------------------------- prefill attention
def _prefill_run(q, k, v, starts, lens, scale):
    from swiftllm_b200.worker.kernels.prefill_attn import prefill_attention
    i32 = lambda x: torch.as_tensor(np.asarray(x), dtype=torch.int32).to(DEV)
    st = NS(num_prefill_seqs=len(lens), prefill_seq_start_locs=i32(starts), prefill_seq_lens=i32(lens),
            max_prefill_len=int(max(lens)), softmax_scale=scale)
    o = torch.zeros(q.shape, dtype=q.dtype, device=DEV)
    prefill_attention(q.to(DEV), k.to(DEV), v.to(DEV), o, None, None, st)
    return o.cpu()


@pytest.fixture(params=["gen2-tcgen05", "gen1-mma.sync"])
def prefill_gen(request, monkeypatch):
    monkeypatch.setenv("SLLM_PREFILL_ATTN_GEN", "1" if request.param.startswith("gen1") else "0")
    return request.param


def test_prefill_attention_golden(golden, prefill_gen):
    """vs the reference's Triton prefill kernel run under the interpreter."""
    z = golden("prefill_attention")
    q, k, v = T(z["q"]), T(z["k"]), T(z["v"])
    o = _prefill_run(q, k, v, z["start_locs"], z["seq_lens"], float(z["scale"]))
    o64 = K.prefill_attention_exact(q, k, v, z["start_locs"], z["seq_lens"], float(z["scale"]))
    assert (o.double() - T(z["o"]).double()).abs().max() <= 2e-3 * o64.abs().max()
    check_attention(o, o64, q.shape[1], z["seq_lens"], starts=z["start_locs"], what="prefill")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("geom", [dict(nq=4, nkv=2, D=64), dict(nq=8, nkv=2, D=128), dict(nq=4, nkv=4, D=128),
                                  dict(nq=12, nkv=4, D=64), dict(nq=24, nkv=8, D=128), dict(nq=40, nkv=8, D=128),
                                  dict(nq=12, nkv=2, D=128), dict(nq=28, nkv=4, D=128), dict(nq=24, nkv=2, D=128)])
def test_prefill_attention_vs_exact_oracle(dtype, geom, prefill_gen):
    nq, nkv, D = geom["nq"], geom["nkv"], geom["D"]
    if D == 64 and prefill_gen.startswith("gen2"):
        pytest.skip("head_dim 64 is served by gen 1 only")
    lens = [1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 300, 513, 700]
    starts = list(np.cumsum([0] + lens[:-1]))
    Tn = sum(lens) + 7                                         # trailing decode rows must be left untouched
    g = torch.Generator().manual_seed(nq + D)
    q = torch.randn(Tn, nq, D, generator=g).to(dtype); k = torch.randn(Tn, nkv, D, generator=g).to(dtype)
    v = torch.randn(Tn, nkv, D, generator=g).to(dtype)
    o = _prefill_run(q, k, v, starts, lens, D ** -0.5)
    o64 = K.prefill_attention_exact(q, k, v, starts, lens, D ** -0.5)
    check_attention(o, o64, nq, lens, starts=starts, what="prefill")
    assert (o[sum(lens):] == 0).all()


@pytest.mark.parametrize("dtype", DTYPES)
def test_prefill_attention_growing_scores_force_rescales(dtype, prefill_gen):
    """Adversarial for the lazy-rescale path of the wgmma kernel: key magnitudes grow along the sequence and differ
    per row parity, so the running max of SOME rows of a warp jumps by more than 2^8 at several kv steps while their
    neighbours' does not (a per-thread decision around warp-collective TMEM loads/stores must not diverge)."""
    nq, nkv, D = 4, 2, 128
    lens = [700, 333]
    starts = [0, 700]
    Tn = sum(lens)
    g = torch.Generator().manual_seed(77)
    q = torch.randn(Tn, nq, D, generator=g)
    k = torch.randn(Tn, nkv, D, generator=g)
    v = torch.randn(Tn, nkv, D, generator=g)
    pos = torch.cat([torch.arange(n) for n in lens]).float()
    k = k * (1.0 + pos / 40.0)[:, None, None]                 # scores grow with the key position
    q[::2] *= 6.0                                             # even rows: large logits (frequent rescales); odd rows: small
    q[1::2] *= 0.05
    q, k, v = q.to(dtype), k.to(dtype), v.to(dtype)
    o = _prefill_run(q, k, v, starts, lens, D ** -0.5)
    o64 = K.prefill_attention_exact(q, k, v, starts, lens, D ** -0.5)
    assert torch.isfinite(o.float()).all()
    check_attention(o, o64, nq, lens, starts=starts, tol=2e-3 if dtype == torch.float16 else 1e-2, what="prefill")


def test_prefill_attention_long_sequence_property(prefill_gen):
    """4096-token prompt (the prefill tok/s shape): the last row of causal attention equals decode attention over
    the same keys, so prefill's final row must match the paged-decode kernel's output for the same data."""
    dtype, nq, nkv, D, bs = torch.bfloat16, 8, 2, 128, 16
    Ln = 4096
    g = torch.Generator().manual_seed(5)
    q = torch.randn(Ln, nq, D, generator=g).to(dtype); k = torch.randn(Ln, nkv, D, generator=g).to(dtype)
    v = torch.randn(Ln, nkv, D, generator=g).to(dtype)
    o = _prefill_run(q, k, v, [0], [Ln], D ** -0.5)
    kc = k.view(Ln // bs, bs, nkv, D).permute(0, 2, 1, 3).unsqueeze(1).contiguous()      # [blocks, 1, nkv, bs, D]
    vc = v.view(Ln // bs, bs, nkv, D).permute(0, 2, 1, 3).unsqueeze(1).contiguous()
    bt = torch.arange(Ln // bs, dtype=torch.int32).unsqueeze(0)
    od = _paged_run(q[-1:].contiguous(), kc, vc, bt, [0], [Ln], D ** -0.5, bs, 0)
    ref = K.paged_attention_exact(q[-1:], kc, vc, bt, [0], [Ln], D ** -0.5, bs, 0)
    check_attention(o[-1], ref[0], nq, [Ln], what="prefill")
    check_attention(od, ref, nq, [Ln], what="decode")
    # spot-check a few earlier rows against the fp64 definition
    for r in (0, 1, 127, 128, 2047, 3000):
        rr = K.paged_attention_exact(q[r:r + 1], kc, vc, bt, [0], [r + 1], D ** -0.5, bs, 0)
        check_attention(o[r], rr[0], nq, [r + 1], what="prefill")


# ----------------------------------------------------------------------------- row-strided q/k/v (fused QKV GEMM output)
@pytest.mark.parametrize("dtype", DTYPES)
def test_kernels_accept_fused_qkv_column_slices(dtype, paged_gen, prefill_gen):
    check_fused_qkv_column_slices(dtype, 8, 2)


def check_fused_qkv_column_slices(dtype, nq, nkv):
    """q, k, v as column slices of one [T, (nq + 2 nkv) D] buffer (what the fused QKV GEMM produces) must give exactly
    the results of separate contiguous tensors: rotary, KV store, prefill attention, chunked prefill attention, paged
    attention; the attention outputs also match the fp64 definition."""
    from swiftllm_b200.worker.kernels.rotary_emb import rotary_embedding_inplace
    from swiftllm_b200.worker.kernels.kvcache_mgmt import store_kvcache
    from swiftllm_b200.worker.kernels.prefill_attn import prefill_attention, prefill_attention_paged
    from swiftllm_b200.worker.kernels.paged_attn import paged_attention
    D, bs, L = 128, 16, 2
    plens, dlens = [130, 17], [300, 45, 64]
    Tp, Bd = sum(plens), len(dlens)
    Tn = Tp + Bd
    g = torch.Generator().manual_seed(21)
    qkv = torch.randn(Tn, (nq + 2 * nkv) * D, generator=g).to(dtype).to(DEV)
    def views(buf):
        q = buf[:, : nq * D].unflatten(1, (nq, D)); k = buf[:, nq * D:(nq + nkv) * D].unflatten(1, (nkv, D))
        v = buf[:, (nq + nkv) * D:].unflatten(1, (nkv, D))
        return q, k, v
    qs, ks, vs = views(qkv.clone())
    qc, kc_, vc_ = [t.contiguous() for t in views(qkv.clone())]
    ang = torch.rand(Tn, D // 2, generator=g) * 6.28
    st_rot = NS(position_cos=torch.cos(ang).to(dtype).to(DEV), position_sin=torch.sin(ang).to(dtype).to(DEV))
    rotary_embedding_inplace(qs, ks, st_rot); rotary_embedding_inplace(qc, kc_, st_rot)
    assert torch.equal(qs, qc) and torch.equal(ks, kc_)
    # block tables: prefill seqs 0,1 then decoding seqs 2,3,4 (their earlier tokens are random cache content)
    need = [(n + bs - 1) // bs for n in plens + dlens]
    nblk = sum(need) + 2
    bt = torch.full((5, max(need)), -1, dtype=torch.int32); p = 0
    for s_, n in enumerate(need):
        bt[s_, :n] = torch.arange(p, p + n, dtype=torch.int32); p += n
    bt = bt.to(DEV)
    i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=DEV)
    st = NS(seq_ids=i32([0, 1, 2, 3, 4]), num_prefill_seqs=2, num_decoding_seqs=Bd, num_prefill_tokens=Tp,
            prefill_seq_start_locs=i32([0, plens[0]]), prefill_seq_lens=i32(plens), max_prefill_len=max(plens),
            decoding_seq_lens=i32(dlens), max_decoding_len=max(dlens), softmax_scale=D ** -0.5, paged_attn_seq_block_size=0)
    cache0 = torch.randn(nblk, L, nkv, bs, D, generator=g).to(dtype).to(DEV)
    k1, v1, k2, v2 = cache0.clone(), cache0.flip(0).clone(), cache0.clone(), cache0.flip(0).clone()
    store_kvcache(ks, vs, k1, v1, bt, None, None, st, 1); store_kvcache(kc_, vc_, k2, v2, bt, None, None, st, 1)
    assert torch.equal(k1, k2) and torch.equal(v1, v2)
    o1 = torch.zeros(Tp, nq, D, dtype=dtype, device=DEV); o2 = torch.zeros_like(o1)
    prefill_attention(qs[:Tp], ks[:Tp], vs[:Tp], o1, None, None, st); prefill_attention(qc[:Tp].contiguous(), kc_[:Tp].contiguous(), vc_[:Tp].contiguous(), o2, None, None, st)
    assert torch.equal(o1, o2)
    starts = [0, plens[0]]
    ref = K.prefill_attention_exact(qc[:Tp].cpu(), kc_[:Tp].cpu(), vc_[:Tp].cpu(), starts, plens, D ** -0.5)
    check_attention(o1, ref, nq, plens, starts=starts, what="prefill")
    # chunked prefill over the cache just written: the prompts' last 40 / 9 tokens as chunks after their prefixes
    chunk, prefix = [40, 9], [plens[0] - 40, plens[1] - 9]
    qpk = torch.cat([qc[prefix[0]:plens[0]], qc[plens[0] + prefix[1]:Tp]])
    stc = NS(num_prefill_seqs=2, seq_ids=st.seq_ids, prefill_seq_start_locs=i32([0, chunk[0]]), prefill_seq_lens=i32(chunk),
             prefill_prefix_lens=i32(prefix), max_prefill_len=max(chunk), softmax_scale=D ** -0.5)
    qbuf = torch.zeros(sum(chunk), (nq + 2 * nkv) * D, dtype=dtype, device=DEV)
    qbuf[:, : nq * D] = qpk.flatten(1)
    qstr = qbuf[:, : nq * D].unflatten(1, (nq, D))                                                  # row stride (nq + 2 nkv) D
    p1 = torch.zeros(sum(chunk), nq, D, dtype=dtype, device=DEV); p2 = torch.zeros_like(p1)
    prefill_attention_paged(qstr, k1, v1, bt, p1, None, None, stc, 1)
    prefill_attention_paged(qpk.contiguous(), k1, v1, bt, p2, None, None, stc, 1)
    assert torch.equal(p1, p2)
    ref = K.prefix_prefill_attention_exact(qpk.cpu(), k1.cpu(), v1.cpu(), bt.cpu().numpy(), [0, 1], [0, chunk[0]], chunk, prefix,
                                           D ** -0.5, bs, 1)
    check_attention(p1, ref, nq, chunk, starts=[0, chunk[0]], prefix=prefix, what="paged_prefill")
    d1 = torch.zeros(Bd, nq * D, dtype=dtype, device=DEV); d2 = torch.zeros_like(d1)
    paged_attention(qs[Tp:], k1, v1, bt, None, NS(block_size=bs), st, 1, d1)
    paged_attention(qc[Tp:].contiguous(), k1, v1, bt, None, NS(block_size=bs), st, 1, d2)
    assert torch.equal(d1, d2)
    ref = K.paged_attention_exact(qc[Tp:].cpu(), k1.cpu(), v1.cpu(), bt.cpu(), [2, 3, 4], dlens, D ** -0.5, bs, 1)
    check_attention(d1, ref, nq, dlens, tol=2e-3 if dtype == torch.float16 else 1e-2, what="decode")
