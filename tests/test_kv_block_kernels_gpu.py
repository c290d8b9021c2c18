"""GPU: the KV-cache store and block-table kernels (csrc/kvcache.cu, csrc/rotary_store.cu, csrc/swap_gather.cu) bit for bit
against their restatements (tests/fork_oracle.py, oracle/kernels.py), at the sizes where their launch geometry changes
(tests/kv_geometry.py): allocator batches of one to three scan passes and on both sides of the 48 KB shared-memory edge, free
maps spanning many 16384-block windows, every page geometry of the stores, model-sized pages for the copies and block ids past
element offset 2^31.

Every cache and table starts as random bits (NaN payloads included) and whole buffers are compared, so a kernel that writes
where it must not is caught too.

Order matters in this file: cudaFuncSetAttribute lasts for the process, so an allocator batch of 6126 ... 6143 (which needs the
raised shared-memory limit only because of the kernel's static shared memory) must run before any batch above 12288 (which
raises it on dynamic shared memory alone); ALLOC_BATCHES is ascending and test_allocator_batches is the first allocator test."""
import types

import numpy as np
import pytest
import torch

import fork_oracle as FO
import kv_geometry as KG
from oracle import kernels as K

pytestmark = pytest.mark.gpu
DEV = "cuda"
DTYPES = [torch.float16, torch.bfloat16]


def i32(x):
    return torch.as_tensor(np.asarray(x, dtype=np.int32), device=DEV)


def i64(x):
    return torch.as_tensor(np.asarray(x, dtype=np.int64), device=DEV)


def rand_bits(shape, dtype, seed, device=DEV):
    """Random 16- or 32-bit patterns (NaN payloads and infinities included) in `dtype`."""
    g = torch.Generator(device=device).manual_seed(seed)
    if dtype == torch.int32:
        return torch.randint(-2 ** 31, 2 ** 31 - 1, shape, dtype=torch.int32, device=device, generator=g)
    return torch.randint(-2 ** 15, 2 ** 15, shape, dtype=torch.int16, device=device, generator=g).view(dtype)


def bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a.cpu()), bits(b.cpu()))


# ============================================================================ allocator
def free_map(num_blocks, pattern):
    idx = np.arange(num_blocks)
    if pattern == "all":
        return np.ones(num_blocks, dtype=bool)
    if pattern == "odd":
        return idx % 2 == 1
    if pattern == "every16":
        return idx % 16 == 5
    if pattern == "past-window":
        return idx >= KG.ALLOC_WINDOW
    assert pattern == "straddle"
    free = idx % 7 == 3
    for w in range(KG.ALLOC_WINDOW, num_blocks, KG.ALLOC_WINDOW):
        free[max(0, w - 50):w + 50] = True
    return free


def spread(total, rows, cap, rng):
    """Non-negative needs over `rows` rows (at most `cap` each) summing to `total`: every fifth row and one run of 9 rows need
    nothing (runs of equal start[] values), the rest share the total."""
    need = np.zeros(rows, dtype=np.int64)
    live = np.ones(rows, dtype=bool)
    live[::5] = False
    live[rows // 2: rows // 2 + 9] = False
    if not live.any() or total > cap * int(live.sum()):
        live[:] = True
    ids = np.nonzero(live)[0]
    need[ids] = total // len(ids)
    need[rng.choice(ids, total % len(ids), replace=False)] += 1
    assert need.max() <= cap and need.sum() == total
    return need


def alloc_inputs(batch, total, mbps, bs, rng, have_max=3):
    """Rows of a batch (distinct seq ids out of batch + 5 rows, in random order) that already hold 0 ... have_max - 1 blocks and
    need `total` more between them; returns (num rows, seq_ids, lens, nsab)."""
    rows = batch + 5
    seq_ids = rng.permutation(rows)[:batch]
    have = rng.integers(0, have_max, batch)
    need = spread(total, batch, mbps - have_max, rng)
    tgt = have + need
    lens = np.where(tgt > 0, (tgt - 1) * bs + rng.integers(1, bs + 1, batch), 0)
    nsab = rand_bits((rows,), torch.int32, 7, "cpu").numpy() % 1000      # rows outside the batch: any count
    nsab[seq_ids] = have
    return rows, seq_ids, lens, nsab


@pytest.mark.parametrize("batch", KG.ALLOC_BATCHES, ids=KG.batch_id)
def test_allocator_batches(batch):
    """BlockManager.allocate_blocks_for_seqs at every batch: the ids, the table, the counts and the free map are the
    restatement's, the host mirror agrees with the device, and the device status reports the total."""
    from swiftllm_b200.worker.block_manager import BlockManager
    rng = np.random.default_rng(batch)
    bs, mbps = 16, 40
    total = int(rng.integers(batch, 2 * batch + 1))
    rows, seq_ids, lens, nsab = alloc_inputs(batch, total, mbps, bs, rng)
    num_blocks = 2 * total + 2 * KG.ALLOC_WINDOW + 5
    free = free_map(num_blocks, "odd")
    table = rand_bits((rows, mbps), torch.int32, batch).cpu().numpy()

    bm = BlockManager("gpu", num_blocks, rows, mbps, bs)
    bm.block_table.copy_(torch.from_numpy(table))
    bm.num_seq_allocated_blocks.copy_(torch.from_numpy(nsab.astype(np.int32)))
    bm.is_block_free.copy_(torch.from_numpy(free))
    bm._host_nsab[:] = nsab
    bm.num_free_blocks = int(free.sum())

    want_ids = FO.allocate(nsab, table, free, seq_ids.tolist(), lens.tolist(), bs)
    assert len(want_ids) == total
    got = bm.allocate_blocks_for_seqs(i32(seq_ids), i32(lens), seq_ids_list=seq_ids.tolist(), target_lens_list=lens.tolist())
    assert bm.check_device_status() == total
    assert got.tolist() == want_ids
    assert np.array_equal(bm.block_table.cpu().numpy(), table)
    assert np.array_equal(bm.num_seq_allocated_blocks.cpu().numpy(), nsab)
    assert np.array_equal(bm._host_nsab, nsab) and bm.num_free_blocks == int(free.sum())
    assert np.array_equal(bm.is_block_free.cpu().numpy(), free)


@pytest.mark.parametrize("case", KG.FREE_MAPS, ids=KG.free_map_id)
def test_allocator_free_maps(case):
    """The wrapper on fragmented free maps: 1025 rows (two scan passes) take every free block when at most 30 per row cover
    them (exactly enough), else 30750 blocks spread over many windows; new_out has slack that must keep its bits."""
    from swiftllm_b200.worker.kernels.block_mgmt import allocate_blocks_for_seqs
    num_blocks, pattern = case
    rng = np.random.default_rng(num_blocks + len(pattern))
    bs, mbps, batch = 8, 36, 1025
    free = free_map(num_blocks, pattern)
    nfree = int(free.sum())
    total = min(nfree, 30 * batch)
    rows, seq_ids, lens, nsab = alloc_inputs(batch, total, mbps, bs, rng, have_max=6)
    table = rand_bits((rows, mbps), torch.int32, num_blocks).cpu().numpy()
    d_nsab, d_table, d_free = i32(nsab), i32(table), torch.from_numpy(free).to(DEV)
    new_out = rand_bits((2 * (total + 3),), torch.int32, 3).view(torch.int64)
    slack = new_out[total:].clone()
    status = i32([-1, -1])

    want_ids = FO.allocate(nsab, table, free, seq_ids.tolist(), lens.tolist(), bs)
    if nfree > 200:
        assert len(KG.windows(want_ids)) >= min(2, KG.cdiv(num_blocks, KG.ALLOC_WINDOW)), sorted(KG.windows(want_ids))
    allocate_blocks_for_seqs(d_nsab, d_table, d_free, i32(seq_ids), i32(lens), bs, new_out, status)
    assert status.tolist() == [total, 0]
    assert new_out[:total].tolist() == want_ids and torch.equal(new_out[total:], slack)
    assert np.array_equal(d_table.cpu().numpy(), table) and np.array_equal(d_nsab.cpu().numpy(), nsab)
    assert np.array_equal(d_free.cpu().numpy(), free)
    if total == nfree:
        assert not free.any()


STATUS_CASES = [("have>target",), ("target>mbps",), ("short",), ("new_out small",), ("have>target", "target>mbps"),
                ("short", "new_out small"), ("have>target", "new_out small"), ("target>mbps", "short")]


@pytest.mark.parametrize("batch", [33, 2049])
@pytest.mark.parametrize("faults", STATUS_CASES, ids=lambda f: "+".join(f))
def test_allocator_status_word(faults, batch):
    """Inputs the host would refuse, given to the wrapper: status [0, flags] as the restatement states it, and the table,
    counts, free map and new_out keep every bit.  The faulty rows sit in the last scan pass."""
    from swiftllm_b200.worker.kernels.block_mgmt import allocate_blocks_for_seqs
    rng = np.random.default_rng(batch + len(faults))
    bs, mbps = 16, 40
    total = 3 * batch
    rows, seq_ids, lens, nsab = alloc_inputs(batch, total, mbps, bs, rng)
    num_blocks = total + 100
    free = free_map(num_blocks, "all")
    if "have>target" in faults:
        k = batch - 2
        nsab[seq_ids[k]] = (lens[k] + bs - 1) // bs + 1
    if "target>mbps" in faults:
        lens[batch - 1] = mbps * bs + 1
    need = int(np.maximum((lens + bs - 1) // bs - nsab[seq_ids], 0).sum())
    if "short" in faults:
        free[np.nonzero(free)[0][need - 1:]] = False            # one block short
    cap = need - 1 if "new_out small" in faults else need + 4
    want = FO.allocate_status(nsab, free, seq_ids, lens, bs, mbps, cap)
    expect_flags = sum(KG.ALLOC_FLAGS[f] for f in faults if not (f == "short" and ("target>mbps" in faults or "have>target" in faults)))
    assert want == [0, expect_flags]
    table = rand_bits((rows, mbps), torch.int32, 11).cpu().numpy()
    d_nsab, d_table, d_free = i32(nsab), i32(table), torch.from_numpy(free).to(DEV)
    new_out = rand_bits((2 * cap,), torch.int32, 12).view(torch.int64)
    new_out0 = new_out.clone()
    status = i32([-1, -1])
    allocate_blocks_for_seqs(d_nsab, d_table, d_free, i32(seq_ids), i32(lens), bs, new_out, status)
    assert status.tolist() == want
    assert np.array_equal(d_table.cpu().numpy(), table) and np.array_equal(d_nsab.cpu().numpy(), nsab)
    assert np.array_equal(d_free.cpu().numpy(), free) and torch.equal(new_out, new_out0)


def test_allocator_refuses_a_batch_past_its_shared_memory():
    """Batch 25600: BlockManager raises before it reserves (mirror, free count and device unchanged), and the wrapper's launcher
    refuses it with nothing written."""
    from swiftllm_b200.worker.block_manager import BlockManager
    from swiftllm_b200.worker.kernels.block_mgmt import allocate_blocks_for_seqs
    batch, bs, mbps = KG.MAX_ALLOC_BATCH + 1, 16, 4
    assert KG.alloc_band(batch) == "refused"
    bm = BlockManager("gpu", 3 * batch, batch, mbps, bs)
    bm.block_table.copy_(rand_bits((batch, mbps), torch.int32, 5))
    table0, nsab0, free0 = bm.block_table.clone(), bm.num_seq_allocated_blocks.clone(), bm.is_block_free.clone()
    sids, lens = list(range(batch)), [17] * batch
    with pytest.raises(RuntimeError, match="at most 25599"):
        bm.allocate_blocks_for_seqs(i32(sids), i32(lens), seq_ids_list=sids, target_lens_list=lens)
    assert bm.num_free_blocks == 3 * batch and not bm._host_nsab.any()
    status = i32([-1, -1])
    with pytest.raises(RuntimeError, match="too large"):
        allocate_blocks_for_seqs(bm.num_seq_allocated_blocks, bm.block_table, bm.is_block_free, i32(sids), i32(lens), bs, None,
                                 status)
    torch.cuda.synchronize()
    assert torch.equal(bm.block_table, table0) and torch.equal(bm.num_seq_allocated_blocks, nsab0)
    assert torch.equal(bm.is_block_free, free0) and status.tolist() == [-1, -1]


# ============================================================================ other block-table kernels
def table_state(rng, batch, extra_rows=97, mbps=2048):
    """Rows of 32, 33 and 2048 blocks among rows of 0 ... 70, distinct valid block ids in each defined prefix, random bits past
    it; a random free map and random extra-owner counts.  Returns (nsab, table, is_free, extra, seq_ids, num_blocks)."""
    rows = batch + extra_rows
    counts = rng.integers(0, 71, rows)
    counts[rng.choice(rows, 6, replace=False)] = [32, 33, 2048, 32, 33, 2048]
    nb = int(counts.sum()) + 50
    ids = rng.permutation(nb)
    table = rand_bits((rows, mbps), torch.int32, int(rng.integers(1 << 30)), "cpu").numpy()
    p = 0
    for r in range(rows):
        table[r, :counts[r]] = ids[p:p + counts[r]]
        p += counts[r]
    seq_ids = rng.permutation(rows)[:batch]
    if batch:
        big = np.nonzero(counts >= 32)[0]
        seq_ids = rng.permutation(np.union1d(np.setdiff1d(seq_ids, big)[:batch - len(big)], big))
    is_free = rng.random(nb) < 0.5
    extra = rng.integers(0, 3, nb)
    return counts.astype(np.int64), table, is_free, extra, seq_ids, nb


def _dev(nsab, table, is_free, extra=None):
    out = [i32(nsab), i32(table), torch.from_numpy(is_free.copy()).to(DEV)]
    return out + ([i32(extra)] if extra is not None else [])


def _check(d, nsab, table, is_free, extra=None):
    assert np.array_equal(d[0].cpu().numpy(), nsab), "num_seq_allocated_blocks"
    assert np.array_equal(d[1].cpu().numpy(), table), "block_table"
    assert np.array_equal(d[2].cpu().numpy(), is_free), "is_block_free"
    if extra is not None:
        assert np.array_equal(d[3].cpu().numpy(), extra), "block_extra_refs"


def test_set_unset_gather_at_scale():
    from swiftllm_b200.worker.kernels import block_mgmt as BM
    rng = np.random.default_rng(1)
    nsab, table, is_free, _, seq_ids, nb = table_state(rng, 1003)
    assert len(seq_ids) >= 1000
    # set: grow rows by 0 ... 40 blocks (the 2048-block rows by none)
    need = np.minimum(rng.integers(0, 41, len(seq_ids)), 2048 - nsab[seq_ids])
    need[rng.choice(len(seq_ids), 3, replace=False)] = [32, 33, 0]
    need = np.minimum(need, 2048 - nsab[seq_ids])
    cand = rng.integers(0, 1 << 31, int(need.sum()))
    d = _dev(nsab, table, is_free)
    K.set_block_table_and_num_seq_alloc_blocks(nsab, table, cand, seq_ids, need)
    BM.set_block_table_and_num_seq_alloc_blocks(d[0], d[1], i64(cand), i32(seq_ids), i32(need))
    _check(d, nsab, table, is_free)
    # unset half the rows, gather the other half (all valid ids: restore them first)
    nsab2, table2, is_free2, _, seq_ids2, _ = table_state(rng, 1001)
    half = len(seq_ids2) // 2
    d = _dev(nsab2, table2, is_free2)
    K.unset_block_table_and_num_seq_alloc_blocks(nsab2, table2, seq_ids2[:half], is_free2)
    BM.unset_block_table_and_num_seq_alloc_blocks(d[0], d[1], i32(seq_ids2[:half]), d[2])
    _check(d, nsab2, table2, is_free2)
    want = K.gather_allocated_blocks_and_unset(nsab2, table2, seq_ids2[half:], is_free2)
    got = BM.gather_allocated_blocks_and_unset(d[0], d[1], i32(seq_ids2[half:]), d[2])
    assert np.array_equal(got.cpu().numpy(), want)
    _check(d, nsab2, table2, is_free2)


def test_truncate_at_scale():
    from swiftllm_b200.worker.kernels.block_mgmt import truncate_blocks_for_seqs
    rng = np.random.default_rng(2)
    nsab, table, is_free, extra, seq_ids, _ = table_state(rng, 1002)
    bs = 16
    n = nsab[seq_ids]
    kind = rng.integers(0, 5, len(seq_ids))
    lens = np.select([kind == 0, kind == 1, kind == 2, kind == 3],
                     [0, n * bs, n * bs + 1 + rng.integers(0, 1000, len(seq_ids)), (n // 2) * bs + 1],
                     rng.integers(0, np.maximum(n, 1) * bs + 1))
    extra[:] = 0
    d = _dev(nsab, table, is_free)
    FO.truncate(nsab, table, is_free, extra, seq_ids, lens, bs)
    truncate_blocks_for_seqs(d[0], d[1], d[2], i32(seq_ids), i32(lens), bs)
    _check(d, nsab, table, is_free)


def test_fork_at_scale():
    from swiftllm_b200.worker.kernels.block_mgmt import fork_blocks_for_seqs
    rng = np.random.default_rng(3)
    nsab, table, is_free, extra, _, _ = table_state(rng, 0, extra_rows=2100)
    bs = 8
    held = np.nonzero(nsab > 0)[0]
    big = np.nonzero(np.isin(nsab, [32, 33, 2048]))[0]
    src = np.concatenate([big, rng.choice(held, 1000 - len(big))])        # several entries share a src
    rest = np.setdiff1d(np.arange(len(nsab)), src)
    dst = rng.choice(rest, len(src), replace=False)
    nsab[dst] = 0
    kind = rng.integers(0, 4, len(src))
    full = nsab[src] * bs
    lens = np.select([kind == 0, kind == 1], [full, (full // bs) * bs - bs + 1], rng.integers(1, full + 1))
    lens = np.maximum(lens, 1)
    d = _dev(nsab, table, is_free, extra)
    FO.fork_rows(nsab, table, extra, src, dst, lens, bs)
    fork_blocks_for_seqs(d[0], d[1], d[3], i32(src), i32(dst), i32(lens), bs)
    _check(d, nsab, table, is_free, extra)


def test_release_at_scale():
    """One block held by 64 rows, all released in one launch: exactly one release frees it.  Then gathered and plain releases
    of the other rows in turn."""
    from swiftllm_b200.worker.kernels.block_mgmt import release_blocks_for_seqs
    rng = np.random.default_rng(4)
    nsab, table, is_free, extra, owners, nb = table_state(rng, 1500)
    shared_rows = rng.choice(owners[nsab[owners] < 32], 64, replace=False)
    nsab[shared_rows] = 1
    used = set(np.concatenate([table[r, :nsab[r]] for r in range(len(nsab))]).tolist())
    X = next(b for b in range(nb) if b not in used)
    table[shared_rows, 0] = X
    is_free[:] = True
    for r in owners:
        is_free[table[r, :nsab[r]]] = False
    extra[:] = 0
    extra[X] = 63
    others = rng.permutation(np.setdiff1d(owners, shared_rows))
    launches = [(rng.permutation(np.concatenate([shared_rows, others[:400]])), False), (others[400:900], True),
                (others[900:], False)]
    d = _dev(nsab, table, is_free, extra)
    for sids, how in launches:
        want = FO.release(nsab, table, is_free, extra, sids)
        total = len(want) if how else None
        got = release_blocks_for_seqs(d[0], d[1], d[2], d[3], i32(sids), total_blocks=total)
        if how:
            assert np.array_equal(got.cpu().numpy(), np.asarray(want, dtype=np.int32))
        _check(d, nsab, table, is_free, extra)
    assert is_free[X] and extra[X] == 0


# ============================================================================ stores
def store_layout(bs, seqs_blocks, rng, layers=3):
    """Block table over distinct, scattered block ids for sequences needing the given numbers of blocks (random bits past them)."""
    mbps = max(seqs_blocks) + 3
    nb = sum(seqs_blocks) + 7
    ids = rng.permutation(nb)
    table = rand_bits((len(seqs_blocks), mbps), torch.int32, int(rng.integers(1 << 30)), "cpu")
    p = 0
    for r, n in enumerate(seqs_blocks):
        table[r, :n] = torch.from_numpy(ids[p:p + n].astype(np.int32))
        p += n
    return table, nb


def caches(nb, layers, nkv, bs, D, dtype, seed):
    kc = rand_bits((nb, layers, nkv, bs, D), dtype, seed, "cpu")
    vc = rand_bits((nb, layers, nkv, bs, D), dtype, seed + 1, "cpu")
    return kc, vc


def fused_qkv(T, nq, nkv, D, dtype, seed, finite_qk=False):
    """[T, (nq + 2 nkv) D] of random bits (q and k finite normals when `finite_qk`), and its q, k, v views."""
    buf = rand_bits((T, (nq + 2 * nkv) * D), dtype, seed, "cpu")
    if finite_qk:
        g = torch.Generator().manual_seed(seed)
        buf[:, :(nq + nkv) * D] = torch.randn(T, (nq + nkv) * D, generator=g).to(dtype)
    return buf


def views(buf, nq, nkv, D):
    T = buf.shape[0]
    return (buf[:, :nq * D].view(T, nq, D), buf[:, nq * D:(nq + nkv) * D].view(T, nkv, D),
            buf[:, (nq + nkv) * D:].view(T, nkv, D))


def _store_state(**kw):
    base = dict(num_prefill_seqs=0, num_decoding_seqs=0, num_prefill_tokens=0, max_prefill_len=0, prefill_seq_start_locs=None,
                prefill_seq_lens=None, decoding_seq_lens=None)
    base.update(kw)
    return types.SimpleNamespace(**base)


STORE_CASES = [(bs, h) for bs in KG.BLOCK_SIZES for h in KG.HEADS]


def store_id(c):
    return f"bs{c[0]}-{KG.heads_id(c[1])}"


def _dtype(case):
    return DTYPES[STORE_CASES.index(case) % 2]


@pytest.mark.parametrize("case", STORE_CASES, ids=store_id)
def test_store_prefill_and_decode(case):
    """store_kvcache: prompts of several pages, of exactly one page, of one token and a partial page, then decode rows at the
    first and last slot of a page; k / v are row-strided views of one fused QKV buffer; layer 2 of 3."""
    from swiftllm_b200.worker.kernels.kvcache_mgmt import store_kvcache
    bs, (nq, nkv, D) = case
    dtype = _dtype(case)
    rng = np.random.default_rng(bs * 1000 + nq)
    plens = [3 * bs + 1, bs, 1, min(2 * bs + 5, 300)]
    dlens = [1, bs, bs + 1, 4 * bs - 1, 5]
    lens = plens + dlens
    table, nb = store_layout(bs, [KG.cdiv(n, bs) for n in lens], rng)
    kc, vc = caches(nb, 3, nkv, bs, D, dtype, bs + nq)
    Tp = sum(plens)
    buf = fused_qkv(Tp + len(dlens), nq, nkv, D, dtype, 3 * bs + nkv)
    _, k, v = views(buf, nq, nkv, D)
    starts = np.cumsum([0] + plens[:-1]).tolist()
    sids = list(range(len(lens)))
    kcd, vcd, bufd = kc.to(DEV), vc.to(DEV), buf.to(DEV)
    _, kd, vd = views(bufd, nq, nkv, D)
    st = _store_state(seq_ids=i32(sids), num_prefill_seqs=len(plens), num_decoding_seqs=len(dlens), num_prefill_tokens=Tp,
                      prefill_seq_start_locs=i32(starts), prefill_seq_lens=i32(plens), max_prefill_len=max(plens),
                      decoding_seq_lens=i32(dlens))
    store_kvcache(kd, vd, kcd, vcd, table.to(DEV), None, None, st, 2)
    K.store_kvcache_inplace(k, v, kc, vc, table, sids, starts, plens, dlens, len(plens), Tp, bs, 2)
    assert same(kcd, kc) and same(vcd, vc) and same(bufd, buf)


@pytest.mark.parametrize("case", STORE_CASES, ids=store_id)
def test_store_chunked(case):
    """store_kvcache_chunked: chunks that start and end mid-page, fill pages exactly, cover one token, are empty, or start a
    sequence; with decode rows in the same call."""
    from swiftllm_b200.worker.kernels.kvcache_mgmt import store_kvcache
    bs, (nq, nkv, D) = case
    dtype = _dtype(case)
    rng = np.random.default_rng(bs * 1000 + nq + 1)
    prefix = [bs + 1, 2 * bs, 5, 7, 0, 3 * bs - 1]
    chunk = [2 * bs + 1, 2 * bs, 1, 0, bs + 3, 2]
    dlens = [2, 3 * bs, bs + 1]
    lens = [p + c for p, c in zip(prefix, chunk)] + dlens
    table, nb = store_layout(bs, [max(1, KG.cdiv(n, bs)) for n in lens], rng)
    kc, vc = caches(nb, 3, nkv, bs, D, dtype, bs + nq + 5)
    Tp = sum(chunk)
    buf = fused_qkv(Tp + len(dlens), nq, nkv, D, dtype, 5 * bs + nkv)
    _, k, v = views(buf, nq, nkv, D)
    starts = np.cumsum([0] + chunk[:-1]).tolist()
    sids = list(range(len(lens)))
    kcd, vcd, bufd = kc.to(DEV), vc.to(DEV), buf.to(DEV)
    _, kd, vd = views(bufd, nq, nkv, D)
    st = _store_state(seq_ids=i32(sids), num_prefill_seqs=len(chunk), num_decoding_seqs=len(dlens), num_prefill_tokens=Tp,
                      prefill_seq_start_locs=i32(starts), prefill_seq_lens=i32(chunk), max_prefill_len=max(chunk),
                      decoding_seq_lens=i32(dlens), prefill_prefix_lens=i32(prefix))
    store_kvcache(kd, vd, kcd, vcd, table.to(DEV), None, None, st, 1)
    K.store_kvcache_inplace(k, v, kc, vc, table, sids, starts, chunk, dlens, len(chunk), Tp, bs, 1, prefill_prefix_lens=prefix)
    assert same(kcd, kc) and same(vcd, vc) and same(bufd, buf)


def _rotary_inputs(case, B, seed):
    bs, (nq, nkv, D) = case
    dtype = _dtype(case)
    rng = np.random.default_rng(seed)
    dlens = rng.integers(1, 6 * bs + 1, B)
    dlens[:3] = [1, bs, bs + 1]
    table, nb = store_layout(bs, [KG.cdiv(int(n), bs) for n in dlens], rng)
    kc, vc = caches(nb, 3, nkv, bs, D, dtype, seed)
    buf = fused_qkv(B, nq, nkv, D, dtype, seed + 2, finite_qk=True)
    g = torch.Generator().manual_seed(seed + 3)
    cos = (torch.rand(B, D // 2, generator=g) * 2 - 1).to(dtype)
    sin = (torch.rand(B, D // 2, generator=g) * 2 - 1).to(dtype)
    return dtype, dlens, table, kc, vc, buf, cos, sin


@pytest.mark.parametrize("case", STORE_CASES, ids=store_id)
def test_rotary_store_decode_equals_rotary_then_store(case):
    """The fused decode launch (37 rows) leaves the same q, k and caches as rotary_embedding_inplace followed by store_kvcache,
    and as the restatement."""
    from swiftllm_b200.worker.kernels.kvcache_mgmt import rotary_store_kvcache_decode, store_kvcache
    from swiftllm_b200.worker.kernels.rotary_emb import rotary_embedding_inplace
    bs, (nq, nkv, D) = case
    B = 37
    dtype, dlens, table, kc, vc, buf, cos, sin = _rotary_inputs(case, B, bs * 100 + nq)
    assert KG.rotary_store_grid(B, nq, nkv, D) >= 2
    sids = list(range(B))
    st = _store_state(seq_ids=i32(sids), num_decoding_seqs=B, decoding_seq_lens=i32(dlens), position_cos=cos.to(DEV),
                      position_sin=sin.to(DEV))
    # fused
    kca, vca, bufa = kc.to(DEV), vc.to(DEV), buf.to(DEV)
    qa, ka, va = views(bufa, nq, nkv, D)
    rotary_store_kvcache_decode(qa, ka, va, kca, vca, table.to(DEV), st, 2)
    # unfused twin
    kcb, vcb, bufb = kc.to(DEV), vc.to(DEV), buf.to(DEV)
    qb, kb, vb = views(bufb, nq, nkv, D)
    rotary_embedding_inplace(qb, kb, st)
    store_kvcache(kb, vb, kcb, vcb, table.to(DEV), None, None, st, 2)
    assert same(bufa, bufb) and same(kca, kcb) and same(vca, vcb)
    # restatement
    q, k, v = views(buf, nq, nkv, D)
    qr, kr = K.rotary_embedding(q, k, cos, sin)
    q.copy_(qr)
    k.copy_(kr)
    K.store_kvcache_inplace(k, v, kc, vc, table, sids, [], [], dlens.tolist(), 0, 0, bs, 2)
    assert same(bufa, buf) and same(kca, kc) and same(vca, vc)


# ============================================================================ model-sized pages
def _page_cache(nb, shape, seed):
    return rand_bits((nb,) + shape, torch.bfloat16, seed), rand_bits((nb,) + shape, torch.bfloat16, seed + 1)


@pytest.mark.parametrize("page", KG.PAGES, ids=lambda p: p[1])
def test_copy_block_tails_model_pages(page):
    """68 entries (64 with a partial tail, 4 on a page boundary, which copy nothing): the tail page of every layer of K and V
    and the token page move; every other byte keeps its bits."""
    from swiftllm_b200.worker.kernels.block_mgmt import copy_block_tails
    shape, _ = page
    bs = shape[2]
    rng = np.random.default_rng(len(shape) + shape[2])
    n, mbps = 68, 3
    nb = 2 * n + 9
    kc, vc = _page_cache(nb, shape, 21)
    tok = rand_bits((nb, bs), torch.int32, 23)
    table = rand_bits((2 * n, mbps), torch.int32, 24, "cpu").numpy()
    src, dst = np.arange(n), np.arange(n, 2 * n)
    lens = rng.integers(1, mbps * bs, n)
    lens[:4] = [bs, 2 * bs, bs, 2 * bs]
    lens[4:6] = [1, mbps * bs - 1]
    ids = rng.permutation(nb)
    for e in range(n):
        j = int(lens[e]) // bs
        table[src[e], j], table[dst[e], j] = ids[2 * e], ids[2 * e + 1]
    ke, ve, te = kc.clone(), vc.clone(), tok.clone()
    FO.copy_tails(ke, ve, te, table, src, dst, lens, bs)
    copy_block_tails(kc, vc, tok, i32(table), i32(src), i32(dst), i32(lens), bs)
    torch.cuda.synchronize()
    assert torch.equal(bits(kc), bits(ke)) and torch.equal(bits(vc), bits(ve)) and torch.equal(tok, te)


@pytest.mark.parametrize("page", KG.PAGES, ids=lambda p: p[1])
def test_swap_model_pages_both_directions(page):
    """2 x SMs + 3 pages out to a pinned swap space and back in through the device-id kernel, scattered and consecutive ids,
    against the restatement and against the memcpy path on the same pages."""
    from swiftllm_b200 import swiftllm_c
    shape, _ = page
    n = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 3
    rng = np.random.default_rng(shape[2])
    ng, nc = n + 9, n + 5
    kc, vc = _page_cache(ng, shape, 31)
    ks = rand_bits((nc,) + shape, torch.bfloat16, 33, "cpu").pin_memory()
    vs = rand_bits((nc,) + shape, torch.bfloat16, 34, "cpu").pin_memory()
    # distinct ids, the first 40 one run of consecutive ids on both sides
    src = np.concatenate([np.arange(3, 43), rng.permutation(np.setdiff1d(np.arange(ng), np.arange(3, 43)))])[:n]
    dst = np.concatenate([np.arange(1, 41), rng.permutation(np.setdiff1d(np.arange(nc), np.arange(1, 41)))])[:n]
    # out: cache -> swap
    kco, vco, kso, vso = kc.cpu(), vc.cpu(), ks.clone(), vs.clone()
    K.swap_blocks_inplace(src, dst, False, kco, vco, kso, vso)
    ksm, vsm = ks.clone(), vs.clone()
    swiftllm_c.swap_blocks(src.tolist(), dst.tolist(), False, kc, vc, ksm, vsm)
    swiftllm_c.swap_blocks_device(i64(src), i64(dst), False, kc, vc, ks, vs)
    torch.cuda.synchronize()
    assert torch.equal(bits(ks), bits(kso)) and torch.equal(bits(vs), bits(vso))
    assert torch.equal(bits(ksm), bits(kso)) and torch.equal(bits(vsm), bits(vso))
    # in: swap -> other cache blocks
    back = rng.permutation(ng)[:n]
    kco, vco = kc.cpu(), vc.cpu()
    K.swap_blocks_inplace(dst, back, True, kco, vco, ks, vs)
    kcm, vcm = kc.clone(), vc.clone()
    swiftllm_c.swap_blocks(dst.tolist(), back.tolist(), True, kcm, vcm, ks, vs)
    swiftllm_c.swap_blocks_device(i64(dst), i64(back), True, kc, vc, ks, vs)
    torch.cuda.synchronize()
    assert torch.equal(bits(kc.cpu()), bits(kco)) and torch.equal(bits(vc.cpu()), bits(vco))
    assert torch.equal(bits(kcm), bits(kc)) and torch.equal(bits(vcm), bits(vc))


# ============================================================================ past element offset 2^31
BIG_NKV, BIG_BS, BIG_D = 8, 16, 128
BIG_BLOCK_ELEMS = BIG_NKV * BIG_BS * BIG_D                             # one layer
FIRST_BIG = 2 ** 31 // BIG_BLOCK_ELEMS                                # first block whose element offset is 2^31
BIG_BLOCKS = FIRST_BIG + 256


@pytest.fixture(scope="module")
def big_cache():
    """K and V caches of 4 GiB each ([blocks, 1 layer, 8 kv heads, 16, 128] bf16): blocks >= FIRST_BIG start at element offsets
    >= 2^31.  Only the blocks a test touches are written or read."""
    nbytes = 2 * BIG_BLOCKS * BIG_BLOCK_ELEMS * 2
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + (1 << 30):
        pytest.skip(f"needs {nbytes / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free (the GPU is shared)")
    kc = torch.empty(BIG_BLOCKS, 1, BIG_NKV, BIG_BS, BIG_D, dtype=torch.bfloat16, device=DEV)
    vc = torch.empty_like(kc)
    yield kc, vc
    del kc, vc
    torch.cuda.empty_cache()


def test_stores_and_tails_past_2pow31(big_cache):
    """The allocator hands out ids on both sides of FIRST_BIG (through BlockManager); store_kvcache_chunked,
    rotary_store_kvcache_decode and copy_block_tails then write those blocks, bit-exact with the restatements on CPU copies."""
    from swiftllm_b200.worker.block_manager import BlockManager
    from swiftllm_b200.worker.kernels.block_mgmt import copy_block_tails
    from swiftllm_b200.worker.kernels.kvcache_mgmt import rotary_store_kvcache_decode, store_kvcache
    kc, vc = big_cache
    nq, bs, D = 32, BIG_BS, BIG_D
    rng = np.random.default_rng(231)
    rows, mbps = 9, 16
    bm = BlockManager("gpu", BIG_BLOCKS, rows, mbps, bs)
    free = np.zeros(BIG_BLOCKS, dtype=bool)
    free[FIRST_BIG - 20: FIRST_BIG + 200: 3] = True
    bm.is_block_free.copy_(torch.from_numpy(free))
    bm.num_free_blocks = int(free.sum())
    st_o = FO.BlockState(BIG_BLOCKS, rows, mbps, bs)
    st_o.is_free[:] = free
    # rows 0-5: chunked prefill (prefix + chunk) then one decode token; rows 6-8: fork destinations of rows 0-2's tails
    prefix, chunk = [40, 0, 17, 64, 3, 100], [33, 70, 1, 0, 29, 12]
    total_lens = [p + c + 1 for p, c in zip(prefix, chunk)]
    sids = list(range(6))
    want = st_o.allocate(sids, total_lens)
    got = bm.allocate_blocks_for_seqs(i32(sids), i32(total_lens), seq_ids_list=sids, target_lens_list=total_lens)
    assert got.tolist() == want and min(want) < FIRST_BIG <= max(want)
    tail_lens = [40, 70, 17]
    want += st_o.allocate([6, 7, 8], tail_lens)
    bm.allocate_blocks_for_seqs(i32([6, 7, 8]), i32(tail_lens), seq_ids_list=[6, 7, 8], target_lens_list=tail_lens)
    assert np.array_equal(bm.num_seq_allocated_blocks.cpu().numpy(), st_o.nsab)
    ids = sorted(want)
    assert max(ids) * BIG_BLOCK_ELEMS >= 2 ** 31
    for r in range(rows):
        assert bm.block_table[r, :st_o.nsab[r]].tolist() == st_o.table[r, :st_o.nsab[r]].tolist()
    dids = torch.tensor(ids, device=DEV)
    kc[dids] = rand_bits((len(ids), 1, BIG_NKV, bs, D), torch.bfloat16, 40)
    vc[dids] = rand_bits((len(ids), 1, BIG_NKV, bs, D), torch.bfloat16, 41)
    small = {b: i for i, b in enumerate(ids)}
    table = bm.block_table.cpu()
    table_small = torch.tensor([[small.get(int(b), -1) for b in row] for row in table.tolist()], dtype=torch.int32)
    kco, vco = kc[dids].cpu(), vc[dids].cpu()

    def check(what):
        assert torch.equal(bits(kc[dids].cpu()), bits(kco)) and torch.equal(bits(vc[dids].cpu()), bits(vco)), what

    # chunked store: the prefill chunks and decode rows 3-5 at prefix + chunk + 1
    Tp = sum(chunk)
    dl = [p + c + 1 for p, c in zip(prefix[3:], chunk[3:])]
    buf = fused_qkv(Tp + 3, nq, BIG_NKV, D, torch.bfloat16, 42)
    _, k, v = views(buf, nq, BIG_NKV, D)
    starts = np.cumsum([0] + chunk[:-1]).tolist()
    seq_ids = sids + [3, 4, 5]
    st = _store_state(seq_ids=i32(seq_ids), num_prefill_seqs=6, num_decoding_seqs=3, num_prefill_tokens=Tp,
                      prefill_seq_start_locs=i32(starts), prefill_seq_lens=i32(chunk), max_prefill_len=max(chunk),
                      decoding_seq_lens=i32(dl), prefill_prefix_lens=i32(prefix))
    bufd = buf.to(DEV)
    _, kd, vd = views(bufd, nq, BIG_NKV, D)
    store_kvcache(kd, vd, kc, vc, table.to(DEV), None, None, st, 0)
    K.store_kvcache_inplace(k, v, kco, vco, table_small, seq_ids, starts, chunk, dl, 6, Tp, bs, 0, prefill_prefix_lens=prefix)
    check("store_kvcache_chunked")
    # fused decode store of rows 0-2 at prefix + chunk + 1
    dl = [p + c + 1 for p, c in zip(prefix[:3], chunk[:3])]
    buf = fused_qkv(3, nq, BIG_NKV, D, torch.bfloat16, 43, finite_qk=True)
    g = torch.Generator().manual_seed(44)
    cos, sin = (torch.rand(3, D // 2, generator=g) * 2 - 1).to(torch.bfloat16), (torch.rand(3, D // 2, generator=g) * 2 - 1).to(torch.bfloat16)
    st = _store_state(seq_ids=i32([0, 1, 2]), num_decoding_seqs=3, decoding_seq_lens=i32(dl), position_cos=cos.to(DEV),
                      position_sin=sin.to(DEV))
    bufd = buf.to(DEV)
    qd, kd, vd = views(bufd, nq, BIG_NKV, D)
    rotary_store_kvcache_decode(qd, kd, vd, kc, vc, table.to(DEV), st, 0)
    q, k, v = views(buf, nq, BIG_NKV, D)
    qr, kr = K.rotary_embedding(q, k, cos, sin)
    q.copy_(qr)
    k.copy_(kr)
    K.store_kvcache_inplace(k, v, kco, vco, table_small, [0, 1, 2], [], [], dl, 0, 0, bs, 0)
    check("rotary_store_kvcache_decode")
    assert same(bufd, buf)
    # tails of rows 0-2 into rows 6-8
    copy_block_tails(kc, vc, None, table.to(DEV), i32([0, 1, 2]), i32([6, 7, 8]), i32(tail_lens), bs)
    FO.copy_tails(kco, vco, None, table_small.numpy(), [0, 1, 2], [6, 7, 8], tail_lens, bs)
    torch.cuda.synchronize()
    check("copy_block_tails")
