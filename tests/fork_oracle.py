"""Restatement of the block manager with shared blocks (swiftllm_b200.worker.block_manager + csrc/kvcache.cu), in numpy.

State: `table` [max_seqs, max_blocks_per_seq] (row s defined up to nsab[s]), `nsab` [max_seqs], `is_free` [num_blocks],
`extra` [num_blocks] (owners beyond the first; 0 for every free block).  Operations, each the contract of one kernel (or of the
kernels one host call enqueues):
- allocate: every sequence grows to ceil(len / bs) blocks; the lowest free ids, ascending, are handed out in batch order.
- fork: dst row <- the first len // bs blocks of src's row (one more owner each), then `allocate` of the dst rows to len; the
  returned (src block, dst block) pairs are the tail pages to copy.
- release: every block of the sequences loses one owner; a block with no extra owner becomes free.  Returns the ids in batch order.
- truncate: every sequence shrinks to ceil(len / bs) blocks; the blocks past it (never shared) become free.
The functions work in place on the arrays they are given (numpy views of CPU tensors included), so the same code is both the
oracle and the CPU stand-in of the kernels."""
import numpy as np


def allocate(nsab, table, is_free, seq_ids, lens, bs):
    free_ids = np.nonzero(is_free)[0].tolist()
    p, out = 0, []
    for sid, tl in zip(seq_ids, lens):
        have = int(nsab[sid])
        need = max(0, (int(tl) + bs - 1) // bs - have)
        for i in range(need):
            b = free_ids[p]; p += 1
            table[sid, have + i] = b
            is_free[b] = False
            out.append(b)
        nsab[sid] = have + need
    return out


def allocate_status(nsab, is_free, seq_ids, lens, bs, mbps, cap=None):
    """The allocation kernel's status word [new blocks or 0, flags] for a call given these inputs.  Flags: 2 a sequence holds more
    blocks than its target, 4 a target above mbps, 1 too few free blocks (checked only without flag 2 or 4), 8 more new blocks
    than `cap` (the length of new_out, when one is given).  With any flag set the kernel changes nothing."""
    have = np.asarray([int(nsab[s]) for s in seq_ids], dtype=np.int64)
    tgt = (np.asarray(lens, dtype=np.int64) + bs - 1) // bs
    err = (2 if (have > tgt).any() else 0) | (4 if (tgt > mbps).any() else 0)
    total = int(np.maximum(tgt - have, 0).sum())
    if err == 0 and total > 0 and int(np.count_nonzero(is_free)) < total:
        err |= 1
    if cap is not None and total > cap:
        err |= 8
    return [0 if err else total, err]


def fork_rows(nsab, table, extra, src_ids, dst_ids, lens, bs):
    """The fork kernel alone: shares the leading blocks; the tail block comes from `allocate`."""
    for s, d, p in zip(src_ids, dst_ids, lens):
        k = int(p) // bs
        table[d, :k] = table[s, :k]
        for b in table[s, :k]:
            extra[b] += 1
        nsab[d] = k


def tail_pairs(table, src_ids, dst_ids, lens, bs):
    """(source block, destination block) of every entry with a partial tail."""
    return [(int(table[s, int(p) // bs]), int(table[d, int(p) // bs])) for s, d, p in zip(src_ids, dst_ids, lens) if int(p) % bs]


def copy_tails(k_cache, v_cache, token_cache, table, src_ids, dst_ids, lens, bs):
    for sb, db in tail_pairs(table, src_ids, dst_ids, lens, bs):
        k_cache[db] = k_cache[sb]
        v_cache[db] = v_cache[sb]
        if token_cache is not None:
            token_cache[db] = token_cache[sb]


def release(nsab, table, is_free, extra, seq_ids):
    out = []
    for sid in seq_ids:
        for b in table[sid, :int(nsab[sid])].tolist():
            out.append(b)
            if extra[b] > 0:
                extra[b] -= 1
            else:
                is_free[b] = True
        nsab[sid] = 0
    return out


def truncate(nsab, table, is_free, extra, seq_ids, lens, bs):
    for sid, tl in zip(seq_ids, lens):
        n = int(nsab[sid])
        keep = min(n, (int(tl) + bs - 1) // bs)
        for b in table[sid, keep:n]:
            assert extra[b] == 0, "truncation into a shared block"
            is_free[b] = True
        nsab[sid] = keep


class BlockState:
    """One device's block state, as the kernels leave it."""

    def __init__(self, num_blocks, max_seqs, max_blocks_per_seq, block_size):
        self.bs = block_size
        self.table = np.full((max_seqs, max_blocks_per_seq), -1, dtype=np.int64)
        self.nsab = np.zeros((max_seqs,), dtype=np.int64)
        self.is_free = np.ones((num_blocks,), dtype=bool)
        self.extra = np.zeros((num_blocks,), dtype=np.int64)

    def allocate(self, seq_ids, lens):
        return allocate(self.nsab, self.table, self.is_free, seq_ids, lens, self.bs)

    def fork(self, src_ids, dst_ids, lens):
        fork_rows(self.nsab, self.table, self.extra, src_ids, dst_ids, lens, self.bs)
        self.allocate(dst_ids, lens)
        return tail_pairs(self.table, src_ids, dst_ids, lens, self.bs)

    def release(self, seq_ids):
        return release(self.nsab, self.table, self.is_free, self.extra, seq_ids)

    def truncate(self, seq_ids, lens):
        truncate(self.nsab, self.table, self.is_free, self.extra, seq_ids, lens, self.bs)

    def rows(self):
        """seq -> its block ids (sequences holding blocks only)."""
        return {s: self.table[s, :n].tolist() for s, n in enumerate(self.nsab.tolist()) if n}

    def shared(self, sid):
        """Leading blocks of the row with more than one owner."""
        n = 0
        while n < self.nsab[sid] and self.extra[self.table[sid, n]] > 0:
            n += 1
        return n

    def check_invariants(self):
        owners = np.zeros_like(self.extra)
        for row in self.rows().values():
            for b in row:
                owners[b] += 1
        assert np.array_equal(owners > 0, ~self.is_free)
        assert np.array_equal(np.where(owners > 0, owners - 1, 0), self.extra)
