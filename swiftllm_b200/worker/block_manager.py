"""GPU-resident block table / free map, API of the reference's BlockManager (swiftllm/worker/block_manager.py:5-103).

Same observable state (`block_table`, `num_seq_allocated_blocks`, `is_block_free`, `num_free_blocks`) and the same
allocation order (lowest free id first, batch order) - block ids are bit-exact with the reference.  What changed:
allocation is ONE kernel launch with no host<->device sync (the reference does assert(...).all(), .item() and
torch.nonzero, block_manager.py:50,70,75).  The host keeps a mirror of `num_seq_allocated_blocks` so that
exhaustion is detected on the host (RuntimeError, as in the reference) without reading the device.

Shared blocks (addition, `fork_blocks_for_seqs`): a fork makes another sequence's row point at the leading blocks of a row, and
`block_extra_refs` counts the owners of each block beyond the first.  Shared blocks are always a prefix of every row that holds
them.  Until the first fork nothing changes: the same kernels free and gather.  Afterwards release drops one owner per block and
a block becomes free when its last owner lets go; the host keeps the sharing in logical handles (per sequence, the handles of its
leading blocks that have been shared; handle -> the sequences holding it), so `num_free_blocks` and the number of leading shared
blocks of each sequence (`_host_shared`) stay exact without reading the device.  A call updates `_host_shared` only for the rows
whose count it can change, so its host cost does not grow with the number of other live forks.
"""
import numpy as np
import torch

from .kernels.block_mgmt import (MAX_ALLOCATE_BATCH,
                                 allocate_blocks_for_seqs as _allocate_kernel,
                                 fork_blocks_for_seqs as _fork_kernel,
                                 gather_allocated_blocks_and_unset,
                                 release_blocks_for_seqs as _release_kernel,
                                 truncate_blocks_for_seqs as _truncate_kernel,
                                 unset_block_table_and_num_seq_alloc_blocks)


class BlockManager:
    def __init__(self, device_name: str, num_blocks: int, max_seqs_in_block_table: int, max_blocks_per_seq: int,
                 block_size: int, device="cuda"):
        self.device_name = device_name
        self.num_free_blocks = num_blocks
        self.num_blocks = num_blocks
        self.block_size = block_size
        self.max_blocks_per_seq = max_blocks_per_seq

        # seq_id |-> number of blocks allocated for this sequence
        self.num_seq_allocated_blocks = torch.zeros((max_seqs_in_block_table,), dtype=torch.int32, device=device)
        # (seq_id, block_index) |-> block_id   (rows are only defined up to num_seq_allocated_blocks[seq_id])
        self.block_table = torch.empty((max_seqs_in_block_table, max_blocks_per_seq), dtype=torch.int32, device=device)
        # block_id |-> whether this block is free or not
        self.is_block_free = torch.ones((num_blocks,), dtype=torch.bool, device=device)

        self._host_nsab = np.zeros((max_seqs_in_block_table,), dtype=np.int64)   # host mirror
        self._status = torch.zeros((2,), dtype=torch.int32, device=device)

        # block_id |-> owners beyond the first (0 for every free block)
        self.block_extra_refs = torch.zeros((num_blocks,), dtype=torch.int32, device=device)
        self.forked = False             # release is refcount-aware from the first fork on
        self._rows = {}                 # seq_id |-> handles of its leading blocks that have been shared
        self._holders = {}              # handle |-> set of the seq_ids holding it (its owners)
        self._next_handle = 0
        self._host_shared = np.zeros((max_seqs_in_block_table,), dtype=np.int64)   # leading blocks with > 1 owner

    @staticmethod
    def _to_list(t, given):
        if given is not None:
            return [int(x) for x in given]
        return t.tolist()            # device sync: only when the caller has no host copy

    def allocate_blocks_for_seqs(self, seq_ids: torch.Tensor, target_lens: torch.Tensor, *,
                                 seq_ids_list=None, target_lens_list=None, want_new_blocks: bool = True) -> torch.Tensor:
        """Make sure seq #i has ceil(target_lens[i] / block_size) blocks.  Returns the new block ids (int64,
        batch order), like the reference (useful for swapping).  Pass the host lists to avoid a device sync."""
        total = self.reserve_blocks_for_seqs(self._to_list(seq_ids, seq_ids_list), self._to_list(target_lens, target_lens_list))
        new_blocks = torch.empty((total,), dtype=torch.int64, device=self.block_table.device) if want_new_blocks else None
        if total > 0:
            self.allocate_reserved_blocks(seq_ids.to(torch.int32).contiguous(), target_lens.to(torch.int32).contiguous(),
                                          new_blocks)
        return new_blocks

    def reserve_blocks_for_seqs(self, seq_ids_list, target_lens_list) -> int:
        """Host half of allocate_blocks_for_seqs: count ceil(target_lens_list[i] / block_size) blocks for seq #i into the host
        mirror and `num_free_blocks`, and return how many are new.  Raises RuntimeError, changing nothing, when the batch is larger
        than the allocation kernel takes, a sequence would need more than max_blocks_per_seq blocks or the free blocks do not
        suffice; the caller then enqueues nothing."""
        if len(seq_ids_list) > MAX_ALLOCATE_BATCH:
            raise RuntimeError(f"cannot allocate blocks for {len(seq_ids_list)} sequences in one call "
                               f"(at most {MAX_ALLOCATE_BATCH})")
        idx = np.asarray(seq_ids_list, dtype=np.int64)
        target = (np.asarray(target_lens_list, dtype=np.int64) + (self.block_size - 1)) // self.block_size
        have = self._host_nsab[idx]
        assert (have <= target).all(), \
            f"(On {self.device_name}) Logic error: Some sequences have more blocks already allocated than needed."
        if len(idx) and int(target.max()) > self.max_blocks_per_seq:
            raise RuntimeError(f"sequence needs {int(target.max())} blocks > max_blocks_per_seq={self.max_blocks_per_seq}")
        total = int((target - have).sum())
        if total > self.num_free_blocks:
            raise RuntimeError(f"No enough free blocks available on {self.device_name} ({self.num_blocks} in total, "
                               f"{self.num_free_blocks} free, {total} requested)")
        self._host_nsab[idx] = target
        self.num_free_blocks -= total
        return total

    def allocate_reserved_blocks(self, seq_ids: torch.Tensor, target_lens: torch.Tensor, new_blocks=None):
        """Device half of allocate_blocks_for_seqs: one launch of the allocation kernel on this manager's tables, for blocks
        reserve_blocks_for_seqs has counted (int32 contiguous ids and lengths; new ids into `new_blocks` when given).  No host
        work, so a CUDA graph can capture it with static ids and lengths and reserve before each replay."""
        _allocate_kernel(self.num_seq_allocated_blocks, self.block_table, self.is_block_free, seq_ids, target_lens,
                         self.block_size, new_blocks, self._status)

    def fork_blocks_for_seqs(self, src_seq_ids: torch.Tensor, dst_seq_ids: torch.Tensor, lens: torch.Tensor, *,
                             src_seq_ids_list, dst_seq_ids_list, lens_list):
        """dst #i gets the first lens[i] // block_size blocks of src #i (shared, one more owner each) and, when lens[i] is not a
        multiple of block_size, one fresh block allocated like any other (lowest free id first, batch order).  The caller has
        validated the lists (empty, distinct dst rows that are no src; 1 <= lens[i] <= blocks held by src * block_size) and copies
        the tail pages.  Raises RuntimeError, before any device work, when the tail blocks do not fit."""
        bs = self.block_size
        if len(dst_seq_ids_list) > MAX_ALLOCATE_BATCH:
            raise RuntimeError(f"cannot fork {len(dst_seq_ids_list)} sequences in one call (at most {MAX_ALLOCATE_BATCH})")
        tails = sum(1 for p in lens_list if p % bs)
        if tails > self.num_free_blocks:
            raise RuntimeError(f"No enough free blocks available on {self.device_name} ({self.num_blocks} in total, "
                               f"{self.num_free_blocks} free, {tails} requested)")
        for s, d, p in zip(src_seq_ids_list, dst_seq_ids_list, lens_list):
            k = p // bs
            row = self._rows.setdefault(s, [])
            while len(row) < k:             # blocks of src shared for the first time
                self._holders[self._next_handle] = {s}
                row.append(self._next_handle)
                self._next_handle += 1
            self._rows[d] = row[:k]
            for h in row[:k]:
                self._holders[h].add(d)
            self._host_nsab[d] = k
        self.forked = True
        _fork_kernel(self.num_seq_allocated_blocks, self.block_table, self.block_extra_refs, src_seq_ids, dst_seq_ids, lens, bs)
        self.allocate_blocks_for_seqs(dst_seq_ids, lens, seq_ids_list=dst_seq_ids_list, target_lens_list=lens_list,
                                      want_new_blocks=False)
        # a handle that gains an owner had one (src) or already counted as shared: only src and dst rows change
        self._refresh_shared(set(src_seq_ids_list) | set(dst_seq_ids_list))

    def _refresh_shared(self, sids):
        """Recount the leading shared blocks of the given sequences."""
        for sid in sids:
            row = self._rows.get(sid, ())
            n = 0
            while n < len(row) and len(self._holders[row[n]]) > 1:
                n += 1
            self._host_shared[sid] = n

    def _release_host(self, sids) -> int:
        """Host side of a refcount-aware release: drop one owner of every block of the sequences; returns how many become free."""
        freed, changed = 0, set()
        for s in sids:
            row = self._rows.pop(s, [])
            freed += int(self._host_nsab[s]) - len(row)
            for h in row:
                holders = self._holders[h]
                holders.discard(s)
                if not holders:
                    del self._holders[h]
                    freed += 1
                elif len(holders) == 1:     # its last holder no longer shares it
                    changed |= holders
            self._host_nsab[s] = 0
            changed.add(s)
        self._refresh_shared(changed)
        return freed

    def truncate_blocks_for_seqs(self, seq_ids: torch.Tensor, target_lens: torch.Tensor, *, seq_ids_list=None,
                                 target_lens_list=None):
        """Shrink seq #i to ceil(target_lens[i] / block_size) blocks; the blocks past it become free (and are handed out again
        lowest id first).  A target above the current allocation is a logic error.  Pass the host lists to avoid a sync."""
        sids = self._to_list(seq_ids, seq_ids_list)
        lens = self._to_list(target_lens, target_lens_list)
        if not sids:
            return
        idx = np.asarray(sids, dtype=np.int64)
        target = (np.asarray(lens, dtype=np.int64) + (self.block_size - 1)) // self.block_size
        have = self._host_nsab[idx]
        assert (target <= have).all(), \
            f"(On {self.device_name}) Logic error: truncating sequences to more blocks than they hold."
        total = int((have - target).sum())
        if total == 0:
            return
        if self.forked:
            # every position a step writes lies past the sequence's shared blocks and a truncation keeps at least one written
            # position, so only private blocks are given back: the plain truncation kernel stays correct
            assert (target >= self._host_shared[idx]).all(), \
                f"(On {self.device_name}) Logic error: truncating into blocks shared with a fork."
            for s, t in zip(sids, target.tolist()):
                for h in self._rows.get(s, [])[t:]:
                    del self._holders[h]
                if s in self._rows:
                    del self._rows[s][t:]
        _truncate_kernel(self.num_seq_allocated_blocks, self.block_table, self.is_block_free,
                         seq_ids.to(torch.int32).contiguous(), target_lens.to(torch.int32).contiguous(), self.block_size)
        self._host_nsab[idx] = target
        self.num_free_blocks += total

    def check_device_status(self):
        """Debug/test helper (syncs): the allocator kernel's own error flag."""
        n, err = self._status.tolist()
        if err:
            raise RuntimeError(f"device-side block allocation failed on {self.device_name} (flag {err})")
        return n

    def free_blocks_for_seqs(self, seq_ids: torch.Tensor, *, seq_ids_list=None):
        sids = self._to_list(seq_ids, seq_ids_list)
        if not sids:
            return
        idx = np.asarray(sids, dtype=np.int64)
        total = int(self._host_nsab[idx].sum())
        if total == 0:
            return                      # nothing allocated for these sequences on this device
        if self.forked:
            self.num_free_blocks += self._release_host(sids)
            _release_kernel(self.num_seq_allocated_blocks, self.block_table, self.is_block_free, self.block_extra_refs,
                            seq_ids.to(torch.int32))
            return
        self.num_free_blocks += total
        self._host_nsab[idx] = 0
        unset_block_table_and_num_seq_alloc_blocks(self.num_seq_allocated_blocks, self.block_table,
                                                   seq_ids.to(torch.int32), self.is_block_free)

    def gather_allocated_blocks_and_free(self, seq_ids: torch.Tensor, *, seq_ids_list=None) -> torch.Tensor:
        sids = self._to_list(seq_ids, seq_ids_list)
        idx = np.asarray(sids, dtype=np.int64)
        total = int(self._host_nsab[idx].sum()) if sids else 0
        if self.forked and sids:
            self.num_free_blocks += self._release_host(sids)
            return _release_kernel(self.num_seq_allocated_blocks, self.block_table, self.is_block_free, self.block_extra_refs,
                                   seq_ids.to(torch.int32), total_blocks=total)
        gathered = gather_allocated_blocks_and_unset(self.num_seq_allocated_blocks, self.block_table,
                                                     seq_ids.to(torch.int32), self.is_block_free, total_blocks=total)
        if sids:
            self._host_nsab[idx] = 0
        self.num_free_blocks += total
        return gathered

    def get_num_allocated_blocks(self, seq_ids: torch.Tensor) -> torch.Tensor:
        return self.num_seq_allocated_blocks[seq_ids.long()]

    def get_num_allocated_blocks_host(self, seq_ids_list) -> list:
        return self._host_nsab[np.asarray(seq_ids_list, dtype=np.int64)].tolist()

    def get_num_shared_blocks_host(self, seq_ids_list) -> list:
        """Leading blocks each sequence shares with a fork (host mirror, no sync)."""
        return self._host_shared[np.asarray(seq_ids_list, dtype=np.int64)].tolist()
