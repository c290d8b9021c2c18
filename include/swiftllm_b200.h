/*
 * swiftllm_b200.h - C ABI of the H100-native (sm_90a) data plane that replaces every kernel in
 * swiftLLM's `swiftllm/worker/kernels/` plus the native `swiftllm_c` module.
 *
 * Drop-in boundary: the reference binds its kernels as Python functions on torch tensors (one wrapper
 * per op, in place / into caller-provided outputs, current CUDA stream).  This library exports exactly
 * one entry point per wrapper, taking raw device pointers, sizes, a dtype tag and the stream; the host
 * package `swiftllm_b200/worker/kernels/*.py` binds them with ctypes under the reference's own names and
 * signatures (see INTEGRATION.md for the stub a swiftLLM maintainer would add).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the parameter name says `host_`;
 *   - tensors are contiguous in the reference's layouts (cited per function);
 *   - all functions enqueue on `stream` (a cudaStream_t) and return immediately;
 *   - return value: 0 on success, non-zero on error (`sllm_last_error()` gives the message).  Invalid
 *     shapes are rejected before anything is launched (the reference raises AssertionError there);
 *   - no CPU fallback exists: on a non-sm_90 device every launch fails with an error.
 *
 * Reference paths below are relative to the swiftLLM repository root.
 */
#ifndef SWIFTLLM_B200_H
#define SWIFTLLM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SLLM_ABI_VERSION 1

typedef enum { SLLM_F16 = 0, SLLM_BF16 = 1 } sllm_dtype_t;
typedef void* sllm_stream_t; /* cudaStream_t */

/* ---- library ---- */
int sllm_abi_version(void);
const char* sllm_last_error(void);          /* thread-local message of the last failing call */
int sllm_device_check(int device);          /* 0 iff `device` is compute capability 10.x */

/* ---- RMSNorm: swiftllm/worker/kernels/rmsnorm.py:26-37 (rmsnorm_inplace), :67-89 (fused_add_rmsnorm_inplace)
 * x [num_tokens, hidden] in place; weight [hidden].  fused: residual <- x + residual (rounded to dtype),
 * x <- rmsnorm(residual) * weight.  hidden % 8 == 0. */
int sllm_rmsnorm_inplace(void* x, const void* weight, float eps, int64_t num_tokens, int hidden,
                         sllm_dtype_t dtype, sllm_stream_t stream);
int sllm_fused_add_rmsnorm_inplace(void* x, void* residual, const void* weight, float eps, int64_t num_tokens,
                                   int hidden, sllm_dtype_t dtype, sllm_stream_t stream);

/* ---- Rotary embedding: swiftllm/worker/kernels/rotary_emb.py:44-58 (rotary_embedding_inplace)
 * q [T, nq, D], k [T, nkv, D] in place; cos/sin [T, D/2] (infer_state.position_cos/sin).  NeoX half-split.
 * D % 16 == 0.  *_row_stride: elements between consecutive token rows (nq*D / nkv*D when contiguous, as in the
 * reference; larger when q/k/v are column slices of one fused QKV GEMM output); heads stay contiguous within a token. */
int sllm_rotary_embedding_inplace(void* q, void* k, const void* cos, const void* sin, int64_t num_tokens,
                                  int num_q_heads, int num_kv_heads, int head_dim, int64_t q_row_stride,
                                  int64_t k_row_stride, sllm_dtype_t dtype, sllm_stream_t stream);

/* ---- SwiGLU gate: swiftllm/worker/kernels/silu_and_mul.py:25-34 (silu_and_mul_inplace)
 * x [T, 2*ffn_inter_dim] = [up | gate]; x[:, :F] <- up * silu(gate).  F % 8 == 0. */
int sllm_silu_and_mul_inplace(void* x, int64_t num_tokens, int64_t ffn_inter_dim, sllm_dtype_t dtype,
                              sllm_stream_t stream);

/* ---- KV-cache store: swiftllm/worker/kernels/kvcache_mgmt.py:81-122 (store_kvcache)
 * k,v [num_tokens, nkv, D] (prefill tokens first, then one row per decoding seq);
 * caches [num_blocks, num_layers, nkv, block_size, D]; block_table int32 [*, max_blocks_per_seq];
 * seq_ids int32 [num_prefill_seqs + num_decoding_seqs]. */
int sllm_store_kvcache(const void* k, const void* v, void* k_cache, void* v_cache, const int32_t* block_table,
                       const int32_t* seq_ids, const int32_t* prefill_seq_start_locs,
                       const int32_t* prefill_seq_lens, const int32_t* decoding_seq_lens, int num_prefill_seqs,
                       int num_decoding_seqs, int64_t num_prefill_tokens, int max_prefill_len, int cur_layer,
                       int num_layers, int num_kv_heads, int block_size, int head_dim, int max_blocks_per_seq,
                       int64_t k_row_stride, int64_t v_row_stride, sllm_dtype_t dtype, sllm_stream_t stream);

/* ---- Decode-step fusion (new): rotary_embedding_inplace (rotary_emb.py:44-58) + the decode part of store_kvcache
 * (kvcache_mgmt.py:50-79) in ONE launch for a batch of decoding rows only: q [Bd, nq, D] and k [Bd, nkv, D] rotated in place
 * with cos/sin [Bd, D/2]; the rotated k row and the v row of sequence i are written to position decoding_seq_lens[i] - 1 of
 * block-table row seq_ids[i].  Same results, bit for bit, as the two separate calls. */
int sllm_rotary_store_kvcache_decode(void* q, void* k, const void* v, const void* cos, const void* sin, void* k_cache,
                                     void* v_cache, const int32_t* block_table, const int32_t* seq_ids,
                                     const int32_t* decoding_seq_lens, int num_decoding_seqs, int cur_layer,
                                     int num_layers, int num_q_heads, int num_kv_heads, int block_size, int head_dim,
                                     int max_blocks_per_seq, int64_t q_row_stride, int64_t k_row_stride,
                                     int64_t v_row_stride, sllm_dtype_t dtype, sllm_stream_t stream);

/* ---- Paged (decode) attention: swiftllm/worker/kernels/paged_attn.py:152-222 (paged_attention)
 * q [Bd, nq, D]; o [Bd, nq*D]; seq_ids = infer_state.seq_ids[num_prefill_seqs:]; seq_lens = decoding_seq_lens.
 * seq_block_size: tokens per flash-decoding split (multiple of block_size); 0 = let the library choose
 * (v1 single pass when the batch alone fills the GPU, v2 split + merge otherwise).
 * workspace: fp32 scratch for split partials, >= sllm_paged_attention_workspace_bytes(...) bytes
 * (the reference allocates mid_o / mid_o_logexpsum per call, paged_attn.py:170-180). */
int64_t sllm_paged_attention_workspace_bytes(int num_decoding_seqs, int num_q_heads, int head_dim, int max_seq_len,
                                             int seq_block_size, int num_kv_heads);
int sllm_paged_attention(const void* q, const void* k_cache, const void* v_cache, const int32_t* block_table,
                         const int32_t* seq_ids, const int32_t* seq_lens, void* o, void* workspace,
                         int64_t workspace_bytes, float softmax_scale, int num_decoding_seqs, int max_seq_len,
                         int seq_block_size, int cur_layer, int num_layers, int num_q_heads, int num_kv_heads,
                         int block_size, int head_dim, int max_blocks_per_seq, int64_t num_blocks,
                         int64_t q_row_stride, sllm_dtype_t dtype, sllm_stream_t stream);
/* Rank of the KV-cache tensor map the next sm_90a decode or verification launch uses: 4 (one box per 16-token page) where the
 * driver accepts the permuted-stride 4-D map, 2 (the cache as [rows, 128], two boxes per page) where it does not or where
 * SLLM_PAGED_ATTN_KV_MAP=2d is set (read on every launch); -1 while no launch has asked the driver yet. */
int sllm_paged_attention_kv_map_rank(void);

/* ---- Prefill attention: swiftllm/worker/kernels/prefill_attn.py:102-139 (prefill_attention) and the
 * flash_attn_varlen_func call it stands for (swiftllm/worker/layers/transformer_layer.py:86-96).
 * Causal, varlen, packed: q,o [Tp, nq, D]; k,v [Tp, nkv, D]; start_locs/seq_lens int32 [num_prefill_seqs]. */
int sllm_prefill_attention(const void* q, const void* k, const void* v, void* o, const int32_t* prefill_seq_start_locs,
                           const int32_t* prefill_seq_lens, float softmax_scale, int num_prefill_seqs,
                           int max_prefill_len, int64_t num_prefill_tokens, int num_q_heads, int num_kv_heads,
                           int head_dim, int64_t q_row_stride, int64_t k_row_stride, int64_t v_row_stride,
                           sllm_dtype_t dtype, sllm_stream_t stream);

/* ---- Chunked ("prefix-aware") prefill - SURVEY.md §8 f-1.  NEW: the reference's forward cannot express a partial prompt
 * (its prefill attention only sees the packed k/v of the batch: swiftllm/worker/kernels/prefill_attn.py:102-139,
 * swiftllm/worker/layers/transformer_layer.py:86-96; its store always starts at position 0: kvcache_mgmt.py:10-48).
 * Prefill entry i of the batch is the CHUNK of its prompt that covers positions
 * [prefill_prefix_lens[i], prefill_prefix_lens[i] + prefill_seq_lens[i]); earlier positions are already in the cache.
 *   sllm_store_kvcache_chunked   = sllm_store_kvcache with chunk token t written to position prefix + t;
 *   sllm_prefill_attention_paged = causal attention of the chunk's queries (q, o [Tp, nq, D] packed) over positions
 *       0 .. prefix + chunk - 1 read from the paged caches through rows `seq_ids` of the block table (the chunk's own
 *       K/V must have been stored first); query t sees positions <= prefix + t.  With all prefixes 0 it computes
 *       exactly what sllm_prefill_attention computes.  head_dim 64 / 128. */
int sllm_store_kvcache_chunked(const void* k, const void* v, void* k_cache, void* v_cache, const int32_t* block_table,
                               const int32_t* seq_ids, const int32_t* prefill_seq_start_locs,
                               const int32_t* prefill_seq_lens, const int32_t* prefill_prefix_lens,
                               const int32_t* decoding_seq_lens, int num_prefill_seqs, int num_decoding_seqs,
                               int64_t num_prefill_tokens, int max_prefill_len, int cur_layer, int num_layers,
                               int num_kv_heads, int block_size, int head_dim, int max_blocks_per_seq,
                               int64_t k_row_stride, int64_t v_row_stride, sllm_dtype_t dtype, sllm_stream_t stream);
int sllm_prefill_attention_paged(const void* q, const void* k_cache, const void* v_cache, void* o,
                                 const int32_t* block_table, const int32_t* seq_ids,
                                 const int32_t* prefill_seq_start_locs, const int32_t* prefill_seq_lens,
                                 const int32_t* prefill_prefix_lens, float softmax_scale, int num_prefill_seqs,
                                 int max_prefill_len, int64_t num_prefill_tokens, int cur_layer, int num_layers,
                                 int num_q_heads, int num_kv_heads, int block_size, int head_dim,
                                 int max_blocks_per_seq, int64_t num_blocks, int64_t q_row_stride, sllm_dtype_t dtype,
                                 sllm_stream_t stream);

/* ---- Speculative verification (new): the function of sllm_prefill_attention_paged for entries of 1..8 query rows.
 * Entry i has row_counts[i] <= max_rows rows starting at q / o row start_locs[i]; row j sits at position prefix_lens[i] + j
 * (its K/V stored first) and attends to positions 0 .. prefix_lens[i] + j through rows `seq_ids` of the block table.  The
 * entries' rows must tile o's rows [0, num_tokens); max_seq_len >= max_i(prefix_lens[i] + row_counts[i]).  head_dim 128,
 * block_size 16 and (nq / nkv) * max_rows <= 32 run the sm_90a multi-query kernel: one work item per (entry, kv head,
 * split) reads each K/V page once for all the entry's rows and heads, splits as in sllm_paged_attention (over entries x kv
 * heads) merged per row.  Other shapes run sllm_prefill_attention_paged.  workspace: at least
 * sllm_paged_attention_verify_workspace_bytes(...) bytes of device memory (may be NULL when that is 0). */
int64_t sllm_paged_attention_verify_workspace_bytes(int num_seqs, int64_t num_tokens, int num_q_heads, int num_kv_heads,
                                                    int head_dim, int max_seq_len);
int sllm_paged_attention_verify(const void* q, const void* k_cache, const void* v_cache, void* o, const int32_t* block_table,
                                const int32_t* seq_ids, const int32_t* start_locs, const int32_t* row_counts,
                                const int32_t* prefix_lens, void* workspace, int64_t workspace_bytes, float softmax_scale,
                                int num_seqs, int max_rows, int max_seq_len, int64_t num_tokens, int cur_layer, int num_layers,
                                int num_q_heads, int num_kv_heads, int block_size, int head_dim, int max_blocks_per_seq,
                                int64_t num_blocks, int64_t q_row_stride, sllm_dtype_t dtype, sllm_stream_t stream);

/* ---- Block-table maintenance: swiftllm/worker/kernels/block_mgmt.py:26-46, :66-80, :106-127
 * block_table int32 [max_seqs, max_blocks_per_seq]; num_seq_allocated_blocks int32 [max_seqs];
 * is_block_free uint8/bool [num_blocks]; candidate_blocks int64 [sum(block_needed)];
 * block_needed int32 [batch]; block_needed_cumsum int32 [batch] (inclusive). */
int sllm_set_block_table_and_num_seq_alloc_blocks(int32_t* num_seq_allocated_blocks, int32_t* block_table,
                                                  const int64_t* candidate_blocks, const int32_t* seq_ids,
                                                  const int32_t* block_needed, const int32_t* block_needed_cumsum,
                                                  int batch_size, int max_blocks_per_seq, sllm_stream_t stream);
int sllm_unset_block_table_and_num_seq_alloc_blocks(int32_t* num_seq_allocated_blocks, const int32_t* block_table,
                                                    const int32_t* seq_ids, uint8_t* is_block_free, int batch_size,
                                                    int max_blocks_per_seq, sllm_stream_t stream);
/* allocated_cumsum int32 [batch] (inclusive cumsum of num_seq_allocated_blocks[seq_ids]);
 * gathered_block_ids int32 [allocated_cumsum[batch-1]] */
int sllm_gather_allocated_blocks_and_unset(int32_t* num_seq_allocated_blocks, const int32_t* block_table,
                                           const int32_t* seq_ids, uint8_t* is_block_free,
                                           const int32_t* allocated_cumsum, int32_t* gathered_block_ids,
                                           int batch_size, int max_blocks_per_seq, sllm_stream_t stream);
/* Shrink sequence seq_ids[i] to cdiv(target_lens[i], block_size) blocks (new; speculative steps give back blocks that only
 * held rejected drafts): table entries [cdiv(target, block_size), num_seq_allocated_blocks) are marked free and the count is
 * lowered.  A target at or above the current allocation changes nothing.  seq_ids must be distinct. */
int sllm_truncate_blocks_for_seqs(int32_t* num_seq_allocated_blocks, const int32_t* block_table, uint8_t* is_block_free,
                                  const int32_t* seq_ids, const int32_t* target_lens, int batch_size, int block_size,
                                  int max_blocks_per_seq, sllm_stream_t stream);

/* ---- Sync-free block allocation (replaces swiftllm/worker/block_manager.py:43-79: assert + .item() +
 * torch.nonzero).  One launch: for seq i (batch order) needs max(0, cdiv(target_lens[i], block_size) -
 * num_seq_allocated_blocks[seq_ids[i]]) blocks, taken lowest-free-id first - the reference's order - and
 * appended to the block table.  Writes the new ids (int64, batch order) to new_blocks_out (capacity
 * new_blocks_capacity; may be NULL) and {num_new_blocks, error_flag} to status_out (int32[2], error_flag:
 * 1 = not enough free blocks, 2 = a sequence already holds more blocks than its target; on error nothing
 * is modified). */
int sllm_allocate_blocks_for_seqs(int32_t* num_seq_allocated_blocks, int32_t* block_table, uint8_t* is_block_free,
                                  const int32_t* seq_ids, const int32_t* target_lens, int batch_size,
                                  int block_size, int64_t num_blocks, int max_blocks_per_seq,
                                  int64_t* new_blocks_out, int64_t new_blocks_capacity, int32_t* status_out,
                                  sllm_stream_t stream);

/* ---- Shared blocks (new; fork a cached prefix into another sequence).  block_extra_refs int32 [num_blocks]: owners of a block
 * beyond the first, 0 for every free and every freshly allocated block (the allocator above reads only is_block_free).
 * Shared blocks are always the leading blocks of a row.  All three are one launch each, stream-ordered, no host sync.
 *
 * Fork: for every entry i, dst_seq_ids[i]'s row gets the first lens[i] / block_size table entries of src_seq_ids[i]'s row,
 * num_seq_allocated_blocks[dst] is set to that count and each shared block gains one extra owner.  Several entries may name the
 * same src.  The dst rows must be empty; a partial tail block (lens[i] % block_size != 0) is added by a following
 * sllm_allocate_blocks_for_seqs with target lens[i], then filled by sllm_copy_block_tails. */
int sllm_fork_blocks_for_seqs(int32_t* num_seq_allocated_blocks, int32_t* block_table, int32_t* block_extra_refs,
                              const int32_t* src_seq_ids, const int32_t* dst_seq_ids, const int32_t* lens, int batch_size,
                              int block_size, int max_blocks_per_seq, sllm_stream_t stream);
/* For every entry with lens[i] % block_size != 0: copy block lens[i] / block_size of src's row into the same block index of dst's
 * row, ids read from block_table on the device.  Copies block_bytes bytes of k_cache and of v_cache (one block of every layer:
 * [num_blocks][block_bytes] with block_bytes a multiple of 16) and, when token_cache (int32 [num_blocks, block_size]) is not NULL,
 * the block's token page.  batch_size <= 65535. */
int sllm_copy_block_tails(void* k_cache, void* v_cache, int32_t* token_cache, const int32_t* block_table,
                          const int32_t* src_seq_ids, const int32_t* dst_seq_ids, const int32_t* lens, int batch_size,
                          int64_t block_bytes, int block_size, int max_blocks_per_seq, sllm_stream_t stream);
/* Release every block of the given sequences: a block with extra owners loses one, otherwise it becomes free (several owners
 * released in one call: exactly one frees it); num_seq_allocated_blocks[seq] becomes 0.  gathered_block_ids may be NULL; when
 * given, every block id of the sequences is written in batch order as by sllm_gather_allocated_blocks_and_unset
 * (allocated_cumsum: inclusive cumsum of num_seq_allocated_blocks[seq_ids]). */
int sllm_release_blocks_for_seqs(int32_t* num_seq_allocated_blocks, const int32_t* block_table, uint8_t* is_block_free,
                                 int32_t* block_extra_refs, const int32_t* seq_ids, const int32_t* allocated_cumsum,
                                 int32_t* gathered_block_ids, int batch_size, int max_blocks_per_seq, sllm_stream_t stream);

/* ---- Tensor-parallel exchange fused with the op that follows it (new; the reference is single-GPU):
 *   residual <- h(sum over ranks of partial) + residual ;  x_out <- rmsnorm(residual) * weight
 * i.e. the all-reduce after o_proj / down_proj merged with fused_add_rmsnorm_inplace (rmsnorm.py:67-89) in one kernel that
 * reads every rank's partial [num_tokens, hidden] directly over NVLink peer memory, in rank order with fp32 accumulation
 * (bit-identical on all ranks).  host_peer_bufs / host_peer_flags: HOST arrays of `nranks` DEVICE pointers: the partial buffer
 * and the flag pad (uint32 [16 slots][8]) of every rank as mapped into this process (e.g. torch symmetric memory);
 * epoch_state: local device memory, 32 uint32, zeroed once; slot: which of the alternating buffers / flag rows is used.
 * weight == NULL skips the norm (x_out unused). */
int sllm_allreduce_add_rmsnorm(const void* const* host_peer_bufs, void* const* host_peer_flags, int rank, int nranks,
                               int slot, void* epoch_state, void* x_out, void* residual, const void* weight, float eps,
                               int64_t num_tokens, int hidden, sllm_dtype_t dtype, sllm_stream_t stream);

/* Two-shot variant for larger TP degrees: token row t is reduced, added to the residual and normalised by rank t % nranks
 * only, which then stores the normalised row into EVERY rank's x_out buffer (host_peer_xout: HOST array of `nranks` DEVICE
 * pointers, symmetric memory like the partial buffers; the result appears in this rank's own buffer when the call's kernel
 * has finished).  Remote traffic per rank 2*(N-1)/N*T*H instead of (N-1)*T*H bytes; two flag barriers (signal-pad rows
 * `slot` and 8 + `slot`, slot < 8).  `residual` is only maintained for the rows this rank owns; weight is required.
 * mc_buf / mc_xout: NVLS multicast addresses (DEVICE pointers) of the partial buffer of this slot and of x_out, or both NULL.
 * When given, the reduction is ONE multimem.ld_reduce per 16 bytes (the NVSwitch sums all ranks' copies, fp32 accumulation)
 * and the broadcast ONE multimem.st, instead of N peer loads / stores. */
int sllm_allreduce_add_rmsnorm_2shot(const void* const* host_peer_bufs, void* const* host_peer_xout,
                                     void* const* host_peer_flags, const void* mc_buf, void* mc_xout, int rank, int nranks,
                                     int slot, void* epoch_state, void* residual, const void* weight, float eps,
                                     int64_t num_tokens, int hidden, sllm_dtype_t dtype, sllm_stream_t stream);

/* Low-latency variant for decode-sized exchanges (csrc/allreduce_ll.cu): same result as the two-shot call (row t reduced, added
 * to the residual and normalised by rank t % nranks, residual maintained for owned rows only), but WITHOUT barriers: partial rows
 * are pushed to their owner and normalised rows to every rank as 16-byte lines {payload, epoch tag, payload, epoch tag} that the
 * receiver polls ("LL" protocol); the complete plain rows appear in x_out (local).  partial: this rank's [num_tokens, hidden]
 * GEMM output (local).  host_peer_rs_recv / host_peer_ag_recv: HOST arrays of `nranks` DEVICE pointers to every rank's receive
 * buffers OF THIS SLOT (symmetric memory, zeroed once): rs_recv [nranks][rows_per_rank][hidden], ag_recv [>= num_tokens][hidden],
 * 4 bytes per element.  mc_ag_recv: NVLS multicast address of ag_recv (one multimem.st per line instead of nranks-1 peer stores)
 * or NULL.  num_tokens <= nranks * rows_per_rank.  epoch_state as above (shared with the other exchange calls of the slot). */
int sllm_allreduce_add_rmsnorm_ll(const void* partial, void* const* host_peer_rs_recv, void* const* host_peer_ag_recv,
                                  void* mc_ag_recv, int rank, int nranks, int slot, void* epoch_state, void* x_out,
                                  void* residual, const void* weight, float eps, int64_t num_tokens, int hidden,
                                  int64_t rows_per_rank, sllm_dtype_t dtype, sllm_stream_t stream);

/* ---- Block swapping: csrc/src/block_swapping.cpp:22-85 (swiftllm_c.swap_blocks, csrc/src/entrypoints.cpp:5-7)
 * host_src_ids/host_dst_ids: HOST arrays of n block ids.  k_swap/v_swap: HOST memory (pinned or pageable),
 * k_cache/v_cache: device.  block_bytes = bytes of one block (all layers/heads) of k_cache.
 * Consecutive (src,dst) runs are coalesced into one copy each, as the reference does. */
int sllm_swap_blocks(const int64_t* host_src_ids, const int64_t* host_dst_ids, int64_t n, int is_swap_in,
                     void* k_cache, void* v_cache, void* host_k_swap, void* host_v_swap, int64_t block_bytes,
                     sllm_stream_t stream);

/* Sync-free variant (new, SURVEY.md §8 f-4): src_ids / dst_ids are DEVICE arrays (int64) - the gathered source ids and the
 * newly allocated target ids never travel to the host (the reference does `.tolist()` twice per swap, model.py:374-377) - and
 * one kernel moves every block between the cache and the swap space, which must be pinned, device-mapped host memory
 * (cudaHostAlloc / torch pin_memory).  Same data movement as sllm_swap_blocks. */
int sllm_swap_blocks_gathered(const int64_t* src_ids, const int64_t* dst_ids, int64_t n, int is_swap_in, void* k_cache,
                              void* v_cache, void* host_k_swap, void* host_v_swap, int64_t block_bytes,
                              sllm_stream_t stream);

/* ---- Token sampling (new; the reference decodes greedily only, swiftllm/worker/layers/post_layer.py:39):
 * logits [num_rows, logits_row_stride] 16-bit, the first vocab_size columns of row i are the vocabulary entries
 * vocab_offset .. vocab_offset + vocab_size - 1 (a vocabulary shard under tensor parallelism, else vocab_offset 0).
 * Per-row DEVICE arrays [num_rows]: temperature (<= 0: greedy, == torch.argmax), top_k (<= 0 or >= vocab_size: off), top_p
 * (>= 1: off), seed, pos (the sequence length after this step's input; the noise counter).  Ties at the top-k / top-p boundary
 * are kept.  out_tokens int64 [num_rows]: GLOBAL token ids.  out_pairs fp32 [num_rows, 2] or NULL: (best score, global index),
 * the score being the logit for greedy rows and logit / T + Gumbel noise otherwise; the pairs of vocabulary shards merge into
 * the unsharded result for rows without top-k / top-p (largest score, then smallest index).  Deterministic; a row's token
 * depends on its logits and parameters only.  Rejected before launch: unknown dtype, vocab_size <= 0 or larger than 8
 * shared-memory slices (about 819k entries), global indices >= 2^24, a row stride below vocab_size, null pointers. */
int sllm_sample_tokens(const void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride,
                       int64_t vocab_offset, const float* temperature, const int32_t* top_k, const float* top_p,
                       const int64_t* seed, const int32_t* pos, int64_t* out_tokens, float* out_pairs, sllm_dtype_t dtype,
                       sllm_stream_t stream);

/* ---- Truncation filters (new): sllm_sample_tokens with the per-row DEVICE arrays [num_rows] min_p (0: off), typical_p (>= 1:
 * off), xtc_threshold and xtc_probability (0: off), applied in this order after min-p: top-k, top-p, typical-p, XTC.  With
 * x = (m - l) / T, q = expf(-x) and w = round(q * 2^40) over the survivors of the previous filter (Z their exact sum):
 * min-p keeps key >= the smallest key with q >= min_p (before top-k and top-p); typical-p keeps |x - c| <= delta, c =
 * fp32(E / Z) with E = sum round(fp32(q * x) * 2^40), delta the smallest distance whose survivors weigh >= typical_p * Z; XTC,
 * when u = Philox(seed, counter (0, pos, 1, 0)) word 0 drawn as the Gumbel noise's u is < xtc_probability and at least two
 * finite survivors have w >= xtc_threshold * Z, drops the survivors above the smallest key among those (its ties kept; a
 * -inf id is never counted, so threshold 0 stops at the least likely finite survivor).  Every kept
 * set is a key interval; greedy and bad rows, the draw and out_pairs are those of sllm_sample_tokens, and with every filter
 * off the result is its result.  Rejected before launch: what sllm_sample_tokens rejects, and null filter arrays. */
int sllm_sample_tokens_truncated(const void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride,
                                 int64_t vocab_offset, const float* temperature, const int32_t* top_k, const float* top_p,
                                 const int64_t* seed, const int32_t* pos, int64_t* out_tokens, float* out_pairs,
                                 const float* min_p, const float* typical_p, const float* xtc_threshold,
                                 const float* xtc_probability, sllm_dtype_t dtype, sllm_stream_t stream);

/* ---- Token log-probabilities (new; the reference returns token ids only): log_softmax of the raw 16-bit logits (no
 * temperature, no top-k / top-p), logits as in sllm_sample_tokens with the whole vocabulary in each row.
 * m = the largest logit, Z = sum_v round(expf(l_v - m) * 2^40) as an exact 64-bit integer, lse = m + logf(Z * 2^-40) and
 * logprob(v) = l_v - lse, all fp32.  token_ids int64 [num_rows]: out_token_logprob fp32 [num_rows] = logprob(token_ids[i]), NaN
 * for an id outside [0, vocab_size).  top_n in [0, 20]: out_top_ids int32 / out_top_logprobs fp32 [num_rows, top_n] = the
 * min(top_n, vocab_size) ids with the largest logits, ordered by (logit desc, id asc), -0 == +0; later entries are id -1, NaN.
 * A row holding a NaN or +inf (or only -inf) gives NaN logprobs; a -inf logit gives -inf.  Deterministic: a row's outputs
 * depend on its logits only.  Rejected before launch: unknown dtype, vocab_size <= 0 or larger than 8 shared-memory slices,
 * top_n outside [0, 20], a row stride below vocab_size, num_rows outside [0, 2^20], null pointers (out_top_* may be NULL
 * when top_n is 0). */
int sllm_token_logprobs(const void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride,
                        const int64_t* token_ids, int top_n, float* out_token_logprob, int32_t* out_top_ids,
                        float* out_top_logprobs, sllm_dtype_t dtype, sllm_stream_t stream);

/* ---- Prompt log-probabilities (new): sllm_token_logprobs' values for many rows at once (every row of a prefill), plus ranks.
 * target_ids int32 [num_rows]: out_logprob fp32 [num_rows] = logprob(target_ids[i]), bit-identical to sllm_token_logprobs on
 * the same row; out_rank int32 [num_rows] = 1 + the number of ids whose logit is strictly greater (-0 == +0; NaN and inf in the
 * order of sllm_token_logprobs' top-N), so a greedy token has rank 1; an id outside [0, vocab_size) gives NaN and rank -1.
 * top_n in [0, 20]: out_top_ids / out_top_logprobs [num_rows, top_n] as in sllm_token_logprobs.  One CTA per row, no clusters.
 * Deterministic: a row's outputs depend on its logits and target only.  Rejected before launch: unknown dtype, vocab_size
 * outside [1, 2^24], top_n outside [0, 20], a row stride below vocab_size, num_rows outside [0, 2^24], null pointers
 * (out_top_* may be NULL when top_n is 0). */
int sllm_prompt_logprobs(const void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride,
                         const int32_t* target_ids, int top_n, float* out_logprob, int32_t* out_rank, int32_t* out_top_ids,
                         float* out_top_logprobs, sllm_dtype_t dtype, sllm_stream_t stream);

/* ---- Repetition / frequency / presence penalties (new; the reference has no sampling controls), IN PLACE on logits laid out
 * as in sllm_sample_tokens (a vocabulary shard with vocab_offset works).  Per-row DEVICE arrays [num_rows]:
 * repetition_penalty, frequency_penalty, presence_penalty (a row with 1, 0, 0 is skipped: nothing read, recorded or modified),
 * seq_ids (block-table rows), pos (the sequence length after this step's input).  The row's history is positions [0, pos) of its
 * sequence: [0, pos - n_new) read from token_cache int32 [num_blocks, block_size] through block_table int32
 * [*, block_table_stride] (entries id | is_output << 31), the rest its n_new new tokens in input_ids: rows below
 * num_prefill_rows are prefill entries (n_new = prefill_seq_lens[i] prompt tokens ending at input_ids[last_token_indices[i]]),
 * the others decode rows (one output token, input_ids[last_token_indices[i]]).  For every id v of the shard seen in the history:
 * l = l > 0 ? l / r : l * r, then l -= f * c_out(v) + (c_out(v) > 0 ? p : 0), c_out counting output tokens, fp32 without
 * contraction and one rounding to the storage dtype; other entries keep their bits.  The new tokens are then written to
 * positions [pos - n_new, pos) of the pages.  Ids outside the shard, unmapped positions and block ids outside [0, num_blocks)
 * are skipped.  Deterministic (exact integer counts).  Rejected before launch: unknown dtype, vocab_size <= 0 or larger than 8
 * shared-memory slices of 4-byte slots (about 409k entries), global indices >= 2^31, a row stride below vocab_size, block_size
 * outside [1, 65536], a bad block_table_stride, num_blocks < 0, num_prefill_rows outside [0, num_rows], num_rows outside
 * [0, 2^20], null pointers (prefill_seq_lens may be NULL when num_prefill_rows is 0). */
int sllm_apply_penalties(void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride, int64_t vocab_offset,
                         const float* repetition_penalty, const float* frequency_penalty, const float* presence_penalty,
                         const int32_t* seq_ids, const int32_t* pos, const int32_t* input_ids,
                         const int32_t* last_token_indices, const int32_t* prefill_seq_lens, int num_prefill_rows,
                         const int32_t* block_table, int block_table_stride, int block_size, int32_t* token_cache,
                         int64_t num_blocks, sllm_dtype_t dtype, sllm_stream_t stream);

/* ---- N-gram repetition controls (new): sllm_apply_penalties plus a no-repeat n-gram ban and the DRY penalty, from the same one
 * read of the history in the same launch.  Extra per-row DEVICE arrays [num_rows]: no_repeat_ngram_size n (0: no ban),
 * dry_allowed_length A, dry_multiplier (0: no DRY), dry_base, and dry_breakers int32 [num_rows, 16] (global ids, -1 unused).
 * With x[0, L) the history (L = pos, ids compared without the output bit; unmapped positions match nothing), m(j) the longest
 * m <= min(j, 50) with x[j - k] == x[L - k] for k = 1 .. m, and M(v) the largest m(j) over the j with x[j] == v: the ban sets
 * l = -inf where M(v) >= n - 1; DRY, with b the smallest k >= 1 such that x[L - k] is a breaker (infinite if none) and
 * D(v) = min(M(v), b - 1) for a v that is no breaker, subtracts q = multiplier * base^(D - A) (fp32, multiplied out in order)
 * where D >= A.  Per entry: the penalties (rows with any of them), DRY, the ban, one rounding; untouched entries keep their
 * bits.  A row with all eight controls off is skipped.  8-byte cluster slots: vocab_size up to about 204k entries.  Rejected
 * before launch: what sllm_apply_penalties rejects, and null control arrays. */
int sllm_apply_penalties_ngram(void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride,
                               int64_t vocab_offset, const float* repetition_penalty, const float* frequency_penalty,
                               const float* presence_penalty, const int32_t* seq_ids, const int32_t* pos,
                               const int32_t* input_ids, const int32_t* last_token_indices, const int32_t* prefill_seq_lens,
                               int num_prefill_rows, const int32_t* block_table, int block_table_stride, int block_size,
                               int32_t* token_cache, int64_t num_blocks, const int32_t* no_repeat_ngram_size,
                               const int32_t* dry_allowed_length, const float* dry_multiplier, const float* dry_base,
                               const int32_t* dry_breakers, sllm_dtype_t dtype, sllm_stream_t stream);

/* ---- Constrained decoding (new): allowed-token bitmasks and logit bias, IN PLACE on logits laid out as in sllm_sample_tokens
 * (a vocabulary shard with vocab_offset works; bits and bias ids are global indices).  Per-row DEVICE arrays [num_rows]:
 * mask_index (-1: no mask; else a row of masks uint32 [num_masks, mask_words], bit v % 32 of word v / 32 set = id v allowed)
 * and bias_index (-1: no bias; else an entry e of the CSR arrays bias_starts int32 [num_entries + 1], bias_ids int32 [num_bias]
 * (distinct within an entry) and bias_values fp32 [num_bias]).  Every disallowed id becomes -inf; then every allowed id with a
 * bias becomes round(float(l) + b), one fp32 add and one rounding to the storage dtype.  Rows with neither are not touched;
 * allowed unbiased entries keep their bits.  Out-of-range mask / bias indices and bias ids outside the shard are skipped.
 * Deterministic: each logit is written by at most one thread.  Rejected before launch: unknown dtype, vocab_size <= 0, global
 * indices >= 2^31, a row stride below vocab_size, mask_words that do not cover vocab_offset + vocab_size ids (when num_masks >
 * 0), negative or too large counts, null pointers (masks / bias_starts / bias_ids and bias_values may be NULL when their count
 * is 0).  num_rows == 0 is a no-op. */
int sllm_constrain_logits(void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride, int64_t vocab_offset,
                          const int32_t* mask_index, const uint32_t* masks, int64_t num_masks, int mask_words,
                          const int32_t* bias_index, const int32_t* bias_starts, int64_t num_entries, const int32_t* bias_ids,
                          const float* bias_values, int64_t num_bias, sllm_dtype_t dtype, sllm_stream_t stream);

/* ---- Multi-LoRA (new): per-request low-rank adapters added to a projection's 16-bit output y [num_rows, out_features].
 * tiles: DEVICE int32 triples (first row, rows, slot), num_tiles of them; a tile with rows outside [1, 64], a slot outside
 * [0, max_loras), rows past num_rows, or slice_mask[slot] == 0 is skipped (rows 0 pads a CUDA graph's fixed tile count).
 * sllm_lora_shrink: u[t, j] = round(sum_k x[t, k] * A[j, k]) for j < u_cols, A = lora_a + slot * a_slot_stride ([u_cols,
 * in_features] row-major, the adapter's S stacked slices of R rows), fp32 accumulation in an order fixed by in_features alone.
 * sllm_lora_expand: y[t, n] = round(float(y[t, n]) + scales[slot] * sum_j u[t, sl * rank + j] * B[n, j]), B = lora_b + slot *
 * b_slot_stride ([out_features, rank] row-major), sl the slice of column n ([0, slice1), [slice1, slice2), [slice2,
 * out_features)); one fp32 multiply, one fp32 add, one rounding.  Columns of a slice whose bit (1 << sl) is clear in
 * slice_mask[slot] are not written.  Every element of y is written by at most one thread.  Rejected before launch: unknown dtype,
 * counts out of range, in_features not a positive multiple of 32, rank not 16 / 32 / 48 / 64, out_features or slice ends not
 * multiples of 8, strides that do not cover a row or are misaligned, null or misaligned pointers.  num_tiles == 0 is a no-op. */
int sllm_lora_shrink(const void* x, int64_t x_row_stride, int64_t num_rows, int in_features, void* u, int64_t u_row_stride,
                     const void* lora_a, int64_t a_slot_stride, int u_cols, const int32_t* tiles, int64_t num_tiles,
                     const int32_t* slice_mask, int max_loras, sllm_dtype_t dtype, sllm_stream_t stream);
int sllm_lora_expand(void* y, int64_t y_row_stride, int64_t num_rows, int out_features, const void* u, int64_t u_row_stride,
                     const void* lora_b, int64_t b_slot_stride, int rank, int slice1, int slice2, const int32_t* tiles,
                     int64_t num_tiles, const int32_t* slice_mask, const float* scales, int max_loras, sllm_dtype_t dtype,
                     sllm_stream_t stream);

/* ---- FP8 weights (new): per-token e4m3 quantization of GEMM inputs, one CTA per row.  For a row y of the storage dtype:
 * s = fmaxf(amax(|y|) / 448.f, 0x1p-126f) (fp32, IEEE division), q_j = e4m3 round-to-nearest-even with saturation to +-448 of
 * y_j / s (fp32 IEEE division), so y_j ~= q_j * s.  Outputs: q (e4m3 bytes, [rows, cols] row-major) and scales (fp32 [rows]).
 * sllm_fused_add_rmsnorm_quant_fp8: y = the fused add+RMSNorm row of sllm_fused_add_rmsnorm_inplace (the residual is updated
 * exactly as there); x is read, not written.  sllm_silu_and_mul_quant_fp8: y = sllm_silu_and_mul_inplace's row of [up | gate]
 * (x read, not written; row stride >= 2F).  sllm_quant_fp8_rows: y = the given rows (row stride x_row_stride elements).
 * Rejected before launch: unknown dtype, a row length not a positive multiple of 16 (up to 65536 for the first two), counts >=
 * 2^31, strides that do not cover a row or are not multiples of 8, null or misaligned pointers (16-bit operands 16-byte, q
 * 8-byte aligned).  Zero rows are a no-op. */
int sllm_fused_add_rmsnorm_quant_fp8(const void* x, void* residual, const void* weight, float eps, int64_t num_tokens,
                                     int hidden, void* xq, float* scales, sllm_dtype_t dtype, sllm_stream_t stream);
int sllm_silu_and_mul_quant_fp8(const void* x, int64_t x_row_stride, int64_t num_tokens, int64_t F, void* out, float* scales,
                                sllm_dtype_t dtype, sllm_stream_t stream);
int sllm_quant_fp8_rows(const void* x, int64_t x_row_stride, int64_t num_rows, int64_t cols, void* out, float* scales,
                        sllm_dtype_t dtype, sllm_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SWIFTLLM_B200_H */
