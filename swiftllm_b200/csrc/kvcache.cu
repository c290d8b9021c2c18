// KV-cache page store and block-table maintenance (exact integer / byte work, HBM- or latency-bound).
// Reference: swiftllm/worker/kernels/kvcache_mgmt.py, swiftllm/worker/kernels/block_mgmt.py,
//            swiftllm/worker/block_manager.py:43-79 (allocation order).
// Cache layout (part of the contract, model.py:138-148): [num_blocks, num_layers, nkv, block_size, D].
#include "common.cuh"

namespace sllm {

// ------------------------------------------------------------------ store_kvcache, prefill part
// kvcache_mgmt.py:10-48.  grid (cdiv(max_prefill_len, bs), num_prefill_seqs); one CTA moves one page worth of
// tokens: source rows [tok][head][D] -> page [head][tok][D].  16-byte vectors, both sides coalesced per
// D-row.  Algorithmic bytes: 4 * T * nkv * D * sizeof(T) (K and V, read + write).
// PREFIX (chunked prefill, not in the reference): token t of chunk b lands at position prefix_lens[b] + t of its
// sequence, so the first page of a chunk may be entered in the middle; grid.x = cdiv(max_chunk_len, bs) + 1.
template <typename T, bool PREFIX>
__global__ void __launch_bounds__(256) store_kv_prefill_kernel(
    const T* __restrict__ k, const T* __restrict__ v, T* __restrict__ k_cache, T* __restrict__ v_cache,
    const int32_t* __restrict__ block_table, const int32_t* __restrict__ seq_ids,
    const int32_t* __restrict__ start_locs, const int32_t* __restrict__ seq_lens, int cur_layer, int num_layers,
    int nkv, int bs, int D, int max_blocks_per_seq, int64_t k_stride, int64_t v_stride,
    const int32_t* __restrict__ prefix_lens) {
    const int b = blockIdx.y;
    const int len = seq_lens[b];
    int pb = blockIdx.x;          // page of the sequence this CTA fills
    int off0 = 0;                 // first slot of the page that is written
    int ntok;
    int64_t row0;                 // source row of the first token written
    if constexpr (PREFIX) {
        const int pre = prefix_lens[b];
        pb += pre / bs;
        const int lo = max(pb * bs, pre), hi = min(pb * bs + bs, pre + len);
        if (lo >= hi) return;
        off0 = lo - pb * bs;
        ntok = hi - lo;
        row0 = start_locs[b] + (lo - pre);
    } else {
        const int tok0 = pb * bs;
        if (tok0 >= len) return;
        ntok = min(bs, len - tok0);
        row0 = start_locs[b] + tok0;
    }
    const int64_t blk = block_table[(int64_t)seq_ids[b] * max_blocks_per_seq + pb];
    const int64_t dst0 = (blk * num_layers + cur_layer) * (int64_t)nkv * bs * D + (int64_t)off0 * D;
    const int cpr = D >> 3;                     // 16-byte chunks per D-row
    const int items = ntok * nkv * cpr;
    for (int i = threadIdx.x; i < items; i += blockDim.x) {
        const int c = i % cpr, h = (i / cpr) % nkv, t = i / (cpr * nkv);
        const int64_t so = (int64_t)h * D + 8 * c;
        const int64_t d = dst0 + ((int64_t)h * bs + t) * D + 8 * c;
        st_vec8(k_cache + d, ld_vec8_stream(k + (row0 + t) * k_stride + so));
        st_vec8(v_cache + d, ld_vec8_stream(v + (row0 + t) * v_stride + so));
    }
}

// ------------------------------------------------------------------ store_kvcache, decode part
// kvcache_mgmt.py:50-79.  grid (num_decoding_seqs); new row goes to position len-1.
template <typename T>
__global__ void __launch_bounds__(128) store_kv_decode_kernel(
    const T* __restrict__ k, const T* __restrict__ v, T* __restrict__ k_cache, T* __restrict__ v_cache,
    const int32_t* __restrict__ block_table, const int32_t* __restrict__ seq_ids,
    const int32_t* __restrict__ seq_lens, int cur_layer, int num_layers, int nkv, int bs, int D,
    int max_blocks_per_seq, int64_t k_stride, int64_t v_stride) {
    const int b = blockIdx.x;
    const int pos = seq_lens[b] - 1;
    const int64_t blk = block_table[(int64_t)seq_ids[b] * max_blocks_per_seq + pos / bs];
    const int off = pos % bs;
    const int64_t dst0 = (blk * num_layers + cur_layer) * (int64_t)nkv * bs * D + (int64_t)off * D;
    const int cpr = D >> 3;
    for (int i = threadIdx.x; i < nkv * cpr; i += blockDim.x) {
        const int c = i % cpr, h = i / cpr;
        const int64_t so = (int64_t)h * D + 8 * c;
        const int64_t d = dst0 + (int64_t)h * bs * D + 8 * c;
        st_vec8(k_cache + d, ld_vec8(k + (int64_t)b * k_stride + so));
        st_vec8(v_cache + d, ld_vec8(v + (int64_t)b * v_stride + so));
    }
}

// ------------------------------------------------------------------ block_mgmt.py kernels (one warp per sequence)
__global__ void set_block_table_kernel(int32_t* nsab, int32_t* block_table, const int64_t* cand, const int32_t* seq_ids,
                                       const int32_t* need, const int32_t* need_cumsum, int batch, int mbps) {
    const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= batch) return;
    const int lane = threadIdx.x & 31;
    const int64_t sid = seq_ids[b];
    const int n = need[b];
    const int start = need_cumsum[b] - n;
    const int have = nsab[sid];
    for (int i = lane; i < n; i += 32) block_table[sid * mbps + have + i] = (int32_t)cand[start + i];
    __syncwarp();
    if (lane == 0) nsab[sid] = have + n;
}

template <bool GATHER>
__global__ void unset_block_table_kernel(int32_t* nsab, const int32_t* block_table, const int32_t* seq_ids,
                                         uint8_t* is_free, const int32_t* cumsum, int32_t* gathered, int batch,
                                         int mbps) {
    const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= batch) return;
    const int lane = threadIdx.x & 31;
    const int64_t sid = seq_ids[b];
    const int n = nsab[sid];
    const int out0 = GATHER ? (b > 0 ? cumsum[b - 1] : 0) : 0;
    for (int i = lane; i < n; i += 32) {
        const int32_t id = block_table[sid * mbps + i];
        if (GATHER) gathered[out0 + i] = id;
        is_free[id] = 1;
    }
    __syncwarp();
    if (lane == 0) nsab[sid] = 0;
}

// Give back the blocks past ceil(target_lens[b] / bs) of each sequence (speculative steps: blocks that only held rejected
// drafts).  One warp per sequence; a target at or above the allocation changes nothing.
__global__ void truncate_blocks_kernel(int32_t* __restrict__ nsab, const int32_t* __restrict__ block_table,
                                       uint8_t* __restrict__ is_free, const int32_t* __restrict__ seq_ids,
                                       const int32_t* __restrict__ target_lens, int batch, int bs, int mbps) {
    const int b = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= batch) return;
    const int64_t sid = seq_ids[b];
    const int n = nsab[sid];
    const int keep = min(n, (target_lens[b] + bs - 1) / bs);
    for (int i = keep + lane; i < n; i += 32) is_free[block_table[sid * mbps + i]] = 1;
    __syncwarp();
    if (lane == 0) nsab[sid] = keep;
}

// ------------------------------------------------------------------ shared blocks (fork)
// extra_refs[block] = owners beyond the first (0 for every free block and every freshly allocated one), so the allocator,
// which reads only is_free, needs no change.  Shared blocks are always the leading blocks of a row (a fork shares [0, P / bs)).

// dst_ids[b] takes the first lens[b] / bs blocks of src_ids[b]'s row; one warp per entry.  Several entries may name the same src:
// the counts are atomic.  The tail block (lens % bs != 0) is appended afterwards by allocate_blocks_kernel.
__global__ void fork_blocks_kernel(int32_t* __restrict__ nsab, int32_t* __restrict__ block_table, int32_t* __restrict__ extra_refs,
                                   const int32_t* __restrict__ src_ids, const int32_t* __restrict__ dst_ids,
                                   const int32_t* __restrict__ lens, int batch, int bs, int mbps) {
    const int b = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= batch) return;
    const int64_t src = src_ids[b], dst = dst_ids[b];
    const int n = lens[b] / bs;
    for (int i = lane; i < n; i += 32) {
        const int32_t id = block_table[src * mbps + i];
        block_table[dst * mbps + i] = id;
        atomicAdd(extra_refs + id, 1);
    }
    if (lane == 0) nsab[dst] = n;
}

// Copy block lens[b] / bs of src into the same block index of dst, for every entry with lens[b] % bs != 0: the K and V pages of
// every layer (one block of all layers is `block_bytes` contiguous bytes, DESIGN §2) and the block's token page.  Both ids are read
// from the block table.  grid (cdiv(block_bytes, kTailChunk), batch, 2): blockIdx.z picks K or V; each CTA moves one 32 KiB chunk
// with 8 independent 16-byte loads per thread in flight.
constexpr int kTailThreads = 256, kTailUnroll = 8, kTailChunk = kTailThreads * kTailUnroll * 16;

__global__ void __launch_bounds__(kTailThreads) copy_block_tails_kernel(
    char* __restrict__ k_cache, char* __restrict__ v_cache, int32_t* __restrict__ token_cache,
    const int32_t* __restrict__ block_table, const int32_t* __restrict__ src_ids, const int32_t* __restrict__ dst_ids,
    const int32_t* __restrict__ lens, int64_t block_bytes, int bs, int mbps) {
    const int b = blockIdx.y;
    const int len = lens[b];
    if (len % bs == 0) return;
    const int j = len / bs;
    const int64_t sblk = block_table[(int64_t)src_ids[b] * mbps + j];
    const int64_t dblk = block_table[(int64_t)dst_ids[b] * mbps + j];
    char* base = blockIdx.z ? v_cache : k_cache;
    const uint4* s = reinterpret_cast<const uint4*>(base + sblk * block_bytes);
    uint4* d = reinterpret_cast<uint4*>(base + dblk * block_bytes);
    const int64_t nvec = block_bytes >> 4;
    const int64_t v0 = (int64_t)blockIdx.x * (kTailChunk >> 4) + threadIdx.x;
    uint4 r[kTailUnroll];
#pragma unroll
    for (int u = 0; u < kTailUnroll; u++) {
        const int64_t v = v0 + u * kTailThreads;
        if (v < nvec) r[u] = __ldcs(s + v);
    }
#pragma unroll
    for (int u = 0; u < kTailUnroll; u++) {
        const int64_t v = v0 + u * kTailThreads;
        if (v < nvec) __stcs(d + v, r[u]);
    }
    if (token_cache && blockIdx.x == 0 && blockIdx.z == 0)
        for (int t = threadIdx.x; t < bs; t += kTailThreads) token_cache[dblk * bs + t] = token_cache[sblk * bs + t];
}

// Drop one owner of every block of each sequence: a block with extra owners loses one, the releaser that finds none frees it
// (so of several owners released in one launch exactly one frees the block).  GATHER also writes every block id of the
// sequences in batch order (the swap plan).  One warp per sequence.
template <bool GATHER>
__global__ void release_blocks_kernel(int32_t* __restrict__ nsab, const int32_t* __restrict__ block_table,
                                      uint8_t* __restrict__ is_free, int32_t* __restrict__ extra_refs,
                                      const int32_t* __restrict__ seq_ids, const int32_t* __restrict__ cumsum,
                                      int32_t* __restrict__ gathered, int batch, int mbps) {
    const int b = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= batch) return;
    const int64_t sid = seq_ids[b];
    const int n = nsab[sid];
    const int out0 = GATHER ? (b > 0 ? cumsum[b - 1] : 0) : 0;
    for (int i = lane; i < n; i += 32) {
        const int32_t id = block_table[sid * mbps + i];
        if (GATHER) gathered[out0 + i] = id;
        int old = extra_refs[id];
        while (old > 0) {
            const int prev = atomicCAS(extra_refs + id, old, old - 1);
            if (prev == old) break;
            old = prev;
        }
        if (old == 0) is_free[id] = 1;
    }
    __syncwarp();
    if (lane == 0) nsab[sid] = 0;
}

// ------------------------------------------------------------------ sync-free allocation
// Replaces block_manager.py:43-79 (assert(...).all() + sum().item() + torch.nonzero()[:n]) by one launch of a
// single CTA.  Ordering contract (bit-exact block ids): the n lowest-numbered free blocks, ascending, are
// handed to the sequences in batch order - exactly what `torch.nonzero(is_block_free)[:n]` followed by
// block_mgmt.py:19-23 produces.
__device__ __forceinline__ int block_exclusive_scan(int v, int* warp_sums, int& block_total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int n = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += n;
    }
    __syncthreads();                      // protect warp_sums from the previous use
    if (lane == 31) warp_sums[warp] = inc;
    __syncthreads();
    int base = 0, tot = 0;
    for (int w = 0; w < nwarps; w++) {
        int s = warp_sums[w];
        if (w < warp) base += s;
        tot += s;
    }
    block_total = tot;
    return base + inc - v;
}

__global__ void __launch_bounds__(1024) allocate_blocks_kernel(
    int32_t* __restrict__ nsab, int32_t* __restrict__ block_table, uint8_t* __restrict__ is_free,
    const int32_t* __restrict__ seq_ids, const int32_t* __restrict__ target_lens, int batch, int bs,
    int64_t num_blocks, int mbps, int64_t* __restrict__ new_out, int64_t cap, int32_t* __restrict__ status) {
    extern __shared__ int32_t sm[];       // start[batch+1] exclusive scan of need, have[batch]
    int32_t* start = sm;
    int32_t* have = sm + batch + 1;
    __shared__ int warp_sums[32];
    __shared__ int s_err;
    if (threadIdx.x == 0) s_err = 0;
    __syncthreads();

    // 1. per-sequence need and its exclusive scan (batch order)
    int carry = 0;
    for (int b0 = 0; b0 < batch; b0 += blockDim.x) {
        const int b = b0 + threadIdx.x;
        int need = 0;
        if (b < batch) {
            const int h = nsab[seq_ids[b]];
            const int tgt = (target_lens[b] + bs - 1) / bs;
            if (h > tgt) atomicOr(&s_err, 2);
            if (tgt > mbps) atomicOr(&s_err, 4);
            need = max(0, tgt - h);
            have[b] = h;
        }
        int tot;
        const int ex = block_exclusive_scan(need, warp_sums, tot);
        if (b < batch) start[b] = carry + ex;
        carry += tot;
    }
    const int total = carry;
    if (threadIdx.x == 0) start[batch] = total;
    __syncthreads();

    // 2. count the free blocks (nothing may be modified if there are too few)
    const int64_t per_iter = (int64_t)blockDim.x * 16;
    int free_cnt = 0;
    if (s_err == 0 && total > 0) {
        int mine = 0;
        for (int64_t base = 0; base < num_blocks; base += per_iter) {
            const int64_t p = base + (int64_t)threadIdx.x * 16;
            if (p + 16 <= num_blocks && ((reinterpret_cast<uintptr_t>(is_free + p) & 15) == 0)) {
                const uint4 u = *reinterpret_cast<const uint4*>(is_free + p);
                const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
                for (int j = 0; j < 4; j++) mine += __popc(__vcmpne4(w[j], 0u) & 0x01010101u);
            } else {
                for (int j = 0; j < 16 && p + j < num_blocks; j++) mine += is_free[p + j] != 0;
            }
        }
        int tot;
        block_exclusive_scan(mine, warp_sums, tot);
        free_cnt = tot;
        if (free_cnt < total && threadIdx.x == 0) s_err |= 1;
    }
    __syncthreads();
    const int err = s_err | ((new_out != nullptr && total > cap) ? 8 : 0);
    if (threadIdx.x == 0) { status[0] = err ? 0 : total; status[1] = err; }
    if (err != 0 || total == 0) return;

    // 3. hand out the `total` lowest free ids in ascending order
    int running = 0;
    for (int64_t base = 0; base < num_blocks && running < total; base += per_iter) {
        const int64_t p = base + (int64_t)threadIdx.x * 16;
        uint8_t f[16];
        int mine = 0;
#pragma unroll
        for (int j = 0; j < 16; j++) {
            f[j] = (p + j < num_blocks) ? is_free[p + j] : 0;
            mine += f[j] != 0;
        }
        int tot;
        int rank = running + block_exclusive_scan(mine, warp_sums, tot);
#pragma unroll
        for (int j = 0; j < 16; j++) {
            if (f[j] && rank < total) {
                // sequence that owns candidate #rank: last b with start[b] <= rank
                int lo = 0, hi = batch;             // invariant start[lo] <= rank < start[hi]
                while (hi - lo > 1) {
                    const int mid = (lo + hi) >> 1;
                    if (start[mid] <= rank) lo = mid; else hi = mid;
                }
                const int64_t sid = seq_ids[lo];
                block_table[sid * mbps + have[lo] + (rank - start[lo])] = (int32_t)(p + j);
                if (new_out) new_out[rank] = p + j;
                is_free[p + j] = 0;
            }
            rank += f[j] != 0;
        }
        running += tot;
    }
    __syncthreads();
    for (int b = threadIdx.x; b < batch; b += blockDim.x) nsab[seq_ids[b]] = have[b] + (start[b + 1] - start[b]);
}

}  // namespace sllm

using namespace sllm;

// prefix_lens == nullptr: the reference's contract (every prefill entry starts at position 0)
static int store_kvcache_impl(const void* k, const void* v, void* k_cache, void* v_cache, const int32_t* block_table,
                              const int32_t* seq_ids, const int32_t* prefill_seq_start_locs, const int32_t* prefill_seq_lens,
                              const int32_t* prefix_lens, const int32_t* decoding_seq_lens, int num_prefill_seqs,
                              int num_decoding_seqs, int64_t num_prefill_tokens, int max_prefill_len, int cur_layer,
                              int num_layers, int nkv, int block_size, int head_dim, int max_blocks_per_seq,
                              int64_t k_row_stride, int64_t v_row_stride, sllm_dtype_t dtype, sllm_stream_t stream_) {
    SLLM_REQUIRE(head_dim > 0 && head_dim % 8 == 0, "store_kvcache: head_dim (%d) must be a multiple of 8", head_dim);
    SLLM_REQUIRE(k_row_stride >= (int64_t)nkv * head_dim && v_row_stride >= (int64_t)nkv * head_dim && k_row_stride % 8 == 0 &&
                 v_row_stride % 8 == 0, "store_kvcache: bad row strides (%lld, %lld)", (long long)k_row_stride, (long long)v_row_stride);
    SLLM_REQUIRE(block_size > 0 && nkv > 0 && num_layers > 0 && cur_layer >= 0 && cur_layer < num_layers,
                 "store_kvcache: bad cache geometry (layer %d of %d)", cur_layer, num_layers);
    SLLM_REQUIRE(num_prefill_seqs >= 0 && num_decoding_seqs >= 0, "store_kvcache: negative batch");
    if (num_prefill_seqs + num_decoding_seqs == 0) return 0;
    SLLM_REQUIRE(k && v && k_cache && v_cache && block_table && seq_ids, "store_kvcache: null pointer");
    cudaStream_t stream = (cudaStream_t)stream_;
    if (num_prefill_seqs > 0 && max_prefill_len > 0) {
        SLLM_REQUIRE(prefill_seq_start_locs && prefill_seq_lens, "store_kvcache: null prefill metadata");
        if (prefix_lens) {
            dim3 grid(cdiv(max_prefill_len, block_size) + 1, num_prefill_seqs);
            SLLM_DISPATCH_DTYPE(dtype, (store_kv_prefill_kernel<T, true><<<grid, 256, 0, stream>>>(
                                           (const T*)k, (const T*)v, (T*)k_cache, (T*)v_cache, block_table, seq_ids,
                                           prefill_seq_start_locs, prefill_seq_lens, cur_layer, num_layers, nkv, block_size,
                                           head_dim, max_blocks_per_seq, k_row_stride, v_row_stride, prefix_lens)));
        } else {
            dim3 grid(cdiv(max_prefill_len, block_size), num_prefill_seqs);
            SLLM_DISPATCH_DTYPE(dtype, (store_kv_prefill_kernel<T, false><<<grid, 256, 0, stream>>>(
                                           (const T*)k, (const T*)v, (T*)k_cache, (T*)v_cache, block_table, seq_ids,
                                           prefill_seq_start_locs, prefill_seq_lens, cur_layer, num_layers, nkv, block_size,
                                           head_dim, max_blocks_per_seq, k_row_stride, v_row_stride, nullptr)));
        }
        int e = check_launch("store_kvcache(prefill)");
        if (e) return e;
    }
    if (num_decoding_seqs > 0) {
        SLLM_REQUIRE(decoding_seq_lens, "store_kvcache: null decoding_seq_lens");
        const size_t elem = 2;
        const char* kd = (const char*)k + (size_t)num_prefill_tokens * (size_t)k_row_stride * elem;
        const char* vd = (const char*)v + (size_t)num_prefill_tokens * (size_t)v_row_stride * elem;
        SLLM_DISPATCH_DTYPE(dtype, (store_kv_decode_kernel<T><<<num_decoding_seqs, 128, 0, stream>>>(
                                       (const T*)kd, (const T*)vd, (T*)k_cache, (T*)v_cache, block_table,
                                       seq_ids + num_prefill_seqs, decoding_seq_lens, cur_layer, num_layers, nkv,
                                       block_size, head_dim, max_blocks_per_seq, k_row_stride, v_row_stride)));
        return check_launch("store_kvcache(decode)");
    }
    return 0;
}

extern "C" {

int sllm_store_kvcache(const void* k, const void* v, void* k_cache, void* v_cache, const int32_t* block_table,
                       const int32_t* seq_ids, const int32_t* prefill_seq_start_locs, const int32_t* prefill_seq_lens,
                       const int32_t* decoding_seq_lens, int num_prefill_seqs, int num_decoding_seqs,
                       int64_t num_prefill_tokens, int max_prefill_len, int cur_layer, int num_layers, int nkv,
                       int block_size, int head_dim, int max_blocks_per_seq, int64_t k_row_stride, int64_t v_row_stride,
                       sllm_dtype_t dtype, sllm_stream_t stream) {
    return store_kvcache_impl(k, v, k_cache, v_cache, block_table, seq_ids, prefill_seq_start_locs, prefill_seq_lens, nullptr,
                              decoding_seq_lens, num_prefill_seqs, num_decoding_seqs, num_prefill_tokens, max_prefill_len,
                              cur_layer, num_layers, nkv, block_size, head_dim, max_blocks_per_seq, k_row_stride, v_row_stride,
                              dtype, stream);
}

int sllm_store_kvcache_chunked(const void* k, const void* v, void* k_cache, void* v_cache, const int32_t* block_table,
                               const int32_t* seq_ids, const int32_t* prefill_seq_start_locs, const int32_t* prefill_seq_lens,
                               const int32_t* prefill_prefix_lens, const int32_t* decoding_seq_lens, int num_prefill_seqs,
                               int num_decoding_seqs, int64_t num_prefill_tokens, int max_prefill_len, int cur_layer,
                               int num_layers, int nkv, int block_size, int head_dim, int max_blocks_per_seq,
                               int64_t k_row_stride, int64_t v_row_stride, sllm_dtype_t dtype, sllm_stream_t stream) {
    SLLM_REQUIRE(num_prefill_seqs == 0 || prefill_prefix_lens, "store_kvcache_chunked: null prefill_prefix_lens");
    return store_kvcache_impl(k, v, k_cache, v_cache, block_table, seq_ids, prefill_seq_start_locs, prefill_seq_lens,
                              prefill_prefix_lens, decoding_seq_lens, num_prefill_seqs, num_decoding_seqs, num_prefill_tokens,
                              max_prefill_len, cur_layer, num_layers, nkv, block_size, head_dim, max_blocks_per_seq,
                              k_row_stride, v_row_stride, dtype, stream);
}

int sllm_set_block_table_and_num_seq_alloc_blocks(int32_t* nsab, int32_t* block_table, const int64_t* cand,
                                                  const int32_t* seq_ids, const int32_t* need, const int32_t* need_cumsum,
                                                  int batch, int mbps, sllm_stream_t stream) {
    if (batch <= 0) return 0;
    SLLM_REQUIRE(nsab && block_table && seq_ids && need && need_cumsum, "set_block_table: null pointer");
    set_block_table_kernel<<<cdiv(batch, 4), 128, 0, (cudaStream_t)stream>>>(nsab, block_table, cand, seq_ids, need,
                                                                              need_cumsum, batch, mbps);
    return check_launch("set_block_table_and_num_seq_alloc_blocks");
}

int sllm_unset_block_table_and_num_seq_alloc_blocks(int32_t* nsab, const int32_t* block_table, const int32_t* seq_ids,
                                                    uint8_t* is_free, int batch, int mbps, sllm_stream_t stream) {
    if (batch <= 0) return 0;
    SLLM_REQUIRE(nsab && block_table && seq_ids && is_free, "unset_block_table: null pointer");
    unset_block_table_kernel<false><<<cdiv(batch, 4), 128, 0, (cudaStream_t)stream>>>(nsab, block_table, seq_ids, is_free,
                                                                                       nullptr, nullptr, batch, mbps);
    return check_launch("unset_block_table_and_num_seq_alloc_blocks");
}

int sllm_gather_allocated_blocks_and_unset(int32_t* nsab, const int32_t* block_table, const int32_t* seq_ids,
                                           uint8_t* is_free, const int32_t* cumsum, int32_t* gathered, int batch,
                                           int mbps, sllm_stream_t stream) {
    if (batch <= 0) return 0;
    SLLM_REQUIRE(nsab && block_table && seq_ids && is_free && cumsum, "gather_allocated_blocks: null pointer");
    unset_block_table_kernel<true><<<cdiv(batch, 4), 128, 0, (cudaStream_t)stream>>>(nsab, block_table, seq_ids, is_free,
                                                                                      cumsum, gathered, batch, mbps);
    return check_launch("gather_allocated_blocks_and_unset");
}

int sllm_truncate_blocks_for_seqs(int32_t* nsab, const int32_t* block_table, uint8_t* is_free, const int32_t* seq_ids,
                                  const int32_t* target_lens, int batch, int block_size, int mbps, sllm_stream_t stream) {
    SLLM_REQUIRE(batch >= 0 && block_size > 0 && mbps > 0, "truncate_blocks: bad sizes");
    if (batch == 0) return 0;
    SLLM_REQUIRE(nsab && block_table && is_free && seq_ids && target_lens, "truncate_blocks: null pointer");
    truncate_blocks_kernel<<<cdiv(batch, 4), 128, 0, (cudaStream_t)stream>>>(nsab, block_table, is_free, seq_ids, target_lens,
                                                                             batch, block_size, mbps);
    return check_launch("truncate_blocks_for_seqs");
}

int sllm_allocate_blocks_for_seqs(int32_t* nsab, int32_t* block_table, uint8_t* is_free, const int32_t* seq_ids,
                                  const int32_t* target_lens, int batch, int block_size, int64_t num_blocks, int mbps,
                                  int64_t* new_out, int64_t cap, int32_t* status, sllm_stream_t stream) {
    SLLM_REQUIRE(batch >= 0 && block_size > 0 && num_blocks >= 0 && mbps > 0, "allocate_blocks: bad sizes");
    SLLM_REQUIRE(status, "allocate_blocks: status_out is required");
    SLLM_REQUIRE(batch == 0 || (nsab && block_table && is_free && seq_ids && target_lens), "allocate_blocks: null pointer");
    const size_t smem = (size_t)(2 * batch + 1) * sizeof(int32_t);
    SLLM_REQUIRE(smem <= 200 * 1024, "allocate_blocks: batch %d too large", batch);
    if (int e = fit_dynamic_smem<allocate_blocks_kernel>(smem, "allocate_blocks_for_seqs")) return e;
    allocate_blocks_kernel<<<1, 1024, smem, (cudaStream_t)stream>>>(nsab, block_table, is_free, seq_ids, target_lens, batch,
                                                                   block_size, num_blocks, mbps, new_out, cap, status);
    return check_launch("allocate_blocks_for_seqs");
}

int sllm_fork_blocks_for_seqs(int32_t* nsab, int32_t* block_table, int32_t* extra_refs, const int32_t* src_seq_ids,
                              const int32_t* dst_seq_ids, const int32_t* lens, int batch, int block_size, int mbps,
                              sllm_stream_t stream) {
    SLLM_REQUIRE(batch >= 0 && block_size > 0 && mbps > 0, "fork_blocks: bad sizes");
    if (batch == 0) return 0;
    SLLM_REQUIRE(nsab && block_table && extra_refs && src_seq_ids && dst_seq_ids && lens, "fork_blocks: null pointer");
    fork_blocks_kernel<<<cdiv(batch, 4), 128, 0, (cudaStream_t)stream>>>(nsab, block_table, extra_refs, src_seq_ids, dst_seq_ids,
                                                                         lens, batch, block_size, mbps);
    return check_launch("fork_blocks_for_seqs");
}

int sllm_copy_block_tails(void* k_cache, void* v_cache, int32_t* token_cache, const int32_t* block_table,
                          const int32_t* src_seq_ids, const int32_t* dst_seq_ids, const int32_t* lens, int batch,
                          int64_t block_bytes, int block_size, int mbps, sllm_stream_t stream) {
    SLLM_REQUIRE(batch >= 0 && block_size > 0 && mbps > 0 && block_bytes > 0 && block_bytes % 16 == 0,
                 "copy_block_tails: bad sizes (block_bytes %lld must be a positive multiple of 16)", (long long)block_bytes);
    if (batch == 0) return 0;
    SLLM_REQUIRE(k_cache && v_cache && block_table && src_seq_ids && dst_seq_ids && lens, "copy_block_tails: null pointer");
    SLLM_REQUIRE(batch <= 65535, "copy_block_tails: batch %d too large", batch);
    dim3 grid(cdiv(block_bytes, kTailChunk), batch, 2);
    copy_block_tails_kernel<<<grid, kTailThreads, 0, (cudaStream_t)stream>>>(
        (char*)k_cache, (char*)v_cache, token_cache, block_table, src_seq_ids, dst_seq_ids, lens, block_bytes, block_size, mbps);
    return check_launch("copy_block_tails");
}

int sllm_release_blocks_for_seqs(int32_t* nsab, const int32_t* block_table, uint8_t* is_free, int32_t* extra_refs,
                                 const int32_t* seq_ids, const int32_t* cumsum, int32_t* gathered, int batch, int mbps,
                                 sllm_stream_t stream) {
    SLLM_REQUIRE(batch >= 0 && mbps > 0, "release_blocks: bad sizes");
    if (batch == 0) return 0;
    SLLM_REQUIRE(nsab && block_table && is_free && extra_refs && seq_ids, "release_blocks: null pointer");
    SLLM_REQUIRE(!gathered || cumsum, "release_blocks: gathering needs the cumsum");
    if (gathered)
        release_blocks_kernel<true><<<cdiv(batch, 4), 128, 0, (cudaStream_t)stream>>>(nsab, block_table, is_free, extra_refs,
                                                                                       seq_ids, cumsum, gathered, batch, mbps);
    else
        release_blocks_kernel<false><<<cdiv(batch, 4), 128, 0, (cudaStream_t)stream>>>(nsab, block_table, is_free, extra_refs,
                                                                                        seq_ids, nullptr, nullptr, batch, mbps);
    return check_launch("release_blocks_for_seqs");
}

}  // extern "C"
