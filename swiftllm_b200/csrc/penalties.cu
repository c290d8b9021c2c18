// Repetition / frequency / presence penalties applied in place to [rows, V] 16-bit logits, with the token history read from
// the device-resident token pages (token_cache int32 [num_blocks, block_size], addressed through the block table like a KV page;
// each entry is id | is_output << 31).
// Semantics (restated in numpy by tests/penalties_oracle.py), per row with r, f, p its penalties and the history = positions
// [0, pos) of its sequence (pages for [0, pos - n_new), this step's n_new input tokens for the rest):
//   c_out(v)  number of output tokens equal to v; seen(v): v occurs among the prompt or output tokens;
//   seen v    l = float(logit); l = l > 0 ? l / r : l * r; t = f * float(c_out); t = t + p if c_out > 0; l = l - t; stored
//             rounded once to the storage dtype (round to nearest even).  fp32, IEEE, no contraction;
//   other v   the entry keeps its bits.
// Ids outside [vocab_offset, vocab_offset + vocab_size) are not this launch's (absent); an invalid id or block id in the history
// is skipped, never dereferenced.  Rows with r == 1, f == 0, p == 0 are skipped entirely (nothing read, recorded or modified).
// After counting, the row's new tokens are written to positions [pos - n_new, pos) of its pages - disjoint from what is read.
//
// Layout: one thread-block cluster of C CTAs per penalised row.  The cluster keeps a u32 slot per vocabulary id of the launch's
// shard in distributed shared memory, CTA k owning ids [k * slice, (k + 1) * slice): bit 31 = seen in the prompt, the low bits
// count output tokens (exact up to 2^31 - 1).  Every CTA counts a strided share of the history into whichever CTA owns each id;
// lanes of a warp holding the same (id, kind) are merged first (__match_any_sync), so one id repeated thousands of times costs one
// DSMEM atomic per warp, not one per occurrence.  After a cluster barrier each CTA rewrites the entries of its slice whose slot
// is non-zero.  Counts are integers: the result does not depend on the order of the atomics, the cluster size or the batch.
// Algorithmic bytes per penalised row: 4 * pos (history) + 4 * n_new (pages written) + 4 * distinct ids (logits read / written).
#include "vocab_select.cuh"

namespace sllm {
namespace {

constexpr uint32_t kOutputBit = 0x80000000u;       // token page word: id | kOutputBit for an output token
constexpr uint32_t kSeenInPrompt = 0x80000000u;    // cluster slot: set when the id occurs among the prompt tokens
constexpr uint32_t kAbsentId = 0x7fffffffu;        // recorded for a negative input id: >= vocab_offset + vocab_size always

// Cluster size for 4-byte slots: the smallest that fits a slice in shared memory, raised towards rows * C >= the SM count.
int penalty_cluster_size(int64_t rows, int V) {
    int c = 1;
    while (c < kMaxCluster && (((int64_t)V + c - 1) / c + 3) / 4 * 4 * 4 > kMaxSliceBytes) c *= 2;
    while (c < kMaxCluster && rows * c * 2 <= 132) c *= 2;
    return c;
}

template <typename T> __device__ __forceinline__ float to_f32(T x);
template <> __device__ __forceinline__ float to_f32<__half>(__half x) { return __half2float(x); }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 x) { return __bfloat162float(x); }
template <typename T> __device__ __forceinline__ T from_f32(float x);
template <> __device__ __forceinline__ __half from_f32<__half>(float x) { return __float2half_rn(x); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }

template <typename T>
__global__ void __launch_bounds__(kThreads) penalty_kernel(
    T* __restrict__ logits, int64_t row_stride, int V, int64_t vocab_offset, int slice, const float* __restrict__ rep,
    const float* __restrict__ freq, const float* __restrict__ pres, const int32_t* __restrict__ seq_ids,
    const int32_t* __restrict__ pos, const int32_t* __restrict__ input_ids, const int32_t* __restrict__ last_token_indices,
    const int32_t* __restrict__ prefill_seq_lens, int num_prefill_rows, const int32_t* __restrict__ block_table,
    int block_table_stride, int block_size, int32_t* token_cache, int64_t num_blocks) {
    extern __shared__ uint32_t slots[];

    cg::cluster_group cluster = cg::this_cluster();
    const unsigned C = cluster.num_blocks(), rank = cluster.block_rank();
    const int64_t row = blockIdx.x / C;
    const float r = rep[row], f = freq[row], p = pres[row];
    if (r == 1.f && f == 0.f && p == 0.f) return;                     // the whole cluster leaves, before any DSMEM access

    const int begin = (int)rank * slice;
    const int n = max(0, min(V, begin + slice) - begin);
    for (int i = 4 * threadIdx.x; i < slice; i += 4 * blockDim.x) *reinterpret_cast<uint4*>(slots + i) = make_uint4(0, 0, 0, 0);

    // ---- the row's history: positions [0, hist) from the pages, then its n_new input tokens
    const int P = pos[row];
    const bool prefill = row < num_prefill_rows;
    const int n_new = max(0, prefill ? prefill_seq_lens[row] : 1);
    const int64_t first_in = (int64_t)last_token_indices[row] - n_new + 1;
    const uint32_t new_flag = prefill ? 0u : kOutputBit;
    auto new_word = [&](int j) -> uint32_t {                         // page word of the row's j-th new token
        const int32_t id = input_ids[first_in + j];
        return (id >= 0 ? (uint32_t)id : kAbsentId) | new_flag;
    };
    const int hist = max(0, P - n_new);
    const int max_pos = block_table_stride * block_size;             // positions the block-table row can address
    const int32_t* bt = block_table + (int64_t)seq_ids[row] * block_table_stride;
    auto page_slot = [&](int q) -> int64_t {                          // index into token_cache of position q, -1 if unmapped
        if (q < 0 || q >= max_pos) return -1;
        const int64_t b = bt[q / block_size];
        return (b >= 0 && b < num_blocks) ? b * block_size + q % block_size : -1;
    };
    cluster.sync();                                                   // every slot zeroed before any CTA adds to it

    const int total = hist + n_new;
    const int lane = threadIdx.x & 31;
    for (int i0 = (int)(rank * blockDim.x + (threadIdx.x & ~31)); i0 < total; i0 += (int)(C * blockDim.x)) {
        const int i = i0 + lane;
        uint32_t word = 0;
        bool valid = false;
        if (i < hist) {
            const int64_t s = page_slot(i);
            if (s >= 0) { word = (uint32_t)token_cache[s]; valid = true; }
        } else if (i < total) {
            word = new_word(i - hist);
            valid = true;
        }
        const bool is_out = (word & kOutputBit) != 0;
        const int64_t local = (int64_t)(word & ~kOutputBit) - vocab_offset;
        valid = valid && local >= 0 && local < V;
        const unsigned long long key = valid ? ((unsigned long long)local << 1) | (is_out ? 1ull : 0ull) : ~0ull;
        const unsigned peers = __match_any_sync(0xffffffffu, key);
        if (valid && lane == __ffs(peers) - 1) {
            uint32_t* dst = cluster.map_shared_rank(slots, (unsigned)(local / slice)) + (local % slice);
            if (is_out) atomicAdd(dst, (uint32_t)__popc(peers));
            else atomicOr(dst, kSeenInPrompt);
        }
    }
    cluster.sync();                                                   // all counts in place

    // ---- rewrite the seen entries of this CTA's slice
    T* dst = logits + row * row_stride + begin;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        const uint32_t c = slots[j];
        if (c == 0) continue;
        const uint32_t c_out = c & ~kSeenInPrompt;
        float l = to_f32<T>(dst[j]);
        l = l > 0.f ? __fdiv_rn(l, r) : __fmul_rn(l, r);
        float t = __fmul_rn(f, __uint2float_rn(c_out));
        if (c_out > 0) t = __fadd_rn(t, p);
        dst[j] = from_f32<T>(__fsub_rn(l, t));
    }

    // ---- record this step's tokens at positions [P - n_new, P)
    for (int j = (int)(rank * blockDim.x + threadIdx.x); j < n_new; j += (int)(C * blockDim.x)) {
        const int64_t s = page_slot(P - n_new + j);
        if (s >= 0) token_cache[s] = (int32_t)new_word(j);
    }
    // no DSMEM access after the last barrier: peers may leave
}

template <typename T>
int launch(void* logits, int64_t rows, int V, int64_t row_stride, int64_t vocab_offset, const float* rep, const float* freq,
           const float* pres, const int32_t* seq_ids, const int32_t* pos, const int32_t* input_ids,
           const int32_t* last_token_indices, const int32_t* prefill_seq_lens, int num_prefill_rows,
           const int32_t* block_table, int block_table_stride, int block_size, int32_t* token_cache, int64_t num_blocks,
           cudaStream_t stream) {
    const int C = penalty_cluster_size(rows, V);
    const int slice = ((V + C - 1) / C + 3) & ~3;
    static unsigned long long configured = 0;
    if (first_use_on_this_device(configured))
        cudaFuncSetAttribute(penalty_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSliceBytes);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(rows * C));
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = (size_t)slice * sizeof(uint32_t);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, penalty_kernel<T>, (T*)logits, row_stride, V, vocab_offset, slice, rep, freq, pres,
                                       seq_ids, pos, input_ids, last_token_indices, prefill_seq_lens, num_prefill_rows,
                                       block_table, block_table_stride, block_size, token_cache, num_blocks);
    if (e != cudaSuccess) {
        set_error("apply_penalties: %s", cudaGetErrorString(e));
        return (int)e;
    }
    return check_launch("apply_penalties");
}

}  // namespace
}  // namespace sllm

extern "C" int sllm_apply_penalties(void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride,
                                    int64_t vocab_offset, const float* repetition_penalty, const float* frequency_penalty,
                                    const float* presence_penalty, const int32_t* seq_ids, const int32_t* pos,
                                    const int32_t* input_ids, const int32_t* last_token_indices,
                                    const int32_t* prefill_seq_lens, int num_prefill_rows, const int32_t* block_table,
                                    int block_table_stride, int block_size, int32_t* token_cache, int64_t num_blocks,
                                    sllm_dtype_t dtype, sllm_stream_t stream) {
    using namespace sllm;
    SLLM_REQUIRE(dtype == SLLM_F16 || dtype == SLLM_BF16, "apply_penalties: unsupported dtype tag %d", (int)dtype);
    SLLM_REQUIRE(num_rows >= 0 && num_rows <= (1 << 20), "apply_penalties: num_rows %lld out of range", (long long)num_rows);
    SLLM_REQUIRE(vocab_size > 0, "apply_penalties: vocab_size must be positive, got %d", vocab_size);
    SLLM_REQUIRE(((((int64_t)vocab_size + kMaxCluster - 1) / kMaxCluster + 3) & ~3ll) * 4 <= kMaxSliceBytes,
                 "apply_penalties: vocab_size %d does not fit the shared memory of a %d-CTA cluster", vocab_size, kMaxCluster);
    SLLM_REQUIRE(vocab_offset >= 0 && vocab_offset + vocab_size <= (int64_t)INT32_MAX,
                 "apply_penalties: global vocabulary indices must stay below 2^31 (vocab_offset %lld)", (long long)vocab_offset);
    SLLM_REQUIRE(logits_row_stride >= vocab_size, "apply_penalties: logits_row_stride %lld < vocab_size %d",
                 (long long)logits_row_stride, vocab_size);
    SLLM_REQUIRE(block_size > 0 && block_size <= (1 << 16), "apply_penalties: block_size %d out of range", block_size);
    SLLM_REQUIRE(block_table_stride > 0 && (int64_t)block_table_stride * block_size <= INT32_MAX,
                 "apply_penalties: block_table_stride %d out of range", block_table_stride);
    SLLM_REQUIRE(num_blocks >= 0, "apply_penalties: num_blocks %lld < 0", (long long)num_blocks);
    SLLM_REQUIRE(num_prefill_rows >= 0 && num_prefill_rows <= num_rows, "apply_penalties: num_prefill_rows %d out of range",
                 num_prefill_rows);
    if (num_rows == 0) return 0;
    SLLM_REQUIRE(logits && repetition_penalty && frequency_penalty && presence_penalty && seq_ids && pos && input_ids &&
                 last_token_indices && block_table && token_cache && (num_prefill_rows == 0 || prefill_seq_lens),
                 "apply_penalties: null pointer");
    SLLM_DISPATCH_DTYPE(dtype, return launch<T>(logits, num_rows, vocab_size, logits_row_stride, vocab_offset,
                                                repetition_penalty, frequency_penalty, presence_penalty, seq_ids, pos,
                                                input_ids, last_token_indices, prefill_seq_lens, num_prefill_rows, block_table,
                                                block_table_stride, block_size, token_cache, num_blocks,
                                                (cudaStream_t)stream));
}
