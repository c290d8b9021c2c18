// Constrained decoding: per-row allowed-token bitmasks and per-request logit bias, applied in place to [rows, V] 16-bit logits
// (a vocabulary shard with vocab_offset works; bits and bias ids are GLOBAL vocabulary indices).
// Semantics (restated in numpy by tests/constraints_oracle.py), per row r with m = mask_index[r], e = bias_index[r]:
//   mask     m >= 0: every id v of the shard whose bit (masks[m][v / 32] >> (v % 32)) & 1 is 0 becomes -inf; allowed ids keep
//            their bits (NaN and -0 included).  m < 0: no mask;
//   bias     e >= 0: every allowed id v = bias_ids[j] of the shard, j in [bias_starts[e], bias_starts[e + 1]), becomes
//            round_to_storage(float(l) + bias_values[j]): one IEEE fp32 add, one rounding to nearest even; -inf stays -inf, NaN
//            stays NaN (the canonical 0x7fff).  A bias on a masked id leaves it -inf.  e < 0: no bias;
//   other    rows with m < 0 and e < 0 are not touched (nothing read or written).
// The penalties (csrc/penalties.cu) and the token choice run afterwards, unchanged: vLLM's order (allowed ids / bad words and
// logit bias before penalties and temperature).  Bias ids are distinct within an entry, mask / bias indices outside their arrays
// and bias ids outside the shard are skipped, never dereferenced.
//
// Layout: a 2-D grid, x = row, y = slices of the row; thread i of the launch handles ids i, i + stride, ...: a disallowed id is
// stored as -inf without reading the logit, allowed ids are not touched.  The y = 0 CTA of a row also applies its bias entries.
// The two sets are disjoint (the bias skips masked ids), so every logit is written by at most one thread: no atomics, and the
// result is a pure function of the inputs whatever the grid.  HBM-bound; no clusters, no shared memory.
// Algorithmic bytes per constrained row: 4 * W (mask words, W = ceil(V / 32) of the row's shard) + 2 * disallowed ids (written)
// + 12 * bias entries (id and value read, logit read and written).
#include "common.cuh"

namespace sllm {
namespace {

constexpr int kThreads = 256;
constexpr int kIdsPerThread = 8;                    // ids per thread and row when the grid covers the row once
constexpr int kMaxSlices = 1024;

__device__ __forceinline__ bool allowed(const uint32_t* __restrict__ mask, int64_t v) {
    return (__ldg(mask + (v >> 5)) >> (v & 31)) & 1u;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) constrain_kernel(
    T* __restrict__ logits, int64_t row_stride, int V, int64_t vocab_offset, const int32_t* __restrict__ mask_index,
    const uint32_t* __restrict__ masks, int64_t num_masks, int mask_words, const int32_t* __restrict__ bias_index,
    const int32_t* __restrict__ bias_starts, int64_t num_entries, const int32_t* __restrict__ bias_ids,
    const float* __restrict__ bias_values, int64_t num_bias) {
    const int64_t row = blockIdx.x;
    const int32_t m = mask_index[row], e = bias_index[row];
    const uint32_t* mask = (m >= 0 && m < num_masks) ? masks + (int64_t)m * mask_words : nullptr;
    const bool biased = e >= 0 && e < num_entries;
    if (mask == nullptr && !biased) return;
    T* out = logits + row * row_stride;

    if (mask != nullptr) {
        const T neg_inf = Traits<T>::from_f(-INFINITY);
        const int stride = (int)(gridDim.y * blockDim.x);
        for (int i = (int)(blockIdx.y * blockDim.x + threadIdx.x); i < V; i += stride)
            if (!allowed(mask, vocab_offset + i)) out[i] = neg_inf;
    }
    if (biased && blockIdx.y == 0) {
        const int64_t b0 = max((int64_t)0, (int64_t)bias_starts[e]), b1 = min(num_bias, (int64_t)bias_starts[e + 1]);
        for (int64_t j = b0 + threadIdx.x; j < b1; j += blockDim.x) {
            const int64_t v = bias_ids[j], local = v - vocab_offset;
            if (local < 0 || local >= V || (mask != nullptr && !allowed(mask, v))) continue;
            out[local] = Traits<T>::from_f(__fadd_rn(Traits<T>::to_f(out[local]), bias_values[j]));
        }
    }
}

}  // namespace
}  // namespace sllm

extern "C" int sllm_constrain_logits(void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride,
                                     int64_t vocab_offset, const int32_t* mask_index, const uint32_t* masks, int64_t num_masks,
                                     int mask_words, const int32_t* bias_index, const int32_t* bias_starts,
                                     int64_t num_entries, const int32_t* bias_ids, const float* bias_values, int64_t num_bias,
                                     sllm_dtype_t dtype, sllm_stream_t stream) {
    using namespace sllm;
    SLLM_REQUIRE(dtype == SLLM_F16 || dtype == SLLM_BF16, "constrain_logits: unsupported dtype tag %d", (int)dtype);
    SLLM_REQUIRE(num_rows >= 0 && num_rows <= INT32_MAX, "constrain_logits: num_rows %lld out of range", (long long)num_rows);
    SLLM_REQUIRE(vocab_size > 0, "constrain_logits: vocab_size must be positive, got %d", vocab_size);
    SLLM_REQUIRE(vocab_offset >= 0 && vocab_offset + vocab_size < (int64_t)INT32_MAX + 1,
                 "constrain_logits: global vocabulary indices must stay below 2^31 (vocab_offset %lld)", (long long)vocab_offset);
    SLLM_REQUIRE(logits_row_stride >= vocab_size, "constrain_logits: logits_row_stride %lld < vocab_size %d",
                 (long long)logits_row_stride, vocab_size);
    SLLM_REQUIRE(num_masks >= 0 && num_masks <= INT32_MAX, "constrain_logits: num_masks %lld out of range", (long long)num_masks);
    SLLM_REQUIRE(num_masks == 0 || (mask_words > 0 && 32 * (int64_t)mask_words >= vocab_offset + vocab_size),
                 "constrain_logits: mask_words %d do not cover the global ids below %lld", mask_words,
                 (long long)(vocab_offset + vocab_size));
    SLLM_REQUIRE(num_entries >= 0 && num_entries < INT32_MAX, "constrain_logits: num_entries %lld out of range",
                 (long long)num_entries);
    SLLM_REQUIRE(num_bias >= 0 && num_bias <= INT32_MAX, "constrain_logits: num_bias %lld out of range", (long long)num_bias);
    if (num_rows == 0) return 0;
    SLLM_REQUIRE(logits && mask_index && bias_index && (num_masks == 0 || masks) && (num_entries == 0 || bias_starts) &&
                 (num_bias == 0 || (bias_ids && bias_values)),
                 "constrain_logits: null pointer");
    const int64_t per_slice = (int64_t)kThreads * kIdsPerThread;
    const dim3 grid((unsigned)num_rows, (unsigned)std::min<int64_t>(kMaxSlices, (vocab_size + per_slice - 1) / per_slice));
    SLLM_DISPATCH_DTYPE(dtype, {
        constrain_kernel<T><<<grid, kThreads, 0, (cudaStream_t)stream>>>(
            (T*)logits, logits_row_stride, vocab_size, vocab_offset, mask_index, masks, num_masks, mask_words, bias_index,
            bias_starts, num_entries, bias_ids, bias_values, num_bias);
        return check_launch("constrain_logits");
    });
}
