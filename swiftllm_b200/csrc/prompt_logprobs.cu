// Prompt log-probabilities: for each of many [rows, V] logits rows (every row of a prefill), the log-probability of a given
// target token, its rank and the top-N entries of log_softmax(l).  The values are those of sllm_token_logprobs
// (csrc/logprobs.cu) bit for bit: m (the largest key), Z = sum over v of round(expf(l_v - m) * 2^40) as 64-bit integers,
// lse = m + logf(Z * 2^-40) and l - lse, with the same intrinsics.  Z is an exact integer, so how the row is partitioned among
// threads does not change it.  rank = 1 + the number of ids whose key (vocab_select.cuh: order-preserving, -0 == +0) is strictly
// greater than the target's; a target outside [0, V) gives NaN and rank -1.  Top-N, NaN / +inf rows: as csrc/logprobs.cu.
//
// Layout: one CTA of 512 threads per row, no clusters; two or more CTAs per SM, so one row's arithmetic overlaps another's loads.
//   pass 1  streams the row from HBM: the largest key, the NaN / +inf flag, the count of keys above the target's key and the
//           maxima of 64 disjoint 8-lane groups.  The first kStageKeys keys of the row are kept in shared memory.
//   pass 2  reads the rest of the row again (just read, so mostly from L2) and then the staged keys: Z, and every key >= the
//           N-th largest group maximum (a lower bound of the N-th largest key, since N groups hold a key >= it each) into a
//           candidate buffer of (key, id) pairs.
//   select  each candidate's place among the others by (key desc, id asc); places below N are the top-N.  A row with more than
//           kMaxCand candidates (many ties near its top) takes N block-wide max rounds over its (key, id) pairs instead: exact,
//           slower, and only reached by degenerate rows.
// Algorithmic bytes: rows * V * 2 (logits) + rows * (12 + 8 * top_n).
//
// No fast-math here: expf / logf must be the accurate ones csrc/logprobs.cu uses.
#include "vocab_select.cuh"

namespace sllm {
namespace {

constexpr int kRowThreads = 512;
constexpr int kRowWarps = kRowThreads / 32;
constexpr int kGroups = kRowWarps * 4;                  // 8-lane groups: 64 disjoint maxima >= kPromptMaxTopN
constexpr int kPromptMaxTopN = 20;
constexpr int kMaxCand = 1024;
constexpr int kStageKeys = 48 * 1024;                    // 96 KB of staged keys per CTA: two CTAs of the largest vocabularies per SM
constexpr int kMaxPromptRows = 1 << 24;
constexpr int kMaxPromptVocab = 1 << 24;                 // Z <= V * 2^40 stays below 2^64

// 16 logits bytes that bypass L1; `last_use`: read for the last time, so L2 evicts them first (the part of the row pass 2 reads
// again keeps the normal priority)
__device__ __forceinline__ uint4 ld_row_vec(const uint4* p, bool last_use) {
    uint4 u;
    if (last_use)
        asm volatile("{\n\t.reg .b64 pol;\n\tcreatepolicy.fractional.L2::evict_first.b64 pol, 1.0;\n\t"
                     "ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], pol;\n\t}"
                     : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(p));
    else
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(p));
    return u;
}

__device__ __forceinline__ void keys8(const uint4& u, uint32_t (&k)[8]) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; j++) { k[2 * j] = key_of((uint16_t)(w[j] & 0xffffu)); k[2 * j + 1] = key_of((uint16_t)(w[j] >> 16)); }
}

// (key desc, id asc) as one unsigned order: larger is better, and no two ids share a value
__device__ __forceinline__ unsigned long long pair_of(uint32_t key, int id) {
    return ((unsigned long long)key << 32) | (0xffffffffu - (uint32_t)id);
}

template <typename T>
__global__ void __launch_bounds__(kRowThreads, 2) prompt_logprobs_kernel(
    const T* __restrict__ logits, int64_t row_stride, int V, int stage_vecs, const int32_t* __restrict__ target_ids, int top_n,
    float* __restrict__ out_logprob, int32_t* __restrict__ out_rank, int32_t* __restrict__ out_top_ids,
    float* __restrict__ out_top_logprobs) {
    extern __shared__ uint4 staged[];                    // keys of the row's first vectors, 8 per uint4
    __shared__ uint32_t group_max[kGroups], warp_best[kRowWarps], warp_above[kRowWarps], floor_key;
    __shared__ int warp_bad[kRowWarps], cand_n;
    __shared__ unsigned long long cand[kMaxCand], scratch[32];

    const int64_t row = blockIdx.x;
    const uint16_t* s16 = reinterpret_cast<const uint16_t*>(logits + row * row_stride);
    const int N = min(top_n, V);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int32_t tok = target_ids[row];
    const bool tok_ok = tok >= 0 && tok < V;
    const uint32_t tok_key = tok_ok ? key_of(s16[tok]) : 0xffffffffu;

    // the row as [head scalars][nvec 16-byte vectors][tail scalars]: rows of any alignment stream through vector loads
    const int head = min(V, (int)(((16u - (uint32_t)(reinterpret_cast<uintptr_t>(s16) & 15u)) & 15u) >> 1));
    const int nvec = (V - head) >> 3;
    const int nscalar = V - 8 * nvec;
    const int nstage = min(nvec, stage_vecs);
    const uint4* vsrc = reinterpret_cast<const uint4*>(s16 + head);
    auto scalar_id = [&](int t) { return t < head ? t : 8 * nvec + t; };

    // ---- pass 1: largest key, NaN / +inf flag, keys above the target's, group maxima; stage the first nstage vectors
    if (tid == 0) cand_n = 0;
    uint32_t best = 0, above = 0;
    bool bad = false;
    auto see = [&](uint32_t k) {
        best = max(best, k);
        above += k > tok_key;
        bad |= k >= InfKeys<T>::pos || k < InfKeys<T>::neg;
    };
    for (int j = tid; j < nvec; j += kRowThreads) {
        uint32_t k[8];
        keys8(ld_row_vec(vsrc + j, j < nstage), k);
#pragma unroll
        for (int e = 0; e < 8; e++) see(k[e]);
        if (j < nstage) staged[j] = make_uint4(k[0] | (k[1] << 16), k[2] | (k[3] << 16), k[4] | (k[5] << 16), k[6] | (k[7] << 16));
    }
    for (int t = tid; t < nscalar; t += kRowThreads) see(key_of(s16[scalar_id(t)]));
    uint32_t g = best;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) g = max(g, __shfl_xor_sync(0xffffffffu, g, o));
    if ((lane & 7) == 0) group_max[warp * 4 + (lane >> 3)] = g;
    best = __reduce_max_sync(0xffffffffu, best);
    above = __reduce_add_sync(0xffffffffu, above);
    bad = __any_sync(0xffffffffu, bad);
    if (lane == 0) { warp_best[warp] = best; warp_above[warp] = above; warp_bad[warp] = bad; }
    __syncthreads();
    uint32_t max_key = 0, total_above = 0;
    for (int w = 0; w < kRowWarps; w++) {
        max_key = max(max_key, warp_best[w]);
        total_above += warp_above[w];
        bad |= warp_bad[w] != 0;
    }
    const float m = value_of<T>(max_key);
    bad |= m == -INFINITY;                               // every logit -inf: no distribution (NaN, as log_softmax)

    // ---- the top-N floor: the N-th largest group maximum (a group without keys reports 0, which can only lower it)
    if (N > 0) {
        if (tid < kGroups) {
            const uint32_t v = group_max[tid];
            int gt = 0, ge = 0;
            for (int j = 0; j < kGroups; j++) { gt += group_max[j] > v; ge += group_max[j] >= v; }
            if (gt < N && N <= ge) floor_key = v;        // threads that write hold the same value
        }
        __syncthreads();
    }
    const uint32_t lowest = N > 0 ? floor_key : 0u;

    // ---- pass 2: Z (exact fixed point) and the candidates >= floor; the re-read part first, while it is in L2
    unsigned long long z = 0;
    auto take = [&](uint32_t k, int id) {
        if (!bad) z += __float2ull_rn(__fmul_rn(expf(__fsub_rn(value_of<T>(k), m)), kMassScale));
        if (N > 0 && k >= lowest) {
            const int s = atomicAdd(&cand_n, 1);
            if (s < kMaxCand) cand[s] = pair_of(k, id);
        }
    };
    for (int j = nstage + tid; j < nvec; j += kRowThreads) {
        uint32_t k[8];
        keys8(ld_row_vec(vsrc + j, true), k);
#pragma unroll
        for (int e = 0; e < 8; e++) take(k[e], head + 8 * j + e);
    }
    for (int t = tid; t < nscalar; t += kRowThreads) take(key_of(s16[scalar_id(t)]), scalar_id(t));
    for (int j = tid; j < nstage; j += kRowThreads) {
        const uint4 u = staged[j];
        const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int e = 0; e < 8; e++) take((w[e >> 1] >> (16 * (e & 1))) & 0xffffu, head + 8 * j + e);
    }
    const unsigned long long Z = block_sum_u64(z, scratch);     // ends with every thread past a __syncthreads: cand_n is final
    const float lse = bad ? NAN : __fadd_rn(m, logf(__fmul_rn(__ull2float_rn(Z), 1.0f / kMassScale)));

    // ---- select the top-N: (key desc, id asc)
    const int64_t o = row * top_n;
    auto emit = [&](int place, unsigned long long p) {
        const uint32_t k = (uint32_t)(p >> 32);
        out_top_ids[o + place] = (int32_t)(0xffffffffu - (uint32_t)p);
        out_top_logprobs[o + place] = __fsub_rn(value_of<T>(k), lse);
    };
    const int nc = cand_n;
    if (N > 0 && nc <= kMaxCand) {
        for (int j = tid; j < nc; j += kRowThreads) {
            const unsigned long long p = cand[j];
            int place = 0;
            for (int i = 0; i < nc; i++) place += cand[i] > p;
            if (place < N) emit(place, p);
        }
    } else if (N > 0) {
        // more candidates than the buffer holds: N rounds, each the largest pair below the previous one
        unsigned long long prev = ~0ull;
        for (int r = 0; r < N; r++) {
            unsigned long long b = 0;
            for (int i = tid; i < V; i += kRowThreads) {
                const unsigned long long p = pair_of(key_of(s16[i]), i);
                b = p < prev && p > b ? p : b;
            }
            b = block_max_u64(b, scratch);
            if (tid == 0) emit(r, b);
            prev = b;
        }
    }
    for (int j = N + tid; j < top_n; j += kRowThreads) {
        out_top_ids[o + j] = -1;
        out_top_logprobs[o + j] = NAN;
    }
    if (tid == 0) {
        out_logprob[row] = tok_ok ? __fsub_rn(value_of<T>(tok_key), lse) : NAN;
        out_rank[row] = tok_ok ? (int32_t)(1 + total_above) : -1;
    }
}

template <typename T>
int launch(const void* logits, int64_t rows, int V, int64_t row_stride, const int32_t* target_ids, int top_n, float* out_logprob,
           int32_t* out_rank, int32_t* out_top_ids, float* out_top_logprobs, cudaStream_t stream) {
    static unsigned long long configured = 0;
    if (first_use_on_this_device(configured))
        cudaFuncSetAttribute(prompt_logprobs_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, kStageKeys * 2);
    const int stage_vecs = min(kStageKeys, V) / 8;
    prompt_logprobs_kernel<T><<<(unsigned)rows, kRowThreads, (size_t)stage_vecs * 16, stream>>>(
        (const T*)logits, row_stride, V, stage_vecs, target_ids, top_n, out_logprob, out_rank, out_top_ids, out_top_logprobs);
    return check_launch("prompt_logprobs");
}

}  // namespace
}  // namespace sllm

extern "C" int sllm_prompt_logprobs(const void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride,
                                    const int32_t* target_ids, int top_n, float* out_logprob, int32_t* out_rank,
                                    int32_t* out_top_ids, float* out_top_logprobs, sllm_dtype_t dtype, sllm_stream_t stream) {
    using namespace sllm;
    SLLM_REQUIRE(dtype == SLLM_F16 || dtype == SLLM_BF16, "prompt_logprobs: unsupported dtype tag %d", (int)dtype);
    SLLM_REQUIRE(num_rows >= 0 && num_rows <= kMaxPromptRows, "prompt_logprobs: num_rows %lld outside [0, %d]",
                 (long long)num_rows, kMaxPromptRows);
    SLLM_REQUIRE(vocab_size > 0 && vocab_size <= kMaxPromptVocab, "prompt_logprobs: vocab_size %d outside [1, %d]", vocab_size,
                 kMaxPromptVocab);
    SLLM_REQUIRE(top_n >= 0 && top_n <= kPromptMaxTopN, "prompt_logprobs: top_n %d outside [0, %d]", top_n, kPromptMaxTopN);
    SLLM_REQUIRE(logits_row_stride >= vocab_size, "prompt_logprobs: logits_row_stride %lld < vocab_size %d",
                 (long long)logits_row_stride, vocab_size);
    if (num_rows == 0) return 0;
    SLLM_REQUIRE(logits && target_ids && out_logprob && out_rank && (top_n == 0 || (out_top_ids && out_top_logprobs)),
                 "prompt_logprobs: null pointer");
    SLLM_DISPATCH_DTYPE(dtype, return launch<T>(logits, num_rows, vocab_size, logits_row_stride, target_ids, top_n, out_logprob,
                                                out_rank, out_top_ids, out_top_logprobs, (cudaStream_t)stream));
}
