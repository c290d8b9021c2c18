// Token sampling from [rows, V] logits: greedy, temperature, top-k, top-p, drawn by Gumbel-max with counter-based noise.
// Semantics (restated in numpy by tests/sampling_oracle.py):
//   key(l)   order-preserving uint16 of the 16-bit logit (-0 is mapped to +0, so equal keys <=> equal values);
//   T <= 0   greedy: the largest key, smallest index among equal ones (== torch.argmax for non-NaN rows);
//   top-k    0 < k < V: keep key >= tau_k, the k-th largest key (ties at the boundary are all kept);
//   top-p    p < 1: over the top-k survivors, q_v = exp((l_v - m) / T) with m their max; keep key >= the largest threshold
//            whose mass (counted from the top) is >= p * sum(q) (at least the max is always kept);
//   draw     u = ((x >> 9) + 0.5) * 2^-23 with x = Philox4x32-10(key (seed_lo, seed_hi), counter (v >> 2, pos, 0, 0)) word v & 3,
//            v the GLOBAL vocabulary index; score = l / T - log(-log u) (fp32, IEEE division, logf); the token is the kept
//            index with the largest score, smallest index on ties.
// Both thresholds are exact: keys are 16 bits, so a radix select over the high and then the low byte finds them.  Masses are
// summed as 64-bit fixed-point integers (q * 2^40, rounded), so every sum is exact and independent of the order of additions:
// the result is a pure function of (logits, T, k, p, seed, pos), whatever the cluster size, batch or launch mode.
//
// Layout: one thread-block cluster of C CTAs per row (C chosen on the host so that rows * C covers the GPU at small batch).  Each
// CTA stages its contiguous slice of the row in shared memory as keys (HBM read once), every pass runs from there, and the
// per-CTA histograms / maxima / best (score, index) pairs are merged through distributed shared memory.
// Algorithmic bytes: rows * V * 2 (logits) + rows * 32 (parameters and result).
//
// No fast-math here: logf / expf / division must be the accurate ones the restatement reproduces.
#include "vocab_select.cuh"

namespace sllm {
namespace {

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int i = 0; i < 10; i++) {
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return c;
}

__device__ __forceinline__ float gumbel_of(uint32_t x) {
    const float u = __fmul_rn((float)(x >> 9) + 0.5f, 1.0f / 8388608.0f);     // exact: (n + 0.5) has <= 24 significant bits
    return -logf(-logf(u));
}

// (score, index): larger score wins, then the smaller index
__device__ __forceinline__ bool better(float s, int64_t i, float bs, int64_t bi) {
    return s > bs || (s == bs && i < bi);
}

template <typename T>
__global__ void __launch_bounds__(kThreads) sample_kernel(const T* __restrict__ logits, int64_t row_stride, int V,
                                                          int64_t vocab_offset, int slice, const float* __restrict__ temperature,
                                                          const int32_t* __restrict__ top_k, const float* __restrict__ top_p,
                                                          const int64_t* __restrict__ seed, const int32_t* __restrict__ pos,
                                                          int64_t* __restrict__ out_tokens, float* __restrict__ out_pairs) {
    extern __shared__ uint16_t keys[];
    __shared__ unsigned long long h_cnt_hi[256], h_cnt_lo[256], h_mass_hi[256], h_mass_lo[256], merged[256];
    __shared__ unsigned long long scratch[32];
    __shared__ unsigned long long cta_max;
    __shared__ float cta_score, warp_score[32];
    __shared__ int64_t cta_index, warp_index[32];
    __shared__ int sel_bin;
    __shared__ unsigned long long sel_above;

    cg::cluster_group cluster = cg::this_cluster();
    const unsigned C = cluster.num_blocks(), rank = cluster.block_rank();
    const int64_t row = blockIdx.x / C;
    const int begin = (int)rank * slice;
    const int n = max(0, min(V, begin + slice) - begin);
    const T* src = logits + row * row_stride + begin;

    // ---- stage the slice as keys; local (max key, smallest index)
    for (int i = threadIdx.x; i < 256; i += blockDim.x) h_cnt_hi[i] = h_cnt_lo[i] = h_mass_hi[i] = h_mass_lo[i] = 0;
    unsigned long long best = 0;
    const uint16_t* s16 = reinterpret_cast<const uint16_t*>(src);
    int vec_end = 0;
    if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        vec_end = n & ~7;
        for (int i = 8 * threadIdx.x; i < vec_end; i += 8 * blockDim.x) {
            uint4 u;
            asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(s16 + i));
            const uint32_t w[4] = {u.x, u.y, u.z, u.w};
            uint32_t k[8];
#pragma unroll
            for (int j = 0; j < 4; j++) { k[2 * j] = key_of((uint16_t)(w[j] & 0xffffu)); k[2 * j + 1] = key_of((uint16_t)(w[j] >> 16)); }
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const unsigned long long c = ((unsigned long long)k[j] << 32) | (0xffffffffu - (uint32_t)(begin + i + j));
                best = c > best ? c : best;
            }
            uint4 o = make_uint4(k[0] | (k[1] << 16), k[2] | (k[3] << 16), k[4] | (k[5] << 16), k[6] | (k[7] << 16));
            *reinterpret_cast<uint4*>(keys + i) = o;
        }
    }
    for (int i = vec_end + threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t k = key_of(s16[i]);
        keys[i] = (uint16_t)k;
        const unsigned long long c = ((unsigned long long)k << 32) | (0xffffffffu - (uint32_t)(begin + i));
        best = c > best ? c : best;
    }
    best = block_max_u64(best, scratch);
    if (threadIdx.x == 0) cta_max = best;
    cluster.sync();
    unsigned long long gmax = 0;
    for (unsigned r = 0; r < C; r++) {
        const unsigned long long c = *cluster.map_shared_rank(&cta_max, r);
        gmax = c > gmax ? c : gmax;
    }
    const uint32_t max_key = (uint32_t)(gmax >> 32);
    const int64_t max_index = vocab_offset + (int64_t)(0xffffffffu - (uint32_t)gmax);

    const float temp = temperature[row];
    if (!(temp > 0.f)) {                                              // greedy (every CTA of the cluster takes this branch)
        if (rank == 0 && threadIdx.x == 0) {
            out_tokens[row] = max_index;
            if (out_pairs) { out_pairs[2 * row] = value_of<T>(max_key); out_pairs[2 * row + 1] = (float)max_index; }
        }
        cluster.sync();
        return;
    }

    // ---- top-k threshold
    uint32_t thr = 0;
    const int k = top_k[row];
    if (k > 0 && k < V) {
        for (int i0 = threadIdx.x & ~31; i0 < n; i0 += blockDim.x) {
            const int i = i0 + (threadIdx.x & 31);
            const uint32_t key = i < n ? keys[i] : 0u;
            warp_hist_add(h_cnt_hi, i < n, key >> 8, 1ull);
        }
        merge_hist(cluster, h_cnt_hi, merged);
        select_bin(merged, 0, (double)k, &sel_bin, &sel_above);
        const uint32_t hi = (uint32_t)sel_bin;
        const unsigned long long above = sel_above;
        for (int i0 = threadIdx.x & ~31; i0 < n; i0 += blockDim.x) {
            const int i = i0 + (threadIdx.x & 31);
            const uint32_t key = i < n ? keys[i] : 0u;
            warp_hist_add(h_cnt_lo, i < n && (key >> 8) == hi, key & 255, 1ull);
        }
        merge_hist(cluster, h_cnt_lo, merged);
        select_bin(merged, above, (double)k, &sel_bin, &sel_above);
        thr = (hi << 8) | (uint32_t)sel_bin;
    }

    // ---- top-p threshold over the survivors
    const float p = top_p[row];
    if (p < 1.f) {
        const float m = value_of<T>(max_key);
        auto mass = [&](uint32_t key) {
            const float q = expf(__fdiv_rn(__fsub_rn(value_of<T>(key), m), temp));
            return (unsigned long long)__float2ull_rn(__fmul_rn(q, kMassScale));
        };
        for (int i0 = threadIdx.x & ~31; i0 < n; i0 += blockDim.x) {
            const int i = i0 + (threadIdx.x & 31);
            const uint32_t key = i < n ? keys[i] : 0u;
            const bool in = i < n && key >= thr;
            warp_hist_add(h_mass_hi, in, key >> 8, in ? mass(key) : 0ull);
        }
        merge_hist(cluster, h_mass_hi, merged);
        if (threadIdx.x < 32) {                                       // Z: exact integer total
            unsigned long long z = 0;
            for (int j = threadIdx.x; j < 256; j += 32) z += merged[j];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
            if (threadIdx.x == 0) scratch[0] = z;
        }
        __syncthreads();
        const double target = (double)p * (double)scratch[0];
        select_bin(merged, 0, target, &sel_bin, &sel_above);
        const uint32_t hi = (uint32_t)sel_bin;
        const unsigned long long above = sel_above;
        for (int i0 = threadIdx.x & ~31; i0 < n; i0 += blockDim.x) {
            const int i = i0 + (threadIdx.x & 31);
            const uint32_t key = i < n ? keys[i] : 0u;
            const bool in = i < n && (key >> 8) == hi && key >= thr;
            warp_hist_add(h_mass_lo, in, key & 255, in ? mass(key) : 0ull);
        }
        merge_hist(cluster, h_mass_lo, merged);
        select_bin(merged, above, target, &sel_bin, &sel_above);
        const uint32_t tp = (hi << 8) | (uint32_t)sel_bin;
        thr = tp > thr ? tp : thr;
    }

    // ---- Gumbel-max over the kept tokens; the noise of 4 consecutive GLOBAL indices comes from one Philox call
    const uint64_t sd = (uint64_t)seed[row];
    const uint32_t k0 = (uint32_t)sd, k1 = (uint32_t)(sd >> 32), ctr_pos = (uint32_t)pos[row];
    float bs = -INFINITY;
    int64_t bi = INT64_MAX;
    if (n > 0) {
        const int64_t g0 = (vocab_offset + begin) >> 2, g1 = (vocab_offset + begin + n - 1) >> 2;
        for (int64_t g = g0 + threadIdx.x; g <= g1; g += blockDim.x) {
            uint32_t kk[4];
            bool any = false;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int64_t lv = 4 * g + j - vocab_offset - begin;
                const uint32_t key = (lv >= 0 && lv < n) ? keys[lv] : 0u;
                kk[j] = (lv >= 0 && lv < n && key >= thr) ? key : 0xffffffffu;       // 0xffffffff: not kept
                any |= kk[j] != 0xffffffffu;
            }
            if (!any) continue;
            const uint4 x = philox4x32_10(make_uint4((uint32_t)g, ctr_pos, 0u, 0u), k0, k1);
            const uint32_t xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
            for (int j = 0; j < 4; j++) {
                if (kk[j] == 0xffffffffu) continue;
                const float s = __fadd_rn(__fdiv_rn(value_of<T>(kk[j]), temp), gumbel_of(xs[j]));
                if (better(s, 4 * g + j, bs, bi)) { bs = s; bi = 4 * g + j; }
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float s = __shfl_xor_sync(0xffffffffu, bs, o);
        const int64_t i = __shfl_xor_sync(0xffffffffu, bi, o);
        if (better(s, i, bs, bi)) { bs = s; bi = i; }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { warp_score[warp] = bs; warp_index[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); w++)
            if (better(warp_score[w], warp_index[w], bs, bi)) { bs = warp_score[w]; bi = warp_index[w]; }
        cta_score = bs;
        cta_index = bi;
    }
    cluster.sync();
    if (rank == 0 && threadIdx.x == 0) {
        for (unsigned r = 1; r < C; r++) {
            const float s = *cluster.map_shared_rank(&cta_score, r);
            const int64_t i = *cluster.map_shared_rank(&cta_index, r);
            if (better(s, i, bs, bi)) { bs = s; bi = i; }
        }
        out_tokens[row] = bi;
        if (out_pairs) { out_pairs[2 * row] = bs; out_pairs[2 * row + 1] = (float)bi; }
    }
    cluster.sync();                                                   // peers' shared memory stays valid until rank 0 has read it
}

template <typename T>
int launch(const void* logits, int64_t rows, int V, int64_t row_stride, int64_t vocab_offset, const float* temperature,
           const int32_t* top_k, const float* top_p, const int64_t* seed, const int32_t* pos, int64_t* out_tokens,
           float* out_pairs, cudaStream_t stream) {
    const int C = cluster_size(rows, V);
    const int slice = ((V + C - 1) / C + 7) & ~7;
    const size_t smem = (size_t)slice * sizeof(uint16_t);
    static unsigned long long configured = 0;
    if (first_use_on_this_device(configured))
        cudaFuncSetAttribute(sample_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSliceBytes);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(rows * C));
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, sample_kernel<T>, (const T*)logits, row_stride, V, vocab_offset, slice,
                                       temperature, top_k, top_p, seed, pos, out_tokens, out_pairs);
    if (e != cudaSuccess) {
        set_error("sample_tokens: %s", cudaGetErrorString(e));
        return (int)e;
    }
    return check_launch("sample_tokens");
}

}  // namespace
}  // namespace sllm

extern "C" int sllm_sample_tokens(const void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride,
                                  int64_t vocab_offset, const float* temperature, const int32_t* top_k, const float* top_p,
                                  const int64_t* seed, const int32_t* pos, int64_t* out_tokens, float* out_pairs,
                                  sllm_dtype_t dtype, sllm_stream_t stream) {
    using namespace sllm;
    SLLM_REQUIRE(dtype == SLLM_F16 || dtype == SLLM_BF16, "sample_tokens: unsupported dtype tag %d", (int)dtype);
    SLLM_REQUIRE(num_rows >= 0 && num_rows <= (1 << 20), "sample_tokens: num_rows %lld out of range", (long long)num_rows);
    SLLM_REQUIRE(vocab_size > 0, "sample_tokens: vocab_size must be positive, got %d", vocab_size);
    SLLM_REQUIRE(((int64_t)(vocab_size + kMaxCluster - 1) / kMaxCluster + 7) / 8 * 8 * 2 <= kMaxSliceBytes,
                 "sample_tokens: vocab_size %d does not fit the shared memory of a %d-CTA cluster", vocab_size, kMaxCluster);
    SLLM_REQUIRE(vocab_offset >= 0 && vocab_offset + vocab_size <= (1 << 24),
                 "sample_tokens: global vocabulary indices must stay below 2^24 (vocab_offset %lld)", (long long)vocab_offset);
    SLLM_REQUIRE(logits_row_stride >= vocab_size, "sample_tokens: logits_row_stride %lld < vocab_size %d",
                 (long long)logits_row_stride, vocab_size);
    if (num_rows == 0) return 0;
    SLLM_REQUIRE(logits && temperature && top_k && top_p && seed && pos && out_tokens, "sample_tokens: null pointer");
    SLLM_DISPATCH_DTYPE(dtype, return launch<T>(logits, num_rows, vocab_size, logits_row_stride, vocab_offset, temperature,
                                                top_k, top_p, seed, pos, out_tokens, out_pairs, (cudaStream_t)stream));
}
