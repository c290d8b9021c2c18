// Device helpers shared by the kernels that work on whole vocabulary rows with one thread-block cluster per row
// (sampling.cu, logprobs.cu): the order-preserving 16-bit keys, the cluster geometry, and the exact two-byte radix select over
// per-CTA histograms merged through distributed shared memory.  prompt_logprobs.cu (one CTA per row) uses the keys and the
// block reductions.
#pragma once
#include <cooperative_groups.h>
#include <type_traits>

#include "common.cuh"

namespace sllm {
namespace {

namespace cg = cooperative_groups;

constexpr int kThreads = 1024;
constexpr int kMaxCluster = 8;
constexpr int kMaxSliceBytes = 200 * 1024;
constexpr float kMassScale = 1099511627776.0f;     // 2^40

__device__ __forceinline__ uint32_t key_of(uint16_t bits) {
    if (bits == 0x8000u) bits = 0;                  // -0 -> +0
    return (bits & 0x8000u) ? (~bits & 0xffffu) : (bits | 0x8000u);
}
template <typename T> __device__ __forceinline__ float value_of(uint32_t key) {
    const uint16_t bits = (key & 0x8000u) ? (uint16_t)(key ^ 0x8000u) : (uint16_t)(~key & 0xffffu);
    if constexpr (std::is_same<T, __half>::value) return __half2float(__ushort_as_half(bits));
    else return __uint_as_float((uint32_t)bits << 16);
}

// key_of of +inf and -inf: keys above the first are NaN / +inf, keys below the second are NaN
template <typename T> struct InfKeys;
template <> struct InfKeys<__half> { static constexpr uint32_t pos = 0xfc00u, neg = 0x03ffu; };
template <> struct InfKeys<__nv_bfloat16> { static constexpr uint32_t pos = 0xff80u, neg = 0x007fu; };

// Block-wide sum of a u64 (all threads get it).
__device__ unsigned long long block_sum_u64(unsigned long long v, unsigned long long* scratch) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    v = lane < (int)(blockDim.x >> 5) ? scratch[lane] : 0ull;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Block-wide max of a u64 (all threads get it).
__device__ unsigned long long block_max_u64(unsigned long long v, unsigned long long* scratch) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w > v ? w : v;
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    v = lane < (int)(blockDim.x >> 5) ? scratch[lane] : 0ull;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w > v ? w : v;
    }
    return v;
}

// Sums the 256-bin histogram `hist` of every CTA of the cluster (DSMEM) into `merged`, in rank order.
__device__ void merge_hist(cg::cluster_group& cluster, unsigned long long* hist, unsigned long long* merged) {
    cluster.sync();
    if (threadIdx.x < 256) {
        unsigned long long s = 0;
        for (unsigned r = 0; r < cluster.num_blocks(); r++) s += cluster.map_shared_rank(hist, r)[threadIdx.x];
        merged[threadIdx.x] = s;
    }
    __syncthreads();
}

// hist[bin] += v for every lane with `valid` (called by whole warps).  Logits crowd into a few high-byte bins, so lanes that
// share a bin are summed first (exact integers) and one of them adds the sum; after a few rounds the rest add directly.
__device__ __forceinline__ void warp_hist_add(unsigned long long* hist, bool valid, uint32_t bin, unsigned long long v) {
    const int lane = threadIdx.x & 31;
    unsigned todo = __ballot_sync(0xffffffffu, valid && v != 0);
    for (int round = 0; todo && round < 4; round++) {
        const int leader = __ffs(todo) - 1;
        const uint32_t b = __shfl_sync(0xffffffffu, bin, leader);
        const bool mine = ((todo >> lane) & 1) && bin == b;
        unsigned long long sum = mine ? v : 0ull;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (lane == leader) atomicAdd(&hist[b], sum);
        todo &= ~__ballot_sync(0xffffffffu, mine);
    }
    if ((todo >> lane) & 1) atomicAdd(&hist[bin], v);
}

// Walking the bins from 255 down, the first bin b where above + sum(merged[b..255]) >= target.  Returns b and writes the
// sum of the bins above b (plus `above`) to *above_out.  Run by warp 0; results through shared memory.
__device__ void select_bin(const unsigned long long* merged, unsigned long long above, double target, int* bin_out,
                           unsigned long long* above_out) {
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        unsigned long long s = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) s += merged[255 - 8 * lane - j];
        unsigned long long incl = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long w = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += w;
        }
        const unsigned ok = __ballot_sync(0xffffffffu, (double)(above + incl) >= target);
        const int first = ok ? __ffs(ok) - 1 : 31;
        if (lane == first) {
            unsigned long long c = above + incl - s;
            int b = 255 - 8 * lane - 7;
            for (int j = 0; j < 8; j++) {
                const int bb = 255 - 8 * lane - j;
                if ((double)(c + merged[bb]) >= target) { b = bb; break; }
                c += merged[bb];
            }
            *bin_out = b;
            *above_out = c;
        }
    }
    __syncthreads();
}

// Cluster size: the smallest that fits a slice in shared memory, raised towards rows * C >= the SM count for small batches.
int cluster_size(int64_t rows, int V) {
    int c = 1;
    while (c < kMaxCluster && ((int64_t)(V + c - 1) / c) * 2 > kMaxSliceBytes) c *= 2;
    while (c < kMaxCluster && rows * c * 2 <= 132) c *= 2;
    return c;
}

}  // namespace
}  // namespace sllm
