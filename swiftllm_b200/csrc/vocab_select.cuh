// What the kernels that read whole vocabulary rows of 16-bit logits share (sampling.cu, logprobs.cu, penalties.cu,
// prompt_logprobs.cu):
//   device  the 16-byte row load, the order-preserving 16-bit keys (keys8 / pack8, stage_keys), the (key desc, id asc) pair,
//           the block reductions, the exact two-byte radix select over per-CTA histograms merged through distributed shared
//           memory (select_bin, select_low_byte), the top-N floor (nth_largest) and the fixed-point log-sum-exp terms
//           (mass_of / lse_of) that make both log-probability kernels agree bit for bit;
//   host    the cluster geometry (cluster_geometry, slice_fits) and the cluster launch (launch_cluster) of the kernels that run
//           one thread-block cluster per row.
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
constexpr int kKeyBytes = 2, kKeyAlign = 8;        // staged keys: uint16, slices of whole uint4 vectors

// 16 logits bytes that bypass L1; `evict_first`: read for the last time, so L2 evicts them first
__device__ __forceinline__ uint4 ld_row16(const void* p, bool evict_first = false) {
    uint4 u;
    if (evict_first)
        asm volatile("{\n\t.reg .b64 pol;\n\tcreatepolicy.fractional.L2::evict_first.b64 pol, 1.0;\n\t"
                     "ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], pol;\n\t}"
                     : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(p));
    else
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(p));
    return u;
}

__device__ __forceinline__ uint32_t key_of(uint16_t bits) {
    if (bits == 0x8000u) bits = 0;                  // -0 -> +0
    return (bits & 0x8000u) ? (~bits & 0xffffu) : (bits | 0x8000u);
}
template <typename T> __device__ __forceinline__ float value_of(uint32_t key) {
    const uint16_t bits = (key & 0x8000u) ? (uint16_t)(key ^ 0x8000u) : (uint16_t)(~key & 0xffffu);
    if constexpr (std::is_same<T, __half>::value) return __half2float(__ushort_as_half(bits));
    else return __uint_as_float((uint32_t)bits << 16);
}

// the keys of 8 logits loaded as one uint4, and 8 keys packed back into one
__device__ __forceinline__ void keys8(const uint4& u, uint32_t (&k)[8]) {
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; j++) { k[2 * j] = key_of((uint16_t)(w[j] & 0xffffu)); k[2 * j + 1] = key_of((uint16_t)(w[j] >> 16)); }
}
__device__ __forceinline__ uint4 pack8(const uint32_t (&k)[8]) {
    return make_uint4(k[0] | (k[1] << 16), k[2] | (k[3] << 16), k[4] | (k[5] << 16), k[6] | (k[7] << 16));
}

// (key desc, id asc) as one unsigned order: larger is better, and no two ids share a value
__device__ __forceinline__ unsigned long long pair_of(uint32_t key, int id) {
    return ((unsigned long long)key << 32) | (0xffffffffu - (uint32_t)id);
}

// key_of of +inf and -inf: keys above the first are NaN / +inf, keys below the second are NaN
template <typename T> struct InfKeys;
template <> struct InfKeys<__half> { static constexpr uint32_t pos = 0xfc00u, neg = 0x03ffu; };
template <> struct InfKeys<__nv_bfloat16> { static constexpr uint32_t pos = 0xff80u, neg = 0x007fu; };

// Stages the n logits at src as keys in keys[0 .. n) (16-byte loads when src is 16-byte aligned) and calls see(key, i) for
// every one of them, in the thread that converts it.  Block-wide; no barrier.
template <typename See>
__device__ __forceinline__ void stage_keys(const uint16_t* src, int n, uint16_t* keys, See&& see) {
    int vec_end = 0;
    if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        vec_end = n & ~7;
        for (int i = 8 * threadIdx.x; i < vec_end; i += 8 * blockDim.x) {
            uint32_t k[8];
            keys8(ld_row16(src + i), k);
#pragma unroll
            for (int j = 0; j < 8; j++) see(k[j], i + j);
            *reinterpret_cast<uint4*>(keys + i) = pack8(k);
        }
    }
    for (int i = vec_end + threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t k = key_of(src[i]);
        keys[i] = (uint16_t)k;
        see(k, i);
    }
}

// The fixed-point mass round(expf(l - m) * 2^40) of the logit with key `key` against the row maximum m, and the log-sum-exp
// m + logf(Z * 2^-40) of the exact integer sum Z of those masses: both log-probability kernels compute their values through
// these two, so they agree bit for bit.
template <typename T> __device__ __forceinline__ unsigned long long mass_of(uint32_t key, float m) {
    return __float2ull_rn(__fmul_rn(expf(__fsub_rn(value_of<T>(key), m)), kMassScale));
}
__device__ __forceinline__ float lse_of(float m, unsigned long long Z) {
    return __fadd_rn(m, logf(__fmul_rn(__ull2float_rn(Z), 1.0f / kMassScale)));
}

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

// The N-th largest of a[0 .. count) (1 <= N <= count), written to *out by the threads that hold it (all write the same
// value).  Block-wide, ends with a barrier.
__device__ __forceinline__ void nth_largest(const uint32_t* a, int count, int N, uint32_t* out) {
    if ((int)threadIdx.x < count) {
        const uint32_t v = a[threadIdx.x];
        int gt = 0, ge = 0;
        for (int j = 0; j < count; j++) { gt += a[j] > v; ge += a[j] >= v; }
        if (gt < N && N <= ge) *out = v;
    }
    __syncthreads();
}

// Entries N .. top_n - 1 of one row's top-N outputs: id -1 and NaN.  Thread t of the nt threads taking part.
__device__ __forceinline__ void fill_top_tail(int32_t* ids, float* logprobs, int N, int top_n, int t, int nt) {
    for (int j = N + t; j < top_n; j += nt) {
        ids[j] = -1;
        logprobs[j] = NAN;
    }
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

// The low byte of an exact two-byte radix select over the cluster's keys[0 .. n) slices: the largest key tau such that the
// weight of the counted keys >= tau reaches `target`.  The caller has filled the high-byte histogram (bin key >> 8) of the keys
// for which counts(key) holds, each adding its weight, merged it into `merged` and picked its bin `hi` with select_bin, which
// also gave `above`, the weight of the counted keys in the bins above hi.  This fills this CTA's zeroed low-byte histogram h_lo
// (left in place: bin tau & 255 holds the CTA's keys equal to tau), merges it and picks the low byte.  `above` is read only
// then, so the caller decides whether it stays in shared memory or in a register until that point (which changes register
// allocation, not results).  weight(key, in) is called for every key of the slice and only read where `in` (the key counts
// and lies in bin hi), so a costly weight can skip the other keys.  Returns tau and the weight of the counted keys > tau.
// sel_bin / sel_above: shared scratch of select_bin.
struct Selected { uint32_t tau; unsigned long long above; };
template <typename Counts, typename Weight>
__device__ __forceinline__ Selected select_low_byte(cg::cluster_group& cluster, const uint16_t* keys, int n, uint32_t hi,
                                                    const unsigned long long& above, unsigned long long* merged,
                                                    unsigned long long* h_lo, double target, Counts&& counts, Weight&& weight,
                                                    int* sel_bin, unsigned long long* sel_above) {
    for (int i0 = threadIdx.x & ~31; i0 < n; i0 += blockDim.x) {
        const int i = i0 + (threadIdx.x & 31);
        const uint32_t key = i < n ? keys[i] : 0u;
        const bool in = i < n && (key >> 8) == hi && counts(key);
        warp_hist_add(h_lo, in, key & 255, weight(key, in));
    }
    merge_hist(cluster, h_lo, merged);
    select_bin(merged, above, target, sel_bin, sel_above);
    return {(hi << 8) | (uint32_t)*sel_bin, *sel_above};
}

// The four-byte form of the same select over a 32-bit order of the keys: the largest u such that the weight of the counted
// keys with order(key) >= u reaches `target` (one histogram, DSMEM merge and select_bin per byte, high byte first).  order(key)
// is called for every staged key and only read where counts(key) holds; weight(key) where the key counts and matches the bytes
// chosen so far.  h: this CTA's four zeroed 256-bin histograms (h[256 * j] for byte 3 - j), used once each.  Block-wide; the
// caller guarantees the target is reached (it is at most the total weight).
template <typename Counts, typename Order, typename Weight>
__device__ __forceinline__ uint32_t select_u32(cg::cluster_group& cluster, const uint16_t* keys, int n,
                                               unsigned long long* h, unsigned long long* merged, double target,
                                               Counts&& counts, Order&& order, Weight&& weight, int* sel_bin,
                                               unsigned long long* sel_above) {
    uint32_t prefix = 0;
    unsigned long long above = 0;
#pragma unroll 1
    for (int j = 0; j < 4; j++) {
        const int sh = 24 - 8 * j;
        for (int i0 = threadIdx.x & ~31; i0 < n; i0 += blockDim.x) {
            const int i = i0 + (threadIdx.x & 31);
            const uint32_t key = i < n ? keys[i] : 0u;
            const bool c = i < n && counts(key);
            const uint32_t o = c ? order(key) : 0u;
            const bool in = c && (uint32_t)((unsigned long long)o >> (sh + 8)) == prefix;
            warp_hist_add(h + 256 * j, in, (o >> sh) & 255u, in ? weight(key) : 0ull);
        }
        merge_hist(cluster, h + 256 * j, merged);
        select_bin(merged, above, target, sel_bin, sel_above);
        prefix = (prefix << 8) | (uint32_t)*sel_bin;
        above = *sel_above;
    }
    return prefix;
}

// Block-wide min of a uint32 (all threads get it), through block_max_u64.
__device__ __forceinline__ uint32_t block_min_u32(uint32_t v, unsigned long long* scratch) {
    return 0xffffffffu - (uint32_t)block_max_u64(0xffffffffu - v, scratch);
}

// ---------------------------------------------------------------- host: one thread-block cluster of C CTAs per row

// Whether a row of V entries split over c CTAs, each slice rounded up to `align` entries, fits kMaxSliceBytes per CTA.
inline int64_t slice_of(int64_t V, int c, int align) { return ((V + c - 1) / c + align - 1) / align * align; }
inline bool slice_fits(int64_t V, int c, int bytes_per_entry, int align) {
    return slice_of(V, c, align) * bytes_per_entry <= kMaxSliceBytes;
}

struct ClusterGeometry { int C, slice; };
// C: the smallest cluster whose slices fit in shared memory, raised towards rows * C >= the SM count for small batches.
// The caller has checked slice_fits(V, kMaxCluster, ...).
inline ClusterGeometry cluster_geometry(int64_t rows, int V, int bytes_per_entry, int align) {
    int c = 1;
    while (c < kMaxCluster && !slice_fits(V, c, bytes_per_entry, align)) c *= 2;
    while (c < kMaxCluster && rows * c * 2 <= 132) c *= 2;
    return {c, (int)slice_of(V, c, align)};
}

// Launches Kernel on rows * C CTAs of kThreads in clusters of C, with smem_bytes of dynamic shared memory
template <auto Kernel, typename... Args>
int launch_cluster(int64_t rows, int C, size_t smem_bytes, cudaStream_t stream, const char* name, Args... args) {
    if (int e = fit_dynamic_smem<Kernel>(smem_bytes, name)) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(rows * C));
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, Kernel, args...);
    if (e != cudaSuccess) {
        set_error("%s: %s", name, cudaGetErrorString(e));
        return (int)e;
    }
    return check_launch(name);
}

}  // namespace
}  // namespace sllm
