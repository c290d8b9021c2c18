// Peer-memory parts of the tensor-parallel exchange kernels (allreduce_norm.cu: one-shot and two-shot; allreduce_ll.cu: LL
// push): system-scope flags, volatile peer loads, the rank-ordered fp32 sum, the epoch step and the host-side checks and launch.
// The row epilogue they share with rmsnorm_kernel (add_residual / row_rstd / rms_scale) is in common.cuh.
#pragma once

#include "common.cuh"

namespace sllm {

constexpr int MAX_RANKS = 8;

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// peer data is produced by another GPU while this kernel may already be running: no read-only / L1 caching
__device__ __forceinline__ uint4 ld_peer(const void* p) {
    uint4 u;
    asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(p) : "memory");
    return u;
}
// a store moves bits: the bf16x2 vector form of multimem.st carries any four 32-bit words unchanged
__device__ __forceinline__ void multimem_st(void* mc, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("multimem.st.relaxed.sys.global.v4.bf16x2 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

template <typename T> __device__ __forceinline__ void acc_f32(float (&acc)[8], const Vec8<T>& v) {
#pragma unroll
    for (int j = 0; j < 4; j++) { float2 f = Traits<T>::to_f2(v.v[j]); acc[2 * j] += f.x; acc[2 * j + 1] += f.y; }
}
// h(sum over ranks r < n of the vector at bufs[r] + off), fp32 in rank order -> the same sum on every rank.  All n peer loads are
// issued before the first one is consumed (one NVLink round trip instead of n in series).
template <typename T> __device__ __forceinline__ void peer_sum(Vec8<T>& sum, const void* const* bufs, int n, int64_t off) {
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    uint4 pv[MAX_RANKS];
#pragma unroll
    for (int r = 0; r < MAX_RANKS; r++)
        if (r < n) pv[r] = ld_peer(reinterpret_cast<const T*>(bufs[r]) + off);
#pragma unroll
    for (int r = 0; r < MAX_RANKS; r++)
        if (r < n) acc_f32(acc, *reinterpret_cast<const Vec8<T>*>(&pv[r]));
#pragma unroll
    for (int j = 0; j < 4; j++) sum.v[j] = Traits<T>::from_f2(make_float2(acc[2 * j], acc[2 * j + 1]));
}

// Signal pads: uint32 [16 rows][MAX_RANKS source ranks] per rank; flag row row0 + p.slot.  Thread r < p.nranks tells peer r that
// p.rank reached epoch e (after a system fence: what this thread's CTA wrote before is visible first) ...
template <typename P> __device__ __forceinline__ void publish_flag(const P& p, int row0, uint32_t e) {
    __threadfence_system();
    st_release_sys(p.peer_flags[threadIdx.x] + (row0 + p.slot) * MAX_RANKS + p.rank, e);
}
// ... and waits until peer r's flag in this rank's pad reaches e, or traps after printing `watchdog` (rank, peer, epoch).
template <typename P> __device__ __forceinline__ void wait_flag(const P& p, int row0, uint32_t e, const char* watchdog) {
    const uint32_t* mine = p.peer_flags[p.rank] + (row0 + p.slot) * MAX_RANKS + threadIdx.x;
    uint32_t spins = 0;
    while ((int32_t)(ld_acquire_sys(mine) - e) < 0) {
        if (++spins > (1u << 27)) { printf(watchdog, p.rank, threadIdx.x, e); __trap(); }
    }
}

// Epoch state: uint32 [16 slots] epoch, then [16 slots] done counter.  The last CTA of the launch to get here stores e as the slot's
// epoch, after every CTA has read the old one.
__device__ __forceinline__ void advance_epoch(uint32_t* epoch, int slot, uint32_t e) {
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t* done = epoch + 16 + slot;
        if (atomicAdd(done, 1u) == gridDim.x - 1) { *done = 0; __threadfence(); epoch[slot] = e; }
    }
}

// ---------------------------------------------------------------- host
// rank, slot (< slots) and row shape of an exchange call; `who` starts every message
static inline int check_exchange(const char* who, int rank, int nranks, int slot, int slots, int hidden, int64_t num_tokens) {
    SLLM_REQUIRE(nranks >= 2 && nranks <= MAX_RANKS && rank >= 0 && rank < nranks, "%s: bad rank %d of %d", who, rank, nranks);
    SLLM_REQUIRE(slot >= 0 && slot < slots, "%s: bad slot %d", who, slot);
    SLLM_REQUIRE(hidden > 0 && hidden % 8 == 0 && num_tokens >= 0 && num_tokens < (1LL << 31),
                 "%s: hidden (%d) must be a positive multiple of 8", who, hidden);
    return 0;
}

// The dtype's instantiation, F16 or BF16, launched with row_threads threads and one row of dynamic shared memory
template <auto F16, auto BF16, typename P>
static int launch_exchange(const char* who, const char* kernel, sllm_dtype_t dtype, unsigned grid, int hidden, cudaStream_t st,
                           const P& p) {
    SLLM_REQUIRE(dtype == SLLM_F16 || dtype == SLLM_BF16, "%s: unknown dtype tag %d", who, (int)dtype);
    const size_t smem = (size_t)(hidden / 8) * sizeof(uint4);
    if (int e = dtype == SLLM_F16 ? fit_dynamic_smem<F16>(smem, kernel) : fit_dynamic_smem<BF16>(smem, kernel)) return e;
    (dtype == SLLM_F16 ? F16 : BF16)<<<grid, row_threads(hidden / 8), smem, st>>>(p);
    return check_launch(kernel);
}

}  // namespace sllm
