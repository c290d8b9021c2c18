// Tensor-parallel exchange fused with the op that always follows it (SURVEY.md §8 f-3):
//     x_sum = sum over ranks of the partial GEMM output   (one-shot all-reduce over NVLink peer memory)
//     residual <- h(x_sum) + residual ;  x_out <- rmsnorm(residual) * weight       (rmsnorm.py:39-65 semantics)
// in ONE kernel, instead of ncclAllReduce + fused_add_rmsnorm.  Every rank's partial lives in a symmetric buffer
// that all peers can read through NVLink / NVSwitch (P2P loads); each rank reads all N partials of every row in the
// SAME rank order with fp32 accumulation, so all ranks obtain bit-identical sums (no broadcast step needed).
//
// Synchronisation: a flag per (slot, source rank) in every rank's signal pad.  On entry, block 0 publishes
// "my partial for epoch e is complete" to all peers (system-scope release after the producing GEMM finished in stream
// order); every CTA waits until all N flags of its own pad reach e.  Two symmetric buffers alternate between
// consecutive exchanges, so a rank can only overwrite a buffer after every peer has passed the barrier of the
// exchange in between, i.e. finished reading it.  Epochs live in device memory (CUDA-graph replay safe).
// A watchdog traps instead of hanging if a peer never arrives.
// Flags, peer loads, the rank-ordered sum, the epoch step and the host checks / launch are shared with allreduce_ll.cu
// (exchange.cuh); the add + RMSNorm row epilogue with rmsnorm_kernel (common.cuh).
#include "exchange.cuh"

namespace sllm {

struct ArParams {
    const void* peer_buf[MAX_RANKS];         // partial [T, H] of every rank (peer-mapped device pointers)
    uint32_t* peer_flags[MAX_RANKS];         // signal pad of every rank: uint32 [slots][MAX_RANKS]
    uint32_t* epoch;                         // local device memory: uint32 [slots] epoch, then uint32 [slots] done-counter
    void* x_out; void* residual; const void* weight;
    float eps;
    int rank, nranks, hidden, slot, has_norm;
};

template <typename T>
__global__ void __launch_bounds__(512) allreduce_add_rmsnorm_kernel(const ArParams p) {
    extern __shared__ uint4 row_smem[];
    __shared__ float red[16];
    const int64_t t = blockIdx.x;
    const int nvec = p.hidden >> 3;
    const uint32_t e = p.epoch[p.slot] + 1;                 // epoch of this exchange (same value in every CTA)

    // ---- barrier: my partial is complete (stream order) -> tell every peer; wait for every peer's flag
    if (threadIdx.x < p.nranks) {
        if (blockIdx.x == 0) publish_flag(p, 0, e);
        wait_flag(p, 0, e, "sllm: all-reduce watchdog (rank %d waits for rank %d, epoch %u)\n");
    }
    __syncthreads();

    // ---- one-shot reduction of this token row, then fused add + RMSNorm
    T* rr = reinterpret_cast<T*>(p.residual) + t * p.hidden;
    float ss = 0.f;
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
        Vec8<T> sum;
        peer_sum(sum, p.peer_buf, p.nranks, t * p.hidden + 8 * i);
        add_residual(sum, rr + 8 * i, &row_smem[i], ss);
    }
    if (p.has_norm) {
        const float rstd = row_rstd(warp_sum(ss), red, p.hidden, p.eps);
        T* xo = reinterpret_cast<T*>(p.x_out) + t * p.hidden;
        const T* wt = reinterpret_cast<const T*>(p.weight);
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            const Vec8<T> a = *reinterpret_cast<Vec8<T>*>(&row_smem[i]);
            Vec8<T> o;
            rms_scale(o, a, rstd, wt + 8 * i);
            st_vec8(xo + 8 * i, o);
        }
    }
    advance_epoch(p.epoch, p.slot, e);
}

// ------------------------------------------------------------------ two-shot variant (reduce-scatter + all-gather by token rows)
// The one-shot kernel above makes every rank read all N partials of EVERY row: (N-1) * T * H remote bytes per rank, which is
// what limits it to TP 2..4.  Here token row t is OWNED by rank t % N: the owner alone reduces the row (reads N-1 remote
// partials), adds ITS residual row (the residual stays sharded by rows: only the owner ever needs it again), normalises, and
// pushes the normalised row into every rank's x_out buffer (P2P stores).  Remote traffic per rank: 2 * (N-1)/N * T * H bytes,
// 4x less than one-shot at N = 8.  Two barriers per exchange, both flag-based over peer memory:
//   A  "my partial is complete"           (published by every CTA - idempotent -, awaited by every CTA)
// With NVLS = true the N peer loads become ONE multimem.ld_reduce on the multicast address of the partial buffer (the NVSwitch
// sums the N copies with fp32 accumulation) and the N peer stores ONE multimem.st on the multicast address of x_out.
//   B  "my rows have landed everywhere"   published by the LAST CTA of a rank to finish (after a system fence), and awaited by
//      that same CTA for all ranks before the kernel may end - so the next kernel in the stream sees the whole x_out.
// A single x_out buffer per rank suffices: a peer can only write exchange k+1's rows after barrier A of k+1, i.e. after this
// rank has launched k+1, which is after everything that consumed x_out of exchange k in its stream.
struct Ar2Params {
    const void* peer_buf[MAX_RANKS];         // partial [T, H] of every rank
    void* peer_xout[MAX_RANKS];              // x_out [T, H] of every rank (symmetric, written by the row owners)
    uint32_t* peer_flags[MAX_RANKS];         // signal pad of every rank: uint32 [16][MAX_RANKS]; rows slot (A) and 8 + slot (B)
    uint32_t* epoch;
    void* residual; const void* weight;
    float eps;
    int rank, nranks, hidden, slot, num_tokens;
    // NVLS (template NVLS = true): multicast addresses of the partial buffer (this slot) and of x_out.  One
    // multimem.ld_reduce replaces the N peer loads (the NVSwitch sums the N copies, fp32 accumulation), one multimem.st the N
    // peer stores (the switch broadcasts).
    const void* mc_buf; void* mc_xout;
};

// 8 x 16-bit values summed over all GPUs of the multicast group by the switch (fp32 accumulation, one rounding)
template <typename T> __device__ __forceinline__ Vec8<T> multimem_ld_reduce_add(const T* mc);
template <> __device__ __forceinline__ Vec8<__half> multimem_ld_reduce_add<__half>(const __half* mc) {
    uint4 u;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(mc) : "memory");
    return *reinterpret_cast<Vec8<__half>*>(&u);
}
template <> __device__ __forceinline__ Vec8<__nv_bfloat16> multimem_ld_reduce_add<__nv_bfloat16>(const __nv_bfloat16* mc) {
    uint4 u;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(mc) : "memory");
    return *reinterpret_cast<Vec8<__nv_bfloat16>*>(&u);
}
template <typename T> __device__ __forceinline__ void st_vec8_peer(T* p, const Vec8<T>& v) {
    const uint4 u = *reinterpret_cast<const uint4*>(&v);
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(u.x), "r"(u.y), "r"(u.z), "r"(u.w) : "memory");
}

template <typename T, bool NVLS>
__global__ void __launch_bounds__(512) allreduce_add_rmsnorm_2shot_kernel(const Ar2Params p) {
    extern __shared__ uint4 row_smem[];
    __shared__ float red[16];
    __shared__ int s_last;
    const int64_t t = (int64_t)blockIdx.x * p.nranks + p.rank;     // the row this CTA owns (may be past the end)
    const int nvec = p.hidden >> 3;
    const uint32_t e = p.epoch[p.slot] + 1;

    // ---- barrier A.  EVERY CTA publishes (idempotent: the same epoch value; the partial is complete for all of them by stream
    // order), so progress never depends on CTA 0 being dispatched before the CTAs that wait.
    if (threadIdx.x < p.nranks) {
        publish_flag(p, 0, e);
        wait_flag(p, 0, e, "sllm: two-shot all-reduce watchdog A (rank %d waits for rank %d, epoch %u)\n");
    }
    __syncthreads();

    if (t < p.num_tokens) {
        // ---- reduce my row over all ranks (fixed order), add my residual row, RMSNorm
        T* rr = reinterpret_cast<T*>(p.residual) + t * p.hidden;
        float ss = 0.f;
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            Vec8<T> sum;                                            // h(sum over ranks)
            if constexpr (NVLS) sum = multimem_ld_reduce_add<T>(reinterpret_cast<const T*>(p.mc_buf) + t * p.hidden + 8 * i);
            else peer_sum(sum, p.peer_buf, p.nranks, t * p.hidden + 8 * i);
            add_residual(sum, rr + 8 * i, &row_smem[i], ss);
        }
        const float rstd = row_rstd(warp_sum(ss), red, p.hidden, p.eps);
        const T* wt = reinterpret_cast<const T*>(p.weight);
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            const Vec8<T> a = *reinterpret_cast<Vec8<T>*>(&row_smem[i]);
            Vec8<T> o;
            rms_scale(o, a, rstd, wt + 8 * i);
            // ---- all-gather: the normalised row goes to every rank (own copy included), starting with the next rank so the
            // N owners do not all hit the same destination at the same time
            if constexpr (NVLS) {
                const uint4 u = *reinterpret_cast<const uint4*>(&o);
                multimem_st(reinterpret_cast<T*>(p.mc_xout) + t * p.hidden + 8 * i, u.x, u.y, u.z, u.w);
            } else {
#pragma unroll
                for (int k = 0; k < MAX_RANKS; k++) {
                    if (k < p.nranks) {
                        int r = p.rank + 1 + k;
                        if (r >= p.nranks) r -= p.nranks;
                        st_vec8_peer(reinterpret_cast<T*>(p.peer_xout[r]) + t * p.hidden + 8 * i, o);
                    }
                }
            }
        }
    }

    // ---- barrier B: the last CTA of this rank publishes "all my rows are written" and waits for everybody's
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();                                    // this CTA's peer stores, made visible before the count
        uint32_t* done = p.epoch + 16 + p.slot;
        s_last = atomicAdd(done, 1u) == gridDim.x - 1;
        if (s_last) *done = 0;
    }
    __syncthreads();
    if (!s_last) return;
    if (threadIdx.x < p.nranks) {
        publish_flag(p, 8, e);
        wait_flag(p, 8, e, "sllm: two-shot all-reduce watchdog B (rank %d waits for rank %d, epoch %u)\n");
    }
    __syncthreads();
    if (threadIdx.x == 0) { __threadfence(); p.epoch[p.slot] = e; }     // every CTA of this launch has read the epoch by now
}

}  // namespace sllm

using namespace sllm;

// Two-shot variant: see the kernel comment.  host_peer_xout: HOST array of `nranks` device pointers to every rank's x_out
// buffer [>= num_tokens, hidden] (symmetric memory); the normalised activations appear in THIS rank's buffer.  `residual` is
// only maintained for the rows this rank owns (t % nranks == rank); weight is required.  slot < 8.
// mc_buf / mc_xout: multicast (NVLS) addresses of the partial buffer of this slot and of x_out, or NULL for peer loads / stores.
extern "C" int sllm_allreduce_add_rmsnorm_2shot(const void* const* host_peer_bufs, void* const* host_peer_xout,
                                                void* const* host_peer_flags, const void* mc_buf, void* mc_xout, int rank,
                                                int nranks, int slot, void* epoch_state, void* residual, const void* weight,
                                                float eps, int64_t num_tokens, int hidden, sllm_dtype_t dtype,
                                                sllm_stream_t stream) {
    SLLM_REQUIRE((mc_buf == nullptr) == (mc_xout == nullptr), "allreduce(2-shot): give both multicast addresses or neither");
    if (check_exchange("allreduce(2-shot)", rank, nranks, slot, 8, hidden, num_tokens)) return 1;
    if (num_tokens == 0) return 0;
    SLLM_REQUIRE(host_peer_bufs && host_peer_xout && host_peer_flags && epoch_state && residual && weight, "allreduce(2-shot): null pointer");
    Ar2Params p;
    for (int r = 0; r < nranks; r++) {
        p.peer_buf[r] = host_peer_bufs[r]; p.peer_xout[r] = host_peer_xout[r]; p.peer_flags[r] = (uint32_t*)host_peer_flags[r];
    }
    p.epoch = (uint32_t*)epoch_state; p.residual = residual; p.weight = weight; p.eps = eps;
    p.rank = rank; p.nranks = nranks; p.hidden = hidden; p.slot = slot; p.num_tokens = (int)num_tokens;
    p.mc_buf = mc_buf; p.mc_xout = mc_xout;
    const bool nvls = mc_buf != nullptr;
    const unsigned grid = (unsigned)((num_tokens + nranks - 1) / nranks);        // the same on every rank
    const char* who = "allreduce(2-shot)", *kernel = "allreduce_add_rmsnorm_2shot";
    return nvls ? launch_exchange<allreduce_add_rmsnorm_2shot_kernel<__half, true>, allreduce_add_rmsnorm_2shot_kernel<__nv_bfloat16, true>>(
                      who, kernel, dtype, grid, hidden, (cudaStream_t)stream, p)
                : launch_exchange<allreduce_add_rmsnorm_2shot_kernel<__half, false>, allreduce_add_rmsnorm_2shot_kernel<__nv_bfloat16, false>>(
                      who, kernel, dtype, grid, hidden, (cudaStream_t)stream, p);
}

// host_peer_bufs / host_peer_flags: HOST arrays of `nranks` device pointers (the symmetric buffer and the signal pad of
// every rank as mapped into this process).  epoch_state: local device memory, >= 32 uint32, zero-initialised once.
// weight == NULL: only residual <- h(sum) + residual (no norm output).
extern "C" int sllm_allreduce_add_rmsnorm(const void* const* host_peer_bufs, void* const* host_peer_flags, int rank, int nranks,
                                          int slot, void* epoch_state, void* x_out, void* residual, const void* weight, float eps,
                                          int64_t num_tokens, int hidden, sllm_dtype_t dtype, sllm_stream_t stream) {
    if (check_exchange("allreduce", rank, nranks, slot, 16, hidden, num_tokens)) return 1;
    if (num_tokens == 0) return 0;
    SLLM_REQUIRE(host_peer_bufs && host_peer_flags && epoch_state && residual && (weight == nullptr || x_out), "allreduce: null pointer");
    ArParams p;
    for (int r = 0; r < nranks; r++) { p.peer_buf[r] = host_peer_bufs[r]; p.peer_flags[r] = (uint32_t*)host_peer_flags[r]; }
    p.epoch = (uint32_t*)epoch_state; p.x_out = x_out; p.residual = residual; p.weight = weight; p.eps = eps;
    p.rank = rank; p.nranks = nranks; p.hidden = hidden; p.slot = slot; p.has_norm = weight != nullptr;
    return launch_exchange<allreduce_add_rmsnorm_kernel<__half>, allreduce_add_rmsnorm_kernel<__nv_bfloat16>>(
        "allreduce", "allreduce_add_rmsnorm", dtype, (unsigned)num_tokens, hidden, (cudaStream_t)stream, p);
}
