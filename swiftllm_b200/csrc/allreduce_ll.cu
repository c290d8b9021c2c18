// Tensor-parallel exchange, low-latency variant (SURVEY.md §8 f-3): reduce-scatter + residual add + RMSNorm + all-gather in
// ONE kernel with NO barrier.  Every "publish a flag, wait for everybody's flag" barrier costs one NVLink round trip, and the
// flag-based two-shot kernel (allreduce_norm.cu) pays two of them plus a peer-load round trip plus a system fence.
// Here data is PUSHED and carries its own validity (the NCCL "LL" idea): every 8-byte unit that crosses NVLink is
// {4 bytes of payload, 4-byte epoch tag}; a receiver polls the data itself until the tag equals the epoch of this exchange.
// One one-way latency per phase, nothing else:
//   phase 1 (all rows):       rank r pushes row t of its partial to the row's owner o = t % N     -> o.rs_recv[r][t / N]
//   phase 2 (owned rows):     owner polls the N-1 pushed copies, sums all N partials in rank order (fp32), adds ITS residual
//                             row, RMSNorm, writes the normalised row to its own x_out (plain) and pushes it to every
//                             other rank's ag_recv[t] (N-1 peer stores, or ONE multimem.st through the NVSwitch)
//   phase 3 (non-owned rows): poll ag_recv[t] and unpack it to x_out[t] (plain rows: the next GEMM's input)
// Wire traffic per rank 2 * 2(N-1)/N * T*H*2 B (tags double it) - irrelevant at decode sizes where latency, not bandwidth,
// is the cost; large exchanges (prefill) stay on the flag-based kernels.  Results are bit-identical to the two-shot kernel
// (same owner, same rank order, same rounding points).
//
// Tags: the per-slot epoch e (device memory, advanced by the last CTA to finish; replay-safe inside CUDA graphs).  The previous
// content of a slot's receive buffers carries an older epoch and can never be mistaken for this exchange's data.  Buffer reuse: a
// rank pushes into a peer's line only after it finished the previous exchange that used the line, which needed every row that
// peer owns - rows the peer produced AFTER consuming the line; an owner's broadcast needs this exchange's pushes of every rank,
// i.e. everybody has finished the previous one (tests/test_ll_exchange_protocol_sim.py checks every interleaving it can find).
// Residency: the grid is min(T, 2 x SMs) CTAs, rows are looped.  That is NOT always one wave: the kernel needs 126 (fp16) / 128
// (bf16) registers per thread, so at 512 threads (H >= 4096) only one CTA fits per SM and T > SMs runs in two waves.  It cannot
// deadlock as long as each GPU dispatches CTAs in increasing blockIdx order: grid and row-to-CTA map are the same on every rank,
// so in all three phases CTA c waits only for CTA c of each peer, and the lowest CTA index still unfinished anywhere is then
// resident on every rank where it has not finished.
// Peer loads, multimem.st, the epoch step and the host checks / launch are shared with allreduce_norm.cu (exchange.cuh); the
// add + RMSNorm row epilogue with rmsnorm_kernel (common.cuh).
#include "exchange.cuh"

namespace sllm {

struct LlParams {
    const void* partial;                    // this rank's partial [T, H], plain (local)
    void* rs_recv[MAX_RANKS];               // rs_recv of every rank (peer-mapped): [N src][rows_per_rank][H] in LL format (2x bytes)
    void* ag_recv[MAX_RANKS];               // ag_recv of every rank (peer-mapped): [max_tokens][H] in LL format
    void* mc_ag_recv;                       // multicast address of ag_recv, or NULL
    void* x_out;                            // local plain [T, H]
    void* residual; const void* weight;
    uint32_t* epoch;                        // local: uint32[32]: [slot] epoch, [16 + slot] done counter
    float eps;
    int rank, nranks, hidden, slot, num_tokens, rows_per_rank;   // rows_per_rank = capacity of one source's region of rs_recv
};

// {w0, tag, w1, tag}: two self-validating 8-byte units
__device__ __forceinline__ void st_ll(void* p, uint32_t w0, uint32_t w1, uint32_t tag) {
    asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(w0), "r"(tag), "r"(w1), "r"(tag) : "memory");
}
// `u` = a first (possibly stale) read of the line at p: spin until both 8-byte units of the 16-byte line carry `tag`.
// Callers issue the first reads of ALL their lines before calling this, so the loads are in flight together.
__device__ __forceinline__ uint4 poll_ll(const void* p, uint4 u, uint32_t tag, int rank, int what) {
    uint32_t spins = 0;
    while (u.y != tag || u.w != tag) {
        if (++spins > (1u << 26)) { printf("sllm: LL exchange watchdog (rank %d, phase %d, tag %u, saw %u/%u)\n", rank, what, tag, u.y, u.w); __trap(); }
        u = ld_peer(p);
    }
    return u;
}

template <typename T, bool NVLS>
__global__ void __launch_bounds__(512) allreduce_add_rmsnorm_ll_kernel(const LlParams p) {
    extern __shared__ uint4 row_smem[];
    __shared__ float red[16];
    const int nvec = p.hidden >> 3;                                  // 16-byte plain vectors per row; LL: 2 lines of 16 B each
    const uint32_t e = p.epoch[p.slot] + 1;
    const int64_t ll_row = (int64_t)p.hidden * 4;                    // bytes of one row in LL format
    const int N = p.nranks, me = p.rank;

    // ---- phase 1: push every row I do not own to its owner (never waits)
    for (int t = blockIdx.x; t < p.num_tokens; t += gridDim.x) {
        const int owner = t % N;
        if (owner == me) continue;
        const T* src = reinterpret_cast<const T*>(p.partial) + (int64_t)t * p.hidden;
        char* dst = reinterpret_cast<char*>(p.rs_recv[owner]) + ((int64_t)me * p.rows_per_rank + t / N) * ll_row;
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            const uint4 u = *reinterpret_cast<const uint4*>(src + 8 * i);
            st_ll(dst + 32 * i, u.x, u.y, e);
            st_ll(dst + 32 * i + 16, u.z, u.w, e);
        }
    }

    // ---- phase 2: rows I own - wait for the N-1 pushed partials, reduce in rank order, add residual, RMSNorm, broadcast
    for (int t = blockIdx.x; t < p.num_tokens; t += gridDim.x) {
        if (t % N != me) continue;
        const T* mine = reinterpret_cast<const T*>(p.partial) + (int64_t)t * p.hidden;
        const char* rbase = reinterpret_cast<const char*>(p.rs_recv[me]) + (int64_t)(t / N) * ll_row;
        T* rr = reinterpret_cast<T*>(p.residual) + (int64_t)t * p.hidden;
        float ss = 0.f;
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            // first reads of every source's two lines are issued back to back (independent loads in flight); late lines are
            // re-polled when their turn comes.  Accumulation in fixed rank order, fp32: the same sum as the other kernels.
            uint4 la[MAX_RANKS], lb[MAX_RANKS];
#pragma unroll
            for (int r = 0; r < MAX_RANKS; r++) {
                if (r < N && r != me) {
                    const char* q = rbase + (int64_t)r * p.rows_per_rank * ll_row + 32 * i;
                    la[r] = ld_peer(q); lb[r] = ld_peer(q + 16);
                }
            }
            const Vec8<T> own = ld_vec8(mine + 8 * i);
#pragma unroll
            for (int r = 0; r < MAX_RANKS; r++) {
                if (r < N) {
                    Vec8<T> v;
                    if (r == me) {
                        v = own;
                    } else {
                        const char* q = rbase + (int64_t)r * p.rows_per_rank * ll_row + 32 * i;
                        const uint4 x = poll_ll(q, la[r], e, me, 2), y = poll_ll(q + 16, lb[r], e, me, 2);
                        const uint4 u = make_uint4(x.x, x.z, y.x, y.z);
                        v = *reinterpret_cast<const Vec8<T>*>(&u);
                    }
                    acc_f32(acc, v);
                }
            }
            Vec8<T> sum;
#pragma unroll
            for (int j = 0; j < 4; j++) sum.v[j] = Traits<T>::from_f2(make_float2(acc[2 * j], acc[2 * j + 1]));
            add_residual(sum, rr + 8 * i, &row_smem[i], ss);
        }
        ss = warp_sum(ss);
        __syncthreads();                                             // red[] of the previous row fully consumed
        const float rstd = row_rstd(ss, red, p.hidden, p.eps);
        const T* wt = reinterpret_cast<const T*>(p.weight);
        T* xo = reinterpret_cast<T*>(p.x_out) + (int64_t)t * p.hidden;
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            const Vec8<T> a = *reinterpret_cast<Vec8<T>*>(&row_smem[i]);
            Vec8<T> o;
            rms_scale(o, a, rstd, wt + 8 * i);
            st_vec8(xo + 8 * i, o);                                  // my own copy: plain
            const uint4 u = *reinterpret_cast<const uint4*>(&o);
            const int64_t off = (int64_t)t * ll_row + 32 * i;
            if constexpr (NVLS) {                                    // the switch replicates the line into every rank's ag_recv
                multimem_st(reinterpret_cast<char*>(p.mc_ag_recv) + off, u.x, e, u.y, e);
                multimem_st(reinterpret_cast<char*>(p.mc_ag_recv) + off + 16, u.z, e, u.w, e);
            } else {
#pragma unroll
                for (int k = 1; k < MAX_RANKS; k++) {                // start with the next rank: owners do not all hit one target
                    if (k < N) {
                        int r = me + k;
                        if (r >= N) r -= N;
                        char* d = reinterpret_cast<char*>(p.ag_recv[r]) + off;
                        st_ll(d, u.x, u.y, e);
                        st_ll(d + 16, u.z, u.w, e);
                    }
                }
            }
        }
    }

    // ---- phase 3: rows owned by somebody else - wait for the normalised row, unpack it for the next GEMM
    for (int t = blockIdx.x; t < p.num_tokens; t += gridDim.x) {
        if (t % N == me) continue;
        const char* src = reinterpret_cast<const char*>(p.ag_recv[me]) + (int64_t)t * ll_row;
        T* xo = reinterpret_cast<T*>(p.x_out) + (int64_t)t * p.hidden;
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            uint4 a = ld_peer(src + 32 * i), b = ld_peer(src + 32 * i + 16);
            a = poll_ll(src + 32 * i, a, e, me, 3); b = poll_ll(src + 32 * i + 16, b, e, me, 3);
            *reinterpret_cast<uint4*>(xo + 8 * i) = make_uint4(a.x, a.z, b.x, b.z);
        }
    }

    advance_epoch(p.epoch, p.slot, e);
}

}  // namespace sllm

using namespace sllm;

// host_peer_rs_recv / host_peer_ag_recv: HOST arrays of `nranks` DEVICE pointers to THIS SLOT's receive buffers of every rank
// (symmetric memory): rs_recv = [nranks][rows_per_rank][hidden] and ag_recv = [>= num_tokens][hidden], both in LL format
// (4 bytes per element), zero-initialised once.  partial, x_out, residual, weight, epoch_state: local.  mc_ag_recv: multicast
// address of ag_recv (this slot) or NULL.  num_tokens <= nranks * rows_per_rank.
extern "C" int sllm_allreduce_add_rmsnorm_ll(const void* partial, void* const* host_peer_rs_recv, void* const* host_peer_ag_recv,
                                             void* mc_ag_recv, int rank, int nranks, int slot, void* epoch_state, void* x_out,
                                             void* residual, const void* weight, float eps, int64_t num_tokens, int hidden,
                                             int64_t rows_per_rank, sllm_dtype_t dtype, sllm_stream_t stream) {
    if (check_exchange("allreduce(LL)", rank, nranks, slot, 16, hidden, num_tokens)) return 1;
    if (num_tokens == 0) return 0;
    SLLM_REQUIRE(rows_per_rank > 0 && num_tokens <= rows_per_rank * nranks,
                 "allreduce(LL): %lld tokens exceed the receive buffers (%lld rows per rank x %d ranks)", (long long)num_tokens,
                 (long long)rows_per_rank, nranks);
    SLLM_REQUIRE(partial && host_peer_rs_recv && host_peer_ag_recv && epoch_state && x_out && residual && weight, "allreduce(LL): null pointer");
    LlParams p;
    for (int r = 0; r < nranks; r++) { p.rs_recv[r] = host_peer_rs_recv[r]; p.ag_recv[r] = host_peer_ag_recv[r]; }
    p.partial = partial; p.mc_ag_recv = mc_ag_recv; p.x_out = x_out; p.residual = residual; p.weight = weight;
    p.epoch = (uint32_t*)epoch_state; p.eps = eps; p.rank = rank; p.nranks = nranks; p.hidden = hidden; p.slot = slot;
    p.num_tokens = (int)num_tokens; p.rows_per_rank = (int)rows_per_rank;
    SLLM_REQUIRE((size_t)(hidden / 8) * sizeof(uint4) <= 48 * 1024, "allreduce(LL): hidden %d too large", hidden);
    const int64_t cap = 2LL * num_sms();                             // one wave below 512 threads, two at 512: see the kernel comment
    const unsigned grid = (unsigned)(num_tokens < cap ? num_tokens : cap);
    const bool nvls = mc_ag_recv != nullptr;
    const char* who = "allreduce(LL)", *kernel = "allreduce_add_rmsnorm_ll";
    return nvls ? launch_exchange<allreduce_add_rmsnorm_ll_kernel<__half, true>, allreduce_add_rmsnorm_ll_kernel<__nv_bfloat16, true>>(
                      who, kernel, dtype, grid, hidden, (cudaStream_t)stream, p)
                : launch_exchange<allreduce_add_rmsnorm_ll_kernel<__half, false>, allreduce_add_rmsnorm_ll_kernel<__nv_bfloat16, false>>(
                      who, kernel, dtype, grid, hidden, (cudaStream_t)stream, p);
}
