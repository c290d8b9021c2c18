// Log-probabilities of given tokens and the top-N entries of [rows, V] logits, under the raw model distribution
// log_softmax(l) (no temperature, no top-k / top-p).  Semantics (restated in numpy by tests/logprobs_oracle.py):
//   m          the largest logit, found exactly through the order-preserving keys of sampling.cu (-0 == +0);
//   Z          sum over v of round(expf(l_v - m) * 2^40) as 64-bit integers: exact, so independent of the order of additions;
//   lse        m + logf(Z * 2^-40) in fp32;  logprob(v) = l_v - lse in fp32;
//   token      logprob(token_ids[row]); an id outside [0, V) gives NaN and is never read;
//   top-N      the N = min(top_n, V) ids with the largest keys, ordered by (key desc, id asc): ties at the boundary are broken by
//              the smaller id, so exactly N entries are returned.  Entries N .. top_n - 1 get id -1 and NaN;
//   NaN / +inf a row holding a NaN or +inf, or whose largest logit is -inf, gives NaN logprobs (its top ids still follow the
//              keys); a -inf logit of an otherwise finite row gives -inf.
// The result is a pure function of the row: it does not depend on the batch, the cluster size or the launch mode.
//
// Layout: one thread-block cluster of C CTAs per row; C, the slices, the launch, the staging and the two-byte select are
// vocab_select.cuh's, as in sampling.cu, and Z and lse go through the mass_of / lse_of that prompt_logprobs.cu also uses.
// Each CTA stages its slice as keys in shared memory (HBM read once); the passes are the max (with the NaN / +inf flag and
// per-warp maxima), Z together with the high-byte count histogram, the low-byte histogram (an exact radix select of tau, the
// N-th largest key; only keys >= the N-th largest warp maximum, a lower bound of tau, are counted, which keeps the
// shared-memory atomics few), and one in-order pass that takes every key > tau and the lowest-id ties at tau.  CTAs own
// increasing id ranges, so per-CTA tie counts in rank order tell each CTA how many of its ties to take.  Rank 0 gathers the
// <= 20 survivors over DSMEM and one warp sorts them.
// Algorithmic bytes: rows * V * 2 (logits) + rows * (12 + 8 * top_n).
//
// No fast-math here: expf / logf must be the accurate ones the restatement's tolerance is derived for.
#include "vocab_select.cuh"

namespace sllm {
namespace {

constexpr int kMaxTopN = 20;

template <typename T>
__global__ void __launch_bounds__(kThreads) logprobs_kernel(const T* __restrict__ logits, int64_t row_stride, int V, int slice,
                                                            const int64_t* __restrict__ token_ids, int top_n,
                                                            float* __restrict__ out_token_logprob,
                                                            int32_t* __restrict__ out_top_ids,
                                                            float* __restrict__ out_top_logprobs) {
    extern __shared__ uint16_t keys[];
    __shared__ unsigned long long h_hi[256], h_lo[256], merged[256];
    __shared__ unsigned long long scratch[32];
    __shared__ unsigned long long cta_max, cta_z;
    __shared__ int cta_bad, cand_n, sel_bin, warp_ties[32];
    __shared__ uint32_t warp_max[32], all_warp_max[32 * kMaxCluster], floor_key;
    __shared__ unsigned long long sel_above;
    __shared__ uint32_t cand_key[kMaxTopN];
    __shared__ int32_t cand_id[kMaxTopN];

    cg::cluster_group cluster = cg::this_cluster();
    const unsigned C = cluster.num_blocks(), rank = cluster.block_rank();
    const int64_t row = blockIdx.x / C;
    const int begin = (int)rank * slice;
    const int n = max(0, min(V, begin + slice) - begin);
    const T* src = logits + row * row_stride + begin;
    const int N = min(top_n, V);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // ---- stage the slice as keys; local max key and the NaN / +inf flag
    for (int i = threadIdx.x; i < 256; i += blockDim.x) h_hi[i] = h_lo[i] = 0;
    if (threadIdx.x == 0) cand_n = 0;
    unsigned long long best = 0;
    bool bad = false;
    stage_keys(reinterpret_cast<const uint16_t*>(src), n, keys, [&](uint32_t k, int) {
        best = k > best ? k : best;
        bad |= k >= InfKeys<T>::pos || k < InfKeys<T>::neg;
    });
    const uint32_t wmax = __reduce_max_sync(0xffffffffu, (uint32_t)best);
    if (lane == 0) warp_max[warp] = wmax;
    best = block_max_u64(best, scratch);
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0) { cta_max = best; cta_bad = bad; }
    cluster.sync();
    uint32_t max_key = 0;
    for (unsigned r = 0; r < C; r++) {
        max_key = max(max_key, (uint32_t)*cluster.map_shared_rank(&cta_max, r));
        bad |= *cluster.map_shared_rank(&cta_bad, r) != 0;
    }
    const float m = value_of<T>(max_key);
    bad |= m == -INFINITY;                                            // every logit -inf: no distribution (NaN, as log_softmax)

    // ---- a floor for the top-N select: the N-th largest warp maximum of the row.  The N warps holding the largest maxima have
    // one key >= it each, so tau >= floor, and only keys >= floor (usually a few dozen) enter the histograms below.  (A warp
    // without keys reports 0, which can only lower the floor.)
    const int W = (int)(blockDim.x >> 5) * (int)C;
    if (N > 0) {
        const unsigned wpc = blockDim.x >> 5;
        if (threadIdx.x < W) all_warp_max[threadIdx.x] = cluster.map_shared_rank(warp_max, threadIdx.x / wpc)[threadIdx.x % wpc];
        __syncthreads();
        nth_largest(all_warp_max, W, N, &floor_key);
    }
    const uint32_t lowest = N > 0 ? floor_key : 0u;

    // ---- Z (exact fixed point) and the high-byte counts of the top-N select, in one pass
    unsigned long long z = 0;
    for (int i0 = threadIdx.x & ~31; i0 < n; i0 += blockDim.x) {
        const int i = i0 + lane;
        const uint32_t key = i < n ? keys[i] : 0u;
        if (!bad && i < n) z += mass_of<T>(key, m);
        if (N > 0) warp_hist_add(h_hi, i < n && key >= lowest, key >> 8, 1ull);
    }
    z = block_sum_u64(z, scratch);
    if (threadIdx.x == 0) cta_z = z;

    if (N > 0) {
        // ---- tau = the N-th largest key (radix select over the two bytes of the keys >= floor), `above` = keys > tau in the row
        merge_hist(cluster, h_hi, merged);
        select_bin(merged, 0, (double)N, &sel_bin, &sel_above);
        const Selected sel = select_low_byte(cluster, keys, n, (uint32_t)sel_bin, sel_above, merged, h_lo, (double)N,
                                             [&](uint32_t key) { return key >= lowest; },
                                             [](uint32_t, bool) { return 1ull; }, &sel_bin, &sel_above);
        const uint32_t tau = sel.tau, lo = tau & 255;
        const int need_ties = N - (int)sel.above;                     // >= 1

        // ---- this CTA's share of the ties: the lowest ids first, and CTAs own increasing id ranges
        int prior = 0;
        for (unsigned r = 0; r < rank; r++) prior += (int)cluster.map_shared_rank(h_lo, r)[lo];
        const int quota = min((int)h_lo[lo], max(0, need_ties - prior));

        // ---- keys > tau, and ties whose in-order rank within the CTA is below the quota (<= N survivors per CTA)
        int ties_before_tile = 0;
        for (int t0 = 0; t0 < n; t0 += blockDim.x) {
            const int i = t0 + threadIdx.x;
            const uint32_t key = i < n ? keys[i] : 0u;
            const bool tie = i < n && key == tau;
            const unsigned bal = __ballot_sync(0xffffffffu, tie);
            if (lane == 0) warp_ties[warp] = __popc(bal);
            __syncthreads();
            int before = ties_before_tile + __popc(bal & ((1u << lane) - 1u)), tile = 0;
            for (int w = 0; w < (int)(blockDim.x >> 5); w++) {
                before += w < warp ? warp_ties[w] : 0;
                tile += warp_ties[w];
            }
            if ((i < n && key > tau) || (tie && before < quota)) {
                const int s = atomicAdd(&cand_n, 1);
                cand_key[s] = key;
                cand_id[s] = begin + i;
            }
            ties_before_tile += tile;
            __syncthreads();                                          // warp_ties is rewritten by the next tile
        }
    }
    cluster.sync();

    // ---- rank 0, warp 0: lse, the sorted top-N and the token's logprob
    if (rank == 0 && warp == 0) {
        unsigned long long Z = 0;
        for (unsigned r = 0; r < C; r++) Z += *cluster.map_shared_rank(&cta_z, r);
        const float lse = bad ? NAN : lse_of(m, Z);
        if (N > 0) {
            uint32_t k = 0;
            int32_t id = INT32_MAX;
            int off = 0;
            for (unsigned r = 0; r < C; r++) {
                const int cnt = *cluster.map_shared_rank(&cand_n, r);
                if (lane >= off && lane < off + cnt) {
                    k = cluster.map_shared_rank(cand_key, r)[lane - off];
                    id = cluster.map_shared_rank(cand_id, r)[lane - off];
                }
                off += cnt;
            }
            int place = 0;                                            // rank among the survivors: (key desc, id asc)
            for (int j = 0; j < N; j++) {
                const uint32_t kj = __shfl_sync(0xffffffffu, k, j);
                const int32_t ij = __shfl_sync(0xffffffffu, id, j);
                place += kj > k || (kj == k && ij < id);
            }
            if (lane < N) {
                out_top_ids[row * top_n + place] = id;
                out_top_logprobs[row * top_n + place] = __fsub_rn(value_of<T>(k), lse);
            }
        }
        fill_top_tail(out_top_ids + row * top_n, out_top_logprobs + row * top_n, N, top_n, lane, 32);
        if (lane == 0) {
            const int64_t tok = token_ids[row];
            float lp = NAN;
            if (tok >= 0 && tok < V)
                lp = __fsub_rn(value_of<T>(key_of(reinterpret_cast<const uint16_t*>(logits + row * row_stride)[tok])), lse);
            out_token_logprob[row] = lp;
        }
    }
    cluster.sync();                                                   // peers' shared memory stays valid until rank 0 has read it
}

}  // namespace
}  // namespace sllm

extern "C" int sllm_token_logprobs(const void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride,
                                   const int64_t* token_ids, int top_n, float* out_token_logprob, int32_t* out_top_ids,
                                   float* out_top_logprobs, sllm_dtype_t dtype, sllm_stream_t stream) {
    using namespace sllm;
    SLLM_REQUIRE(dtype == SLLM_F16 || dtype == SLLM_BF16, "token_logprobs: unsupported dtype tag %d", (int)dtype);
    SLLM_REQUIRE(num_rows >= 0 && num_rows <= (1 << 20), "token_logprobs: num_rows %lld out of range", (long long)num_rows);
    SLLM_REQUIRE(vocab_size > 0, "token_logprobs: vocab_size must be positive, got %d", vocab_size);
    SLLM_REQUIRE(slice_fits(vocab_size, kMaxCluster, kKeyBytes, kKeyAlign),
                 "token_logprobs: vocab_size %d does not fit the shared memory of a %d-CTA cluster", vocab_size, kMaxCluster);
    SLLM_REQUIRE(top_n >= 0 && top_n <= kMaxTopN, "token_logprobs: top_n %d outside [0, %d]", top_n, kMaxTopN);
    SLLM_REQUIRE(logits_row_stride >= vocab_size, "token_logprobs: logits_row_stride %lld < vocab_size %d",
                 (long long)logits_row_stride, vocab_size);
    if (num_rows == 0) return 0;
    SLLM_REQUIRE(logits && token_ids && out_token_logprob && (top_n == 0 || (out_top_ids && out_top_logprobs)),
                 "token_logprobs: null pointer");
    const ClusterGeometry g = cluster_geometry(num_rows, vocab_size, kKeyBytes, kKeyAlign);
    SLLM_DISPATCH_DTYPE(dtype, return launch_cluster<logprobs_kernel<T>>(
                                   num_rows, g.C, (size_t)g.slice * kKeyBytes, (cudaStream_t)stream, "token_logprobs",
                                   (const T*)logits, logits_row_stride, vocab_size, g.slice, token_ids, top_n, out_token_logprob,
                                   out_top_ids, out_top_logprobs));
}
