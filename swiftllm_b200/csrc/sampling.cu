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
//   NaN / +inf  a row holding a NaN of either sign or +inf, or whose largest logit is -inf, is drawn greedily whatever T, k and
//            p: the largest key, smallest index among equal ones (a +NaN, else the first +inf, else the argmax of the rest; index
//            0 of an all -inf row).  Its masses and scores are undefined, so this keeps the token a valid id of the row.
// Both thresholds are exact: keys are 16 bits, so a radix select over the high and then the low byte finds them.  Masses are
// summed as 64-bit fixed-point integers (q * 2^40, rounded), so every sum is exact and independent of the order of additions:
// the result is a pure function of (logits, T, k, p, seed, pos), whatever the cluster size, batch or launch mode.
//
// Layout: one thread-block cluster of C CTAs per row (C chosen on the host so that rows * C covers the GPU at small batch).  Each
// CTA stages its contiguous slice of the row in shared memory as keys (HBM read once), every pass runs from there, and the
// per-CTA histograms / maxima / best (score, index) pairs are merged through distributed shared memory.  The staging, the
// two-byte select of both thresholds, the cluster geometry and the launch are those of vocab_select.cuh; the top-p mass
// (divided by T) is this kernel's own.
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

// The per-row filter arrays of the kTrunc instantiation (sllm_sample_tokens_truncated), passed after the other parameters so
// that theirs keep their offsets; the plain instantiation gets null pointers and never reads them.
struct TruncRows {
    const float* min_p;
    const float* typical_p;
    const float* xtc_threshold;
    const float* xtc_probability;
};

// The cluster's (smallest key, largest key, sum of w, sum of e) over the staged keys for which in(key) holds, acc(key, w, e)
// adding that key's terms.  Each CTA posts its part in `slot` (4 words of its shared memory, written once per kernel) and every
// thread reads all of them: a pure function of the row, whatever the cluster size.  Block-wide; ends with a cluster barrier.
struct Span { uint32_t lo, hi; unsigned long long w, e; };
template <typename In, typename Acc>
__device__ __forceinline__ Span cluster_span(cg::cluster_group& cluster, const uint16_t* keys, int n, unsigned long long* slot,
                                             unsigned long long* scratch, In&& in, Acc&& acc) {
    uint32_t lo = 0xffffffffu, hi = 0;
    unsigned long long w = 0, e = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t key = keys[i];
        if (in(key)) {
            lo = min(lo, key);
            hi = max(hi, key);
            acc(key, w, e);
        }
    }
    lo = block_min_u32(lo, scratch);
    hi = (uint32_t)block_max_u64(hi, scratch);
    w = block_sum_u64(w, scratch);
    e = block_sum_u64(e, scratch);
    if (threadIdx.x == 0) { slot[0] = lo; slot[1] = hi; slot[2] = w; slot[3] = e; }
    cluster.sync();
    Span s{0xffffffffu, 0u, 0ull, 0ull};
    for (unsigned r = 0; r < cluster.num_blocks(); r++) {
        const unsigned long long* p = cluster.map_shared_rank(slot, r);
        s.lo = min(s.lo, (uint32_t)p[0]);
        s.hi = max(s.hi, (uint32_t)p[1]);
        s.w += p[2];
        s.e += p[3];
    }
    return s;
}

template <typename T, bool kTrunc>
__global__ void __launch_bounds__(kThreads) sample_kernel(const T* __restrict__ logits, int64_t row_stride, int V,
                                                          int64_t vocab_offset, int slice, const float* __restrict__ temperature,
                                                          const int32_t* __restrict__ top_k, const float* __restrict__ top_p,
                                                          const int64_t* __restrict__ seed, const int32_t* __restrict__ pos,
                                                          int64_t* __restrict__ out_tokens, float* __restrict__ out_pairs,
                                                          TruncRows tr) {
    extern __shared__ uint16_t keys[];
    __shared__ unsigned long long h_cnt_hi[256], h_cnt_lo[256], h_mass_hi[256], h_mass_lo[256], merged[256];
    __shared__ unsigned long long scratch[32];
    __shared__ unsigned long long cta_max;
    __shared__ int cta_bad;
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
    // kTrunc: the four byte histograms of the typical-p select and the per-stage cluster_span slots
    __shared__ unsigned long long h_dist[kTrunc ? 4 * 256 : 1], span_slot[kTrunc ? 4 * 4 : 1];
    if constexpr (kTrunc)
        for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) h_dist[i] = 0;
    unsigned long long best = 0;
    bool bad = false;                                                 // a NaN of either sign or +inf
    stage_keys(reinterpret_cast<const uint16_t*>(src), n, keys, [&](uint32_t k, int i) {
        const unsigned long long c = pair_of(k, begin + i);
        best = c > best ? c : best;
        bad |= k >= InfKeys<T>::pos || k < InfKeys<T>::neg;
    });
    best = block_max_u64(best, scratch);
    bad = __syncthreads_or(bad);
    if (threadIdx.x == 0) { cta_max = best; cta_bad = bad; }
    cluster.sync();
    unsigned long long gmax = 0;
    for (unsigned r = 0; r < C; r++) {
        const unsigned long long c = *cluster.map_shared_rank(&cta_max, r);
        gmax = c > gmax ? c : gmax;
        bad |= *cluster.map_shared_rank(&cta_bad, r) != 0;
    }
    const uint32_t max_key = (uint32_t)(gmax >> 32);
    const int64_t max_index = vocab_offset + (int64_t)(0xffffffffu - (uint32_t)gmax);

    const float temp = temperature[row];
    if (!(temp > 0.f) || bad || max_key <= InfKeys<T>::neg) {        // greedy (every CTA of the cluster takes this branch)
        if (rank == 0 && threadIdx.x == 0) {
            out_tokens[row] = max_index;
            if (out_pairs) { out_pairs[2 * row] = value_of<T>(max_key); out_pairs[2 * row + 1] = (float)max_index; }
        }
        cluster.sync();
        return;
    }

    // ---- kTrunc: min-p, keep key >= the smallest key with q >= min_p (the maximum has q = 1, so some key passes)
    uint32_t thr = 0;
    const float m_row = value_of<T>(max_key);
    if constexpr (kTrunc) {
        const float mp = tr.min_p[row];
        if (mp > 0.f)
            thr = cluster_span(cluster, keys, n, span_slot, scratch,
                               [&](uint32_t key) { return expf(__fdiv_rn(__fsub_rn(value_of<T>(key), m_row), temp)) >= mp; },
                               [](uint32_t, unsigned long long&, unsigned long long&) {}).lo;
    }
    const uint32_t thr_min_p = thr;
    thr = 0;

    // ---- top-k threshold
    const int k = top_k[row];
    if (k > 0 && k < V) {
        for (int i0 = threadIdx.x & ~31; i0 < n; i0 += blockDim.x) {
            const int i = i0 + (threadIdx.x & 31);
            const uint32_t key = i < n ? keys[i] : 0u;
            warp_hist_add(h_cnt_hi, i < n, key >> 8, 1ull);
        }
        merge_hist(cluster, h_cnt_hi, merged);
        select_bin(merged, 0, (double)k, &sel_bin, &sel_above);
        const unsigned long long above = sel_above;
        thr = select_low_byte(cluster, keys, n, (uint32_t)sel_bin, above, merged, h_cnt_lo, (double)k,
                              [](uint32_t) { return true; }, [](uint32_t, bool) { return 1ull; }, &sel_bin, &sel_above).tau;
    }

    if constexpr (kTrunc) thr = thr_min_p > thr ? thr_min_p : thr;

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
        const unsigned long long above = sel_above;
        const uint32_t tp = select_low_byte(cluster, keys, n, (uint32_t)sel_bin, above, merged, h_mass_lo, target,
                                            [&](uint32_t key) { return key >= thr; },
                                            [&](uint32_t key, bool in) { return in ? mass(key) : 0ull; }, &sel_bin,
                                            &sel_above).tau;
        thr = tp > thr ? tp : thr;
    }

    // ---- kTrunc: typical-p and XTC over the survivors [thr, hi]; every kept set stays a key interval
    uint32_t hi = 0xffffu;
    if constexpr (kTrunc) {
        // x = (m - l) / T, q = expf(-x) (bit for bit the top-p q), w = round(q * 2^40), e = round(q * x * 2^40) (0 when w is)
        auto x_of = [&](uint32_t key) { return __fdiv_rn(__fsub_rn(m_row, value_of<T>(key)), temp); };
        auto w_of = [](float x) { return (unsigned long long)__float2ull_rn(__fmul_rn(expf(-x), kMassScale)); };
        auto alive = [&](uint32_t key) { return key >= thr && key <= hi; };
        auto add_w = [&](uint32_t key, unsigned long long& w, unsigned long long&) { w += w_of(x_of(key)); };
        const float typ = tr.typical_p[row];
        unsigned long long Z = 0;
        bool have_z = false;
        if (typ < 1.f) {
            const Span s = cluster_span(cluster, keys, n, span_slot + 4, scratch, alive,
                                        [&](uint32_t key, unsigned long long& w, unsigned long long& e) {
                                            const float x = x_of(key);
                                            const float q = expf(-x);
                                            const unsigned long long wk = __float2ull_rn(__fmul_rn(q, kMassScale));
                                            w += wk;
                                            if (wk) e += __float2ull_rn(__fmul_rn(__fmul_rn(q, x), kMassScale));
                                        });
            const float c = (float)((double)s.e / (double)s.w);
            auto d_bits = [&](uint32_t key) { return __float_as_uint(fabsf(__fsub_rn(x_of(key), c))); };
            // delta: the smallest distance whose survivors with d <= delta weigh >= typical_p * Z (order ~bits: small d first)
            const uint32_t u = select_u32(cluster, keys, n, h_dist, merged, (double)typ * (double)s.w, alive,
                                          [&](uint32_t key) { return ~d_bits(key); },
                                          [&](uint32_t key) { return w_of(x_of(key)); }, &sel_bin, &sel_above);
            const uint32_t delta = ~u;
            const Span k = cluster_span(cluster, keys, n, span_slot + 8, scratch,
                                        [&](uint32_t key) { return alive(key) && d_bits(key) <= delta; }, add_w);
            thr = k.lo;
            hi = k.hi;
            Z = k.w;
            have_z = true;
        }
        const float xp = tr.xtc_probability[row];
        if (xp > 0.f) {
            const uint64_t sd = (uint64_t)seed[row];
            const uint4 r = philox4x32_10(make_uint4(0u, (uint32_t)pos[row], 1u, 0u), (uint32_t)sd, (uint32_t)(sd >> 32));
            if (__fmul_rn((float)(r.x >> 9) + 0.5f, 1.0f / 8388608.0f) < xp) {
                if (!have_z) Z = cluster_span(cluster, keys, n, span_slot + 8, scratch, alive, add_w).w;
                const double bar = (double)tr.xtc_threshold[row] * (double)Z;
                // the top choices, the finite survivors whose w reaches threshold * Z, are the survivors from some key up: their
                // count and smallest key.  A -inf id (masked, banned) is never one, so threshold 0 stops at the least likely
                // finite survivor and the draw can never pick a -inf id over it.
                const Span t = cluster_span(cluster, keys, n, span_slot + 12, scratch,
                                            [&](uint32_t key) {
                                                return alive(key) && key > InfKeys<T>::neg && (double)w_of(x_of(key)) >= bar;
                                            },
                                            [](uint32_t, unsigned long long& w, unsigned long long&) { w += 1; });
                if (t.w >= 2) hi = t.lo;
            }
        }
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
                kk[j] = (lv >= 0 && lv < n && key >= thr && (!kTrunc || key <= hi)) ? key : 0xffffffffu;   // 0xffffffff: not kept
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

}  // namespace
}  // namespace sllm

namespace sllm {
namespace {

// The argument checks and the launch of both entry points; `truncated` selects the kTrunc instantiation.
int sample_tokens(const void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride, int64_t vocab_offset,
                  const float* temperature, const int32_t* top_k, const float* top_p, const int64_t* seed, const int32_t* pos,
                  int64_t* out_tokens, float* out_pairs, bool truncated, TruncRows tr, sllm_dtype_t dtype, cudaStream_t stream,
                  const char* name) {
    SLLM_REQUIRE(dtype == SLLM_F16 || dtype == SLLM_BF16, "%s: unsupported dtype tag %d", name, (int)dtype);
    SLLM_REQUIRE(num_rows >= 0 && num_rows <= (1 << 20), "%s: num_rows %lld out of range", name, (long long)num_rows);
    SLLM_REQUIRE(vocab_size > 0, "%s: vocab_size must be positive, got %d", name, vocab_size);
    SLLM_REQUIRE(slice_fits(vocab_size, kMaxCluster, kKeyBytes, kKeyAlign),
                 "%s: vocab_size %d does not fit the shared memory of a %d-CTA cluster", name, vocab_size, kMaxCluster);
    SLLM_REQUIRE(vocab_offset >= 0 && vocab_offset + vocab_size <= (1 << 24),
                 "%s: global vocabulary indices must stay below 2^24 (vocab_offset %lld)", name, (long long)vocab_offset);
    SLLM_REQUIRE(logits_row_stride >= vocab_size, "%s: logits_row_stride %lld < vocab_size %d", name,
                 (long long)logits_row_stride, vocab_size);
    if (num_rows == 0) return 0;
    SLLM_REQUIRE(logits && temperature && top_k && top_p && seed && pos && out_tokens, "%s: null pointer", name);
    SLLM_REQUIRE(!truncated || (tr.min_p && tr.typical_p && tr.xtc_threshold && tr.xtc_probability),
                 "%s: null filter array", name);
    const ClusterGeometry g = cluster_geometry(num_rows, vocab_size, kKeyBytes, kKeyAlign);
    const size_t smem = (size_t)g.slice * kKeyBytes;
    if (truncated)
        SLLM_DISPATCH_DTYPE(dtype, return launch_cluster<sample_kernel<T, true>>(
                                       num_rows, g.C, smem, stream, name, (const T*)logits, logits_row_stride, vocab_size,
                                       vocab_offset, g.slice, temperature, top_k, top_p, seed, pos, out_tokens, out_pairs, tr));
    SLLM_DISPATCH_DTYPE(dtype, return launch_cluster<sample_kernel<T, false>>(
                                   num_rows, g.C, smem, stream, name, (const T*)logits,
                                   logits_row_stride, vocab_size, vocab_offset, g.slice, temperature, top_k, top_p, seed, pos,
                                   out_tokens, out_pairs, tr));
}

}  // namespace
}  // namespace sllm

extern "C" int sllm_sample_tokens(const void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride,
                                  int64_t vocab_offset, const float* temperature, const int32_t* top_k, const float* top_p,
                                  const int64_t* seed, const int32_t* pos, int64_t* out_tokens, float* out_pairs,
                                  sllm_dtype_t dtype, sllm_stream_t stream) {
    return sllm::sample_tokens(logits, num_rows, vocab_size, logits_row_stride, vocab_offset, temperature, top_k, top_p, seed,
                               pos, out_tokens, out_pairs, false, sllm::TruncRows{}, dtype, (cudaStream_t)stream, "sample_tokens");
}

extern "C" int sllm_sample_tokens_truncated(const void* logits, int64_t num_rows, int vocab_size, int64_t logits_row_stride,
                                            int64_t vocab_offset, const float* temperature, const int32_t* top_k,
                                            const float* top_p, const int64_t* seed, const int32_t* pos, int64_t* out_tokens,
                                            float* out_pairs, const float* min_p, const float* typical_p,
                                            const float* xtc_threshold, const float* xtc_probability, sllm_dtype_t dtype,
                                            sllm_stream_t stream) {
    return sllm::sample_tokens(logits, num_rows, vocab_size, logits_row_stride, vocab_offset, temperature, top_k, top_p, seed,
                               pos, out_tokens, out_pairs, true, sllm::TruncRows{min_p, typical_p, xtc_threshold, xtc_probability},
                               dtype, (cudaStream_t)stream, "sample_tokens_truncated");
}
