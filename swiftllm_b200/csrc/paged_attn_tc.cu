// Paged (decode) attention, generation 2: persistent, warp-specialised TMA + wgmma kernel (sm_90a).
//
// Reference being replaced: swiftllm/worker/kernels/paged_attn.py:9-108 (+ :111-149 via the merge kernel of
// paged_attn.cu when a sequence is split).  Shapes served: head_dim 128, block_size 16, GQA group <= 16, fp16/bf16.
//
// One persistent CTA per SM walks a static list of work items (sequence, kv head, split).  Per 128-token tile:
//   warp 4 (K) / warp 5 (V)  TMA producers: read 8 block-table entries, issue one 4-D tensor-map load per 16-token page
//                    (4 KiB, SWIZZLE_128B atoms [token-group][d-half][8 tok][64 d]) into 3-stage rings, completion on
//                    mbarriers; warp 4 also loads Q of the item (one TMA box per d-half).
//   warps 0-3        one warpgroup that issues the MMAs and runs the softmax, accumulators in registers:
//                    S^T[128 tok x NP heads] = K_tile (A, K-major) . Q^T (B, K-major)       (2 x 8 wgmma m64nNPk16)
//                    tile max per head across the warpgroup, p = exp2(s - m) -> bf16/fp16 P^T tile in shared memory,
//                    O^T[128 d x NP heads] = alpha * O^T + V_tile^T (A, MN-major) . P^T (B, K-major)   (2 x 8 wgmma)
// Tokens are the MMA M dimension (the transposed problem), so no tensor work is spent on padded query rows; the GQA
// group is the N dimension (padded to NP = 8 or 16 by reading neighbouring heads whose columns are never written back).
// HBM roofline: algorithmic bytes = sum_i len_i * nkv * 128 * 2 * sizeof(T) + 2 * Bd * nq * 128 * sizeof(T).
//
// Speculative verification (sllm_paged_attention_verify, paged_attn_verify_kernel) runs the same pipeline body under the VERIFY
// policy: entry i holds rows j < rows_i (query tokens at positions prefix_i + j); row j attends causally to positions
// [0, prefix_i + j].  The wgmma N dimension holds (row j, head h) pairs as column j * g + h (NP = 8, 16 or 32), so each
// (entry, kv head, split) item streams its K/V pages once for every row and head of the entry.  Q is one TMA box (64 d, g heads,
// qrows rows) per d-half over the row-strided packed q: columns of rows past the entry's count hold whatever the box read (the
// next entry's rows, or zero fill) and are never written.
#include "paged_attn_tc.cuh"
#include "tc_helpers.cuh"

namespace sllm {

using namespace tc;

constexpr int TC_D = 128;
constexpr int TC_BS = 16;                 // tokens per page
constexpr int TC_TILE = 128;              // tokens per pipeline stage (8 pages)
constexpr int TC_KSTAGES = 3;             // K ring (freed as soon as S = K.Q^T of the tile has completed)
constexpr int TC_VSTAGES = 3;             // V ring (freed when O = V^T.P^T of the tile has completed)
constexpr int TC_THREADS = 192;           // warps 0..3: MMA + softmax warpgroup, warp 4: K+Q producer, warp 5: V producer
constexpr int TC_NPAD = 16;               // largest wgmma N (heads, padded)
constexpr int TC_K_BYTES = TC_TILE * TC_D * 2;                 // 32 KiB per K (or V) tile

// Shared-memory sizes of an instantiation.  Decode keeps 16 columns at either wgmma width (its Q box is 16 heads wide).
template <bool VERIFY, int NP>
struct Shape {
    static constexpr int COLS = VERIFY ? NP : TC_NPAD;         // columns of the Q and P^T buffers and of the reduction scratch
    static constexpr int Q_BYTES = 2 * COLS * 128;             // [d half][COLS rows][128 B]
    static constexpr int P_BYTES = 2 * COLS * 128;             // [token half][COLS rows][128 B]
    static constexpr int SMEM_BYTES = (TC_KSTAGES + TC_VSTAGES) * TC_K_BYTES + 2 * Q_BYTES + P_BYTES + 2048;
};

struct Barriers {       // all mbarriers of the CTA (shared memory)
    uint64_t k_full[TC_KSTAGES], k_empty[TC_KSTAGES];
    uint64_t v_full[TC_VSTAGES], v_empty[TC_VSTAGES];
    uint64_t q_full[2], q_empty[2];
};

template <bool VERIFY> using Params = std::conditional_t<VERIFY, TcVerifyParams, TcParams>;

// qrow: first row of q and o of the item (decode: the sequence); rows / prefix: verify only
struct Item { int seq, kvh, split, split_start, split_len, ntiles, qrow, rows, prefix; };

template <bool VERIFY>
__device__ __forceinline__ bool get_item(const Params<VERIFY>& p, int idx, Item& it) {
    it.split = idx % p.num_splits;
    it.kvh = (idx / p.num_splits) % p.nkv;
    it.seq = idx / (p.num_splits * p.nkv);
    // every caller is a converged warp: broadcasting the loaded values makes them (and everything derived from them)
    // provably warp-uniform for the compiler
    int len;
    if constexpr (VERIFY) {
        it.rows = __shfl_sync(0xffffffffu, p.row_counts[it.seq], 0);
        it.prefix = __shfl_sync(0xffffffffu, p.prefix_lens[it.seq], 0);
        it.qrow = __shfl_sync(0xffffffffu, p.start_locs[it.seq], 0);
        len = it.prefix + it.rows;                         // the last row sees every stored position
    } else {
        it.qrow = it.seq;
        len = __shfl_sync(0xffffffffu, p.seq_lens[it.seq], 0);
    }
    it.split_start = it.split * p.split_tokens;
    if ((VERIFY && it.rows <= 0) || it.split_start >= len) return false;
    it.split_len = min(p.split_tokens, len - it.split_start);
    it.ntiles = (it.split_len + TC_TILE - 1) / TC_TILE;
    return true;
}

template <typename T, int NP, int TA>      // TA = 1: the A operand is MN-major (V)
__device__ __forceinline__ void wgmma_ss(float (&d)[NP / 2], uint64_t a, uint64_t b, uint32_t scale_d) {
    if constexpr (NP == 8) wgmma_m64n8k16_ss<T, TA, 0>(d, a, b, scale_d);
    else if constexpr (NP == 16) wgmma_m64n16k16_ss<T, TA, 0>(d, a, b, scale_d);
    else wgmma_m64n32k16_ss<T, TA, 0>(d, a, b, scale_d);
}

// One producer warp streams either the K or the V tiles (plus Q when IS_K): 32 block-table entries are fetched per
// 4 tiles (prefetched one group ahead), lanes 0..7 each issue the TMA of one page.
template <bool VERIFY, int NP, bool IS_K>
__device__ __forceinline__ void producer_loop(const Params<VERIFY>& p, const CUtensorMap* map, const CUtensorMap* qmap, uint8_t* ring,
                                              uint64_t* full, uint64_t* empty, int nstages, Barriers* bars, uint8_t* q_sm, int g, int lane) {
    constexpr int QB = Shape<VERIFY, NP>::Q_BYTES;
    uint32_t t = 0, n = 0;
    for (int idx = blockIdx.x; idx < p.num_items; idx += gridDim.x) {
        Item it;
        if (!get_item<VERIFY>(p, idx, it)) continue;
        if (IS_K) {       // Q of this item, 128 d as two 64-wide boxes over q viewed as (128 d | nq heads | rows).  Decode: heads
                          // [kvh*g, +16) of row seq, heads past nq zero-filled by the TMA unit; verify: heads [kvh*g, +g) of rows
                          // [start, +qrows)
            const int qb = n & 1;
            if (lane == 0) {
                mbar_wait(smem_u32(&bars->q_empty[qb]), ((n >> 1) & 1) ^ 1);
                const uint32_t qbar = smem_u32(&bars->q_full[qb]);
                if constexpr (VERIFY) mbar_arrive_expect_tx(qbar, (uint32_t)(256 * g * p.qrows));
                else mbar_arrive_expect_tx(qbar, QB);
                tma_load_3d(smem_u32(q_sm + qb * QB), qmap, qbar, 0, it.kvh * g, it.qrow);
                tma_load_3d(smem_u32(q_sm + qb * QB + QB / 2), qmap, qbar, 64, it.kvh * g, it.qrow);
            }
        }
        const int first_page = it.split_start / TC_BS;
        const int npages = (it.split_len + TC_BS - 1) / TC_BS;
        const int32_t* bt = p.block_table + (int64_t)p.seq_ids[it.seq] * p.max_blocks_per_seq + first_page;
        int next_blk = lane < npages ? bt[lane] : 0;                       // group 0
        for (int tile0 = 0; tile0 < it.ntiles; tile0 += 4) {
            const int my_blk = next_blk;
            const int npg = (tile0 + 4) * 8 + lane;                        // prefetch the next group's entries
            next_blk = (tile0 + 4 < it.ntiles && npg < npages) ? bt[npg] : 0;
            const int nt = min(4, it.ntiles - tile0);
            for (int j = 0; j < nt; j++, t++) {
                const int stage = t % nstages;
                const int valid = min(8, npages - (tile0 + j) * 8);
                const uint32_t bar = smem_u32(&full[stage]);
                if (lane == 0) {
                    mbar_wait(smem_u32(&empty[stage]), ((t / nstages) & 1) ^ 1);
                    mbar_arrive_expect_tx(bar, (uint32_t)valid * TC_BS * TC_D * 2);
                }
                __syncwarp();
                const int blk = __shfl_sync(0xffffffffu, my_blk, j * 8 + (lane & 7));
                if (lane < valid) {
                    // row of the cache viewed as [num_blocks*L*nkv*16 rows, 128]: first token row of this page
                    const int64_t row = (((int64_t)blk * p.num_layers + p.cur_layer) * p.nkv + it.kvh) * TC_BS;
                    const uint32_t dst = smem_u32(ring + stage * TC_K_BYTES) + lane * p.page_stride;
                    if (p.tma_4d) {
                        tma_load_4d(dst, map, bar, 0, 0, 0, (int)(row >> 3));
                    } else {
                        tma_load_2d(dst, map, bar, 0, (int)row);
                        tma_load_2d(dst + p.half_stride, map, bar, 64, (int)row);
                    }
                }
            }
        }
        n++;
    }
}

// The whole CTA of both kernels.  NP = wgmma N: the GQA group padded to 8 or 16 (decode), g * qrows padded to 8, 16 or 32 (VERIFY).
template <typename T, int NP, bool VERIFY>
__device__ __forceinline__ void paged_attn_pipeline(const CUtensorMap* kmap, const CUtensorMap* vmap, const CUtensorMap* qmap,
                                                    const Params<VERIFY>& p) {
    using S = Shape<VERIFY, NP>;
    constexpr int NR = NP / 2;                 // accumulator registers per m64 block
    constexpr int NH = NP / 4;                 // columns owned by one thread
    constexpr int QB = S::Q_BYTES, HALF = S::COLS * 128, NC = S::COLS;
    constexpr int RING_BYTES = (TC_KSTAGES + TC_VSTAGES) * TC_K_BYTES;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* k_sm = smem;                                            // [KSTAGES][32 KiB]
    uint8_t* v_sm = smem + TC_KSTAGES * TC_K_BYTES;                  // [VSTAGES][32 KiB]
    uint8_t* q_sm = smem + RING_BYTES;                               // [2][QB]
    uint8_t* p_sm = q_sm + 2 * QB;                                   // [P_BYTES]
    uint8_t* misc = p_sm + S::P_BYTES;                               // barriers, reduction scratch
    Barriers* bars = reinterpret_cast<Barriers*>(misc);
    float* red = reinterpret_cast<float*>(misc + 256);               // [2 parity][4 warps][NC] maxima, [4 warps][NC] sums

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = p.nq / p.nkv;

    // ---- one-time setup
    {   // zero the V ring (and K): page slots that a short tail tile never loads must hold finite data (P = 0 there).  VERIFY
        // also zeroes the Q buffers: its box fills g * qrows columns and the rest of the NP are never loaded.
        uint4* z = reinterpret_cast<uint4*>(smem);
        for (int i = tid; i < (RING_BYTES + (VERIFY ? 2 * QB : 0)) / 16; i += TC_THREADS) z[i] = make_uint4(0, 0, 0, 0);
    }
    if (tid == 0) {
        for (int i = 0; i < TC_KSTAGES; i++) { mbar_init(smem_u32(&bars->k_full[i]), 1); mbar_init(smem_u32(&bars->k_empty[i]), 128); }
        for (int i = 0; i < TC_VSTAGES; i++) { mbar_init(smem_u32(&bars->v_full[i]), 1); mbar_init(smem_u32(&bars->v_empty[i]), 128); }
        for (int i = 0; i < 2; i++) { mbar_init(smem_u32(&bars->q_full[i]), 1); mbar_init(smem_u32(&bars->q_empty[i]), 128); }
        mbar_fence_init();
        tma_prefetch_desc(kmap); tma_prefetch_desc(vmap); tma_prefetch_desc(qmap);
    }
    fence_proxy_async();
    __syncthreads();

    if (warp == 4) {
        producer_loop<VERIFY, NP, true>(p, kmap, qmap, k_sm, bars->k_full, bars->k_empty, TC_KSTAGES, bars, q_sm, g, lane);
    } else if (warp == 5) {
        producer_loop<VERIFY, NP, false>(p, vmap, qmap, v_sm, bars->v_full, bars->v_empty, TC_VSTAGES, bars, q_sm, g, lane);
    } else {
        // =========================================================== MMA + softmax warpgroup (warps 0..3)
        // Thread (warp w, lane l) owns token rows / d rows r = 16 w + l / 4 + 8 hi + 64 mb (hi, mb in {0, 1}) and the columns
        // hc(c) = 2 (l % 4) + (c & 1) + 8 (c >> 1), c < NH, of the S^T and O^T tiles.  Decode: column hc is head hc of the group;
        // VERIFY: column hc is (row hc / g, head hc % g).
        const uint64_t dk0 = make_smem_desc(smem_u32(k_sm), 16, p.k_sbo);
        const uint64_t dq0 = make_smem_desc(smem_u32(q_sm), 16, 1024);
        const uint64_t dv0 = make_smem_desc(smem_u32(v_sm), p.v_lbo, p.v_sbo);
        const uint64_t dp0 = make_smem_desc(smem_u32(p_sm), 16, 1024);
        const int r0 = 16 * warp + (lane >> 2);
        int hc[NH], crow[NH];
#pragma unroll
        for (int c = 0; c < NH; c++) { hc[c] = 2 * (lane & 3) + (c & 1) + 8 * (c >> 1); crow[c] = VERIFY ? hc[c] / g : 0; }
        uint32_t t = 0, n = 0;
        T* const out = reinterpret_cast<T*>(p.o);
        for (int idx = blockIdx.x; idx < p.num_items; idx += gridDim.x) {
            Item it;
            if (!get_item<VERIFY>(p, idx, it)) continue;
            if constexpr (VERIFY) {
                if (p.num_splits > 1 && it.kvh == 0 && it.split == 0 && tid < it.rows)
                    p.row_lens[it.qrow + tid] = it.prefix + tid + 1;      // visible length of each row: the merge's seq_lens
            }
            // tokens of this split that column c may see: [0, lim).  Decode: the whole split.  VERIFY: <= 0 for a column whose row
            // sees none of the split; columns of rows past the entry's count (not live) see the whole split (finite values) and
            // are never written.
            int lim[NH];
            bool live[NH];
#pragma unroll
            for (int c = 0; c < NH; c++) {
                if constexpr (VERIFY) {
                    live[c] = hc[c] < g * p.qrows && crow[c] < it.rows;
                    lim[c] = live[c] ? min(it.split_len, it.prefix + crow[c] + 1 - it.split_start) : it.split_len;
                } else {
                    lim[c] = it.split_len;
                }
            }
            const int qb = n & 1;
            mbar_wait(smem_u32(&bars->q_full[qb]), (n >> 1) & 1);
            float m_run[NH], m_use[NH], l_part[NH];
            float acc[2][NR];
#pragma unroll
            for (int c = 0; c < NH; c++) { m_run[c] = -INFINITY; l_part[c] = 0.f; }
#pragma unroll
            for (int mb = 0; mb < 2; mb++)
#pragma unroll
                for (int e = 0; e < NR; e++) acc[mb][e] = 0.f;

            for (int j = 0; j < it.ntiles; j++, t++) {
                // ---- S^T = K . Q^T
                const int ks_ = t % TC_KSTAGES;
                mbar_wait(smem_u32(&bars->k_full[ks_]), (t / TC_KSTAGES) & 1);
                float s[2][NR];
                {
                    const uint64_t kd = dk0 + (uint64_t)((ks_ * TC_K_BYTES) >> 4);
                    const uint64_t qd = dq0 + (uint64_t)((qb * QB) >> 4);
                    wgmma_fence();
#pragma unroll
                    for (int mb = 0; mb < 2; mb++)
#pragma unroll
                        for (int kk = 0; kk < 8; kk++) {     // 16 d per wgmma; d-half = kk / 4
                            const uint64_t a = kd + (uint64_t)((mb * 8 * p.k_sbo + (kk >> 2) * p.half_stride + (kk & 3) * 32) >> 4);
                            const uint64_t b = qd + (uint64_t)(((kk >> 2) * HALF + (kk & 3) * 32) >> 4);
                            wgmma_ss<T, NP, 0>(s[mb], a, b, kk > 0);
                        }
                    wgmma_commit();
                    wgmma_wait<0>();
                }
                mbar_arrive(smem_u32(&bars->k_empty[ks_]));                            // K tile consumed
                if (j == it.ntiles - 1) mbar_arrive(smem_u32(&bars->q_empty[qb]));     // Q buffer reusable

                // ---- scale + mask (tail of the split, causal limit of the column), tile max per column across the 128 token rows
                float mx[NH];
#pragma unroll
                for (int c = 0; c < NH; c++) mx[c] = -INFINITY;
#pragma unroll
                for (int mb = 0; mb < 2; mb++)
#pragma unroll
                    for (int e = 0; e < NR; e++) {
                        const int tok = j * TC_TILE + mb * 64 + r0 + 8 * ((e >> 1) & 1);
                        const int c = (e & 1) + 2 * (e >> 2);
                        s[mb][e] = tok < lim[c] ? s[mb][e] * p.scale_log2e : -INFINITY;
                        mx[c] = fmaxf(mx[c], s[mb][e]);
                    }
                float* rp = red + (t & 1) * 4 * NC;
#pragma unroll
                for (int c = 0; c < NH; c++) {
#pragma unroll
                    for (int o = 4; o < 32; o <<= 1) mx[c] = fmaxf(mx[c], __shfl_xor_sync(0xffffffffu, mx[c], o));
                    if (lane < 4) rp[warp * NC + hc[c]] = mx[c];
                }
                named_bar_sync(1, 128);
                float alpha[NH];
#pragma unroll
                for (int c = 0; c < NH; c++) {
                    const int h = hc[c];
                    const float mt = fmaxf(fmaxf(rp[h], rp[NC + h]), fmaxf(rp[2 * NC + h], rp[3 * NC + h]));
                    const float mn = fmaxf(m_run[c], mt);                  // decode: finite, every tile has a valid token
                    // a VERIFY column with no visible token yet keeps max -inf: exponentiate against 0 instead, so its p and
                    // alpha are exactly 0 (never -inf - -inf = NaN); every other column is untouched by it
                    m_use[c] = VERIFY && mn == -INFINITY ? 0.f : mn;
                    alpha[c] = fast_exp2_tc(m_run[c] - m_use[c]);
                    l_part[c] *= alpha[c];
                    m_run[c] = mn;
                }
                // p = exp2(s - m) -> P^T tile (B operand of the PV wgmma): [token half][NC column rows][128 B], SWIZZLE_128B.
                // The previous PV wgmma that read the buffer completed (wgmma_wait) before any thread got here.
#pragma unroll
                for (int mb = 0; mb < 2; mb++)
#pragma unroll
                    for (int e = 0; e < NR; e++) {
                        const int row = mb * 64 + r0 + 8 * ((e >> 1) & 1);
                        const int c = (e & 1) + 2 * (e >> 2);
                        const float pv = fast_exp2_tc(s[mb][e] - m_use[c]);
                        l_part[c] += pv;
                        const int h = hc[c];
                        *reinterpret_cast<T*>(p_sm + mb * HALF + h * 128 + ((((row & 63) >> 3) ^ (h & 7)) << 4) + (row & 7) * 2) =
                            Traits<T>::from_f(pv);
                    }
                fence_proxy_async();
                named_bar_sync(1, 128);

                // ---- O^T = alpha * O^T + V^T . P^T
#pragma unroll
                for (int mb = 0; mb < 2; mb++)
#pragma unroll
                    for (int e = 0; e < NR; e++) acc[mb][e] *= alpha[(e & 1) + 2 * (e >> 2)];
                const int vs = t % TC_VSTAGES;
                mbar_wait(smem_u32(&bars->v_full[vs]), (t / TC_VSTAGES) & 1);
                {
                    const uint64_t vd = dv0 + (uint64_t)((vs * TC_K_BYTES) >> 4);
                    wgmma_fence();
#pragma unroll
                    for (int mb = 0; mb < 2; mb++)
#pragma unroll
                        for (int kt = 0; kt < 8; kt++) {     // 16 tokens (one page) per wgmma
                            const uint64_t a = vd + (uint64_t)((mb * p.half_stride + kt * p.page_stride) >> 4);
                            const uint64_t b = dp0 + (uint64_t)(((kt >> 2) * HALF + (kt & 3) * 32) >> 4);
                            wgmma_ss<T, NP, 1>(acc[mb], a, b, 1);
                        }
                    wgmma_commit();
                    wgmma_wait<0>();
                }
                mbar_arrive(smem_u32(&bars->v_empty[vs]));
            }
            n++;

            // ---- finalise the item: l = sum over the 128 token rows, out = acc / l for live columns that saw a token
            float* rp = red + 8 * NC;
#pragma unroll
            for (int c = 0; c < NH; c++) {
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) l_part[c] += __shfl_xor_sync(0xffffffffu, l_part[c], o);
                if (lane < 4) rp[warp * NC + hc[c]] = l_part[c];
            }
            named_bar_sync(1, 128);
            float L[NH];
#pragma unroll
            for (int c = 0; c < NH; c++) {
                const int h = hc[c];
                L[c] = (rp[h] + rp[NC + h]) + (rp[2 * NC + h] + rp[3 * NC + h]);
            }
            named_bar_sync(1, 128);          // rp is rewritten by the next item
#pragma unroll
            for (int mb = 0; mb < 2; mb++)
#pragma unroll
                for (int e = 0; e < NR; e++) {
                    const int c = (e & 1) + 2 * (e >> 2);
                    // decode writes the heads of the group (the padding columns hold neighbouring heads)
                    if (VERIFY ? live[c] && lim[c] > 0 : hc[c] < g) {
                        const int d = mb * 64 + r0 + 8 * ((e >> 1) & 1);
                        const float val = acc[mb][e] / L[c];
                        const int head = it.kvh * g + (hc[c] - crow[c] * g);
                        const int64_t row = it.qrow + crow[c];
                        if (p.num_splits == 1) {
                            out[(row * p.nq + head) * TC_D + d] = Traits<T>::from_f(val);
                        } else {
                            const int64_t pi = (row * p.nq + head) * p.num_splits + it.split;
                            p.part_o[pi * TC_D + d] = val;
                            if (d == 0) p.part_lse[pi] = log2f(L[c]) + m_run[c];
                        }
                    }
                }
        }
    }
}

template <typename T, int NP>
__global__ void __launch_bounds__(TC_THREADS, 1) paged_attn_tc_kernel(const __grid_constant__ CUtensorMap kmap,
                                                                      const __grid_constant__ CUtensorMap vmap,
                                                                      const __grid_constant__ CUtensorMap qmap,
                                                                      const TcParams p) {
    paged_attn_pipeline<T, NP, false>(&kmap, &vmap, &qmap, p);
}

template <typename T, int NP>
__global__ void __launch_bounds__(TC_THREADS, 1) paged_attn_verify_kernel(const __grid_constant__ CUtensorMap kmap,
                                                                          const __grid_constant__ CUtensorMap vmap,
                                                                          const __grid_constant__ CUtensorMap qmap,
                                                                          const TcVerifyParams p) {
    paged_attn_pipeline<T, NP, true>(&kmap, &vmap, &qmap, p);
}

// ------------------------------------------------------------------ host side
namespace {

int g_kv_4d_ok = -1;            // -1 unknown, 0 the driver rejected the permuted-stride 4-D map, 1 usable (a property of the
                                // driver's tensor-map encoder, identical for every device of the process)

// SLLM_PAGED_ATTN_KV_MAP=2d: the [rows, 128] map even where the driver accepts the 4-D one, so the layout a driver without the
// 4-D map gets can be run and checked anywhere.  Read on every launch; the driver probe (g_kv_4d_ok) is left as it is.
bool kv_map_forced_2d() {
    const char* e = getenv("SLLM_PAGED_ATTN_KV_MAP");
    return e && strcmp(e, "2d") == 0;
}

// The K and V maps of a launch (cached by every argument: a cache tensor keeps its address, and both layouts of one cache can be
// cached at once) and, in `p`, the shared-memory layout their boxes produce: the 4-D page map (64 d | 8 tok | 2 halves |
// rows / 8) with one (64, 8, 2, 2) box per page where the driver accepts it, else the cache as [rows, 128] with two
// (64 d x 16 tokens) boxes per page.
bool kv_maps_and_layout(const TcLaunch& a, CUtensorMap* kmap, CUtensorMap* vmap, TcParams& p) {
    const uint64_t rows = (uint64_t)a.num_blocks * p.num_layers * p.nkv * TC_BS;
    bool ok_4d = false;
    if (!kv_map_forced_2d() && g_kv_4d_ok != 0) {
        const cuuint64_t dims[4] = {64, 8, 2, rows / 8}, strides[3] = {256, 128, 2048};
        const cuuint32_t box[4] = {64, 8, 2, 2};
        ok_4d = cached_tma_map(kmap, a.k_cache, a.dtype, 4, dims, strides, box) &&
                cached_tma_map(vmap, a.v_cache, a.dtype, 4, dims, strides, box);
        if (g_kv_4d_ok < 0) g_kv_4d_ok = ok_4d ? 1 : 0;
    }
    if (!ok_4d && !(cached_rows_map(kmap, a.k_cache, a.dtype, rows, TC_D, TC_D, TC_BS) &&
                    cached_rows_map(vmap, a.v_cache, a.dtype, rows, TC_D, TC_D, TC_BS)))
        return false;
    p.tma_4d = ok_4d;
    if (p.tma_4d) { p.page_stride = 4096; p.half_stride = 1024; p.k_sbo = 2048; p.v_lbo = 1024; p.v_sbo = 2048; }
    else          { p.page_stride = 2048; p.half_stride = 16384; p.k_sbo = 1024; p.v_lbo = 16384; p.v_sbo = 1024; }
    return true;
}

// q as (128 d | nq heads | num_tokens rows), rows q_row_stride elements apart, boxes of (64 d, box_heads, box_rows).  q is a
// transient activation (its address changes from call to call): encoded per launch (host-only, ~1 us), never cached.
bool encode_q_map(CUtensorMap* out, const TcLaunch& a, uint32_t box_heads, uint32_t box_rows) {
    const cuuint64_t dims[3] = {TC_D, (cuuint64_t)a.p.nq, (cuuint64_t)a.num_tokens};
    const cuuint64_t strides[2] = {TC_D * 2, (cuuint64_t)a.q_row_stride * 2};
    const cuuint32_t box[3] = {64, box_heads, box_rows};
    return encode_tma_map(out, a.q, a.dtype, 3, dims, strides, box);
}

}  // namespace

bool tc_paged_supported(int head_dim, int block_size, int nq, int nkv, int64_t num_blocks, int num_layers) {
    if (head_dim != TC_D || block_size != TC_BS) return false;
    if (nkv <= 0 || nq % nkv != 0 || nq / nkv > TC_NPAD) return false;
    if ((int64_t)num_blocks * num_layers * nkv * TC_BS >= (1LL << 31)) return false;     // TMA coordinates are int32
    return get_tensor_map_encoder() != nullptr;
}

// needs kmap, vmap, qmap, p, grid and a (the TcLaunch) in scope
#define SLLM_TC_LAUNCH(KERNEL, VERIFY, TT, NP)                                                                           \
    do {                                                                                                                 \
        constexpr int smem_bytes = Shape<VERIFY, NP>::SMEM_BYTES;                                                        \
        const char* what = VERIFY ? "paged_attention_verify(wgmma)" : "paged_attention(wgmma)";                         \
        if (int e = fit_dynamic_smem<KERNEL<TT, NP>>(smem_bytes, what)) return e;                                        \
        KERNEL<TT, NP><<<grid, TC_THREADS, smem_bytes, a.stream>>>(kmap, vmap, qmap, p);                                 \
    } while (0)

int launch_paged_tc(const TcLaunch& a) {
    TcParams p = a.p;
    const int g = p.nq / p.nkv;
    CUtensorMap kmap, vmap, qmap;
    SLLM_REQUIRE(kv_maps_and_layout(a, &kmap, &vmap, p), "paged_attention: cuTensorMapEncodeTiled failed for the KV cache");
    SLLM_REQUIRE(encode_q_map(&qmap, a, TC_NPAD, 1), "paged_attention: cuTensorMapEncodeTiled failed for q");
    p.num_items = a.num_seqs * p.nkv * p.num_splits;
    const int grid = p.num_items < a.num_sms ? p.num_items : a.num_sms;
    if (a.dtype == SLLM_F16) {
        if (g <= 8) SLLM_TC_LAUNCH(paged_attn_tc_kernel, false, __half, 8); else SLLM_TC_LAUNCH(paged_attn_tc_kernel, false, __half, 16);
    } else {
        if (g <= 8) SLLM_TC_LAUNCH(paged_attn_tc_kernel, false, __nv_bfloat16, 8);
        else SLLM_TC_LAUNCH(paged_attn_tc_kernel, false, __nv_bfloat16, 16);
    }
    return check_launch("paged_attention(wgmma)");
}

// The verify kernel serves head_dim 128, block_size 16 and at most 32 (row, head) columns per item.
bool tc_verify_supported(int head_dim, int block_size, int nq, int nkv, int max_rows, int64_t num_blocks, int num_layers,
                         int64_t num_tokens) {
    return tc_paged_supported(head_dim, block_size, nq, nkv, num_blocks, num_layers) && (nq / nkv) * max_rows <= 32 &&
           num_tokens < (1LL << 31);
}

int launch_paged_verify_tc(const TcLaunch& a) {
    TcVerifyParams p = a.p;
    const int g = p.nq / p.nkv;
    CUtensorMap kmap, vmap, qmap;
    SLLM_REQUIRE(kv_maps_and_layout(a, &kmap, &vmap, p), "paged_attention_verify: cuTensorMapEncodeTiled failed for the KV cache");
    SLLM_REQUIRE(encode_q_map(&qmap, a, g, p.qrows), "paged_attention_verify: cuTensorMapEncodeTiled failed for q");
    p.num_items = a.num_seqs * p.nkv * p.num_splits;
    const int grid = p.num_items < a.num_sms ? p.num_items : a.num_sms;
    const int cols = g * p.qrows;
    if (a.dtype == SLLM_F16) {
        if (cols <= 8) SLLM_TC_LAUNCH(paged_attn_verify_kernel, true, __half, 8);
        else if (cols <= 16) SLLM_TC_LAUNCH(paged_attn_verify_kernel, true, __half, 16);
        else SLLM_TC_LAUNCH(paged_attn_verify_kernel, true, __half, 32);
    } else {
        if (cols <= 8) SLLM_TC_LAUNCH(paged_attn_verify_kernel, true, __nv_bfloat16, 8);
        else if (cols <= 16) SLLM_TC_LAUNCH(paged_attn_verify_kernel, true, __nv_bfloat16, 16);
        else SLLM_TC_LAUNCH(paged_attn_verify_kernel, true, __nv_bfloat16, 32);
    }
    return check_launch("paged_attention_verify(wgmma)");
}
#undef SLLM_TC_LAUNCH

}  // namespace sllm

extern "C" int sllm_paged_attention_kv_map_rank(void) {
    if (sllm::kv_map_forced_2d()) return 2;
    return sllm::g_kv_4d_ok < 0 ? -1 : sllm::g_kv_4d_ok == 1 ? 4 : 2;
}
