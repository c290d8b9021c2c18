// Paged (decode) attention, generation 2: persistent, warp-specialised TMA + wgmma kernel (sm_90a).
//
// Reference being replaced: swiftllm/worker/kernels/paged_attn.py:9-108 (+ :111-149 via the merge kernel of
// paged_attn.cu when a sequence is split).  Shapes served: head_dim 128, block_size 16, GQA group <= 16, fp16/bf16.
//
// One persistent CTA per SM walks a static list of work items (sequence, kv head, split).  Per 128-token tile:
//   warp 4 (K) / warp 5 (V)  TMA producers: read 8 block-table entries, issue one 4-D tensor-map load per 16-token page
//                    (4 KiB, SWIZZLE_128B atoms [token-group][d-half][8 tok][64 d]) into 3-stage rings, completion on
//                    mbarriers; warp 4 also loads Q of the item (a 2-box TMA load).
//   warps 0-3        one warpgroup that issues the MMAs and runs the softmax, accumulators in registers:
//                    S^T[128 tok x NP heads] = K_tile (A, K-major) . Q^T (B, K-major)       (2 x 8 wgmma m64nNPk16)
//                    tile max per head across the warpgroup, p = exp2(s - m) -> bf16/fp16 P^T tile in shared memory,
//                    O^T[128 d x NP heads] = alpha * O^T + V_tile^T (A, MN-major) . P^T (B, K-major)   (2 x 8 wgmma)
// Tokens are the MMA M dimension (the transposed problem), so no tensor work is spent on padded query rows; the GQA
// group is the N dimension (padded to NP = 8 or 16 by reading neighbouring heads whose columns are never written back).
// HBM roofline: algorithmic bytes = sum_i len_i * nkv * 128 * 2 * sizeof(T) + 2 * Bd * nq * 128 * sizeof(T).
#include <mutex>
#include <unordered_map>

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
constexpr int TC_Q_BYTES = 2 * TC_NPAD * 128;                  // [half][16 rows][128 B] = 4 KiB
constexpr int TC_P_BYTES = 2 * TC_NPAD * 128;                  // [token half][16 rows][128 B] = 4 KiB
constexpr int TC_SMEM_BYTES = (TC_KSTAGES + TC_VSTAGES) * TC_K_BYTES + 2 * TC_Q_BYTES + TC_P_BYTES + 2048;

struct TcParams {
    const int32_t* block_table; const int32_t* seq_ids; const int32_t* seq_lens;
    void* o; float* part_o; float* part_lse;
    float scale_log2e;
    int split_tokens, num_splits, cur_layer, num_layers, nq, nkv, max_blocks_per_seq, num_seqs, num_items;
    // shared-memory placement of the 1 KiB atoms of a KV tile and the matching descriptor strides
    int page_stride, tg_stride, half_stride, k_sbo, v_lbo, v_sbo, tma_4d;
};

struct Barriers {       // all mbarriers of the CTA (shared memory)
    uint64_t k_full[TC_KSTAGES], k_empty[TC_KSTAGES];
    uint64_t v_full[TC_VSTAGES], v_empty[TC_VSTAGES];
    uint64_t q_full[2], q_empty[2];
};

struct Item { int seq, kvh, split, split_start, split_len, ntiles; };

__device__ __forceinline__ bool get_item(const TcParams& p, int idx, Item& it) {
    it.split = idx % p.num_splits;
    it.kvh = (idx / p.num_splits) % p.nkv;
    it.seq = idx / (p.num_splits * p.nkv);
    // every caller is a converged warp: broadcasting the loaded length makes it (and everything derived from it)
    // provably warp-uniform for the compiler
    const int len = __shfl_sync(0xffffffffu, p.seq_lens[it.seq], 0);
    it.split_start = it.split * p.split_tokens;
    if (it.split_start >= len) return false;
    it.split_len = min(p.split_tokens, len - it.split_start);
    it.ntiles = (it.split_len + TC_TILE - 1) / TC_TILE;
    return true;
}

// One producer warp streams either the K or the V tiles (plus Q when IS_K): 32 block-table entries are fetched per
// 4 tiles (prefetched one group ahead), lanes 0..7 each issue the TMA of one page.
template <bool IS_K>
__device__ __forceinline__ void producer_loop(const TcParams& p, const CUtensorMap* map, const CUtensorMap* qmap, uint8_t* ring,
                                              uint64_t* full, uint64_t* empty, int nstages, Barriers* bars, uint8_t* q_sm, int g, int lane) {
    uint32_t t = 0, n = 0;
    for (int idx = blockIdx.x; idx < p.num_items; idx += gridDim.x) {
        Item it;
        if (!get_item(p, idx, it)) continue;
        if (IS_K) {       // Q of this item: heads [kvh*g, +16) of sequence seq, 128 d as two 64-wide boxes
            const int qb = n & 1;
            if (lane == 0) {
                mbar_wait(smem_u32(&bars->q_empty[qb]), ((n >> 1) & 1) ^ 1);
                const uint32_t qbar = smem_u32(&bars->q_full[qb]);
                mbar_arrive_expect_tx(qbar, TC_Q_BYTES);
                // q viewed as (128 d | nq heads | Bd sequences): heads past nq are zero-filled by the TMA unit
                tma_load_3d(smem_u32(q_sm + qb * TC_Q_BYTES), qmap, qbar, 0, it.kvh * g, it.seq);
                tma_load_3d(smem_u32(q_sm + qb * TC_Q_BYTES + 2048), qmap, qbar, 64, it.kvh * g, it.seq);
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

template <typename T, int NP>      // NP = wgmma N: the GQA group padded to 8 or 16
__global__ void __launch_bounds__(TC_THREADS, 1) paged_attn_tc_kernel(const __grid_constant__ CUtensorMap kmap,
                                                                      const __grid_constant__ CUtensorMap vmap,
                                                                      const __grid_constant__ CUtensorMap qmap,
                                                                      const TcParams p) {
    constexpr int NR = NP / 2;                 // accumulator registers per m64 block
    constexpr int NH = NP / 4;                 // head columns owned by one thread
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* k_sm = smem;                                            // [KSTAGES][32 KiB]
    uint8_t* v_sm = smem + TC_KSTAGES * TC_K_BYTES;                  // [VSTAGES][32 KiB]
    uint8_t* q_sm = v_sm + TC_VSTAGES * TC_K_BYTES;                  // [2][4 KiB]
    uint8_t* p_sm = q_sm + 2 * TC_Q_BYTES;                           // [4 KiB]
    uint8_t* misc = p_sm + TC_P_BYTES;                               // barriers, reduction scratch
    Barriers* bars = reinterpret_cast<Barriers*>(misc);
    float* red = reinterpret_cast<float*>(misc + 256);               // [2 parity][4 warps][16] maxima, [4 warps][16] sums

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = p.nq / p.nkv;

    // ---- one-time setup
    {   // zero the V ring (and K): page slots that a short tail tile never loads must hold finite data (P = 0 there)
        uint4* z = reinterpret_cast<uint4*>(smem);
        for (int i = tid; i < (TC_KSTAGES + TC_VSTAGES) * TC_K_BYTES / 16; i += TC_THREADS) z[i] = make_uint4(0, 0, 0, 0);
    }
    if (tid == 0) {
        for (int i = 0; i < TC_KSTAGES; i++) { mbar_init(smem_u32(&bars->k_full[i]), 1); mbar_init(smem_u32(&bars->k_empty[i]), 128); }
        for (int i = 0; i < TC_VSTAGES; i++) { mbar_init(smem_u32(&bars->v_full[i]), 1); mbar_init(smem_u32(&bars->v_empty[i]), 128); }
        for (int i = 0; i < 2; i++) { mbar_init(smem_u32(&bars->q_full[i]), 1); mbar_init(smem_u32(&bars->q_empty[i]), 128); }
        mbar_fence_init();
        tma_prefetch_desc(&kmap); tma_prefetch_desc(&vmap); tma_prefetch_desc(&qmap);
    }
    fence_proxy_async();
    __syncthreads();

    if (warp == 4) {
        producer_loop<true>(p, &kmap, &qmap, k_sm, bars->k_full, bars->k_empty, TC_KSTAGES, bars, q_sm, g, lane);
    } else if (warp == 5) {
        producer_loop<false>(p, &vmap, &qmap, v_sm, bars->v_full, bars->v_empty, TC_VSTAGES, bars, q_sm, g, lane);
    } else {
        // =========================================================== MMA + softmax warpgroup (warps 0..3)
        // Thread (warp w, lane l) owns token rows / d rows r = 16 w + l / 4 + 8 hi + 64 mb (hi, mb in {0, 1}) and the head
        // columns hc(c) = 2 (l % 4) + (c & 1) + 8 (c >> 1), c < NH, of the S^T and O^T tiles.
        const uint64_t dk0 = make_smem_desc(smem_u32(k_sm), 16, p.k_sbo);
        const uint64_t dq0 = make_smem_desc(smem_u32(q_sm), 16, 1024);
        const uint64_t dv0 = make_smem_desc(smem_u32(v_sm), p.v_lbo, p.v_sbo);
        const uint64_t dp0 = make_smem_desc(smem_u32(p_sm), 16, 1024);
        const int r0 = 16 * warp + (lane >> 2);
        int hc[NH];
#pragma unroll
        for (int c = 0; c < NH; c++) hc[c] = 2 * (lane & 3) + (c & 1) + 8 * (c >> 1);
        uint32_t t = 0, n = 0;
        T* const out = reinterpret_cast<T*>(p.o);
        for (int idx = blockIdx.x; idx < p.num_items; idx += gridDim.x) {
            Item it;
            if (!get_item(p, idx, it)) continue;
            const int qb = n & 1;
            mbar_wait(smem_u32(&bars->q_full[qb]), (n >> 1) & 1);
            float m_run[NH], l_part[NH];
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
                    const uint64_t qd = dq0 + (uint64_t)((qb * TC_Q_BYTES) >> 4);
                    wgmma_fence();
#pragma unroll
                    for (int mb = 0; mb < 2; mb++)
#pragma unroll
                        for (int kk = 0; kk < 8; kk++) {     // 16 d per wgmma; d-half = kk / 4
                            const uint64_t a = kd + (uint64_t)((mb * 8 * p.k_sbo + (kk >> 2) * p.half_stride + (kk & 3) * 32) >> 4);
                            const uint64_t b = qd + (uint64_t)(((kk >> 2) * 2048 + (kk & 3) * 32) >> 4);
                            if constexpr (NP == 8) wgmma_m64n8k16_ss<T, 0, 0>(s[mb], a, b, kk > 0);
                            else wgmma_m64n16k16_ss<T, 0, 0>(s[mb], a, b, kk > 0);
                        }
                    wgmma_commit();
                    wgmma_wait<0>();
                }
                mbar_arrive(smem_u32(&bars->k_empty[ks_]));                            // K tile consumed
                if (j == it.ntiles - 1) mbar_arrive(smem_u32(&bars->q_empty[qb]));     // Q buffer reusable

                // ---- scale + tail mask, tile max per head across the 128 token rows
                float mx[NH];
#pragma unroll
                for (int c = 0; c < NH; c++) mx[c] = -INFINITY;
#pragma unroll
                for (int mb = 0; mb < 2; mb++)
#pragma unroll
                    for (int e = 0; e < NR; e++) {
                        const int tok = j * TC_TILE + mb * 64 + r0 + 8 * ((e >> 1) & 1);
                        const int c = (e & 1) + 2 * (e >> 2);
                        s[mb][e] = tok < it.split_len ? s[mb][e] * p.scale_log2e : -INFINITY;
                        mx[c] = fmaxf(mx[c], s[mb][e]);
                    }
                float* rp = red + (t & 1) * 64;
#pragma unroll
                for (int c = 0; c < NH; c++) {
#pragma unroll
                    for (int o = 4; o < 32; o <<= 1) mx[c] = fmaxf(mx[c], __shfl_xor_sync(0xffffffffu, mx[c], o));
                    if (lane < 4) rp[warp * 16 + hc[c]] = mx[c];
                }
                named_bar_sync(1, 128);
                float alpha[NH];
#pragma unroll
                for (int c = 0; c < NH; c++) {
                    const int h = hc[c];
                    const float mt = fmaxf(fmaxf(rp[h], rp[16 + h]), fmaxf(rp[32 + h], rp[48 + h]));
                    const float mn = fmaxf(m_run[c], mt);                  // finite: every tile has a valid token
                    alpha[c] = fast_exp2_tc(m_run[c] - mn);
                    l_part[c] *= alpha[c];
                    m_run[c] = mn;
                }
                // p = exp2(s - m) -> P^T tile (B operand of the PV wgmma): [token half][16 head rows][128 B], SWIZZLE_128B.
                // The previous PV wgmma that read the buffer completed (wgmma_wait) before any thread got here.
#pragma unroll
                for (int mb = 0; mb < 2; mb++)
#pragma unroll
                    for (int e = 0; e < NR; e++) {
                        const int row = mb * 64 + r0 + 8 * ((e >> 1) & 1);
                        const int c = (e & 1) + 2 * (e >> 2);
                        const float pv = fast_exp2_tc(s[mb][e] - m_run[c]);
                        l_part[c] += pv;
                        const int h = hc[c];
                        *reinterpret_cast<T*>(p_sm + mb * 2048 + h * 128 + ((((row & 63) >> 3) ^ (h & 7)) << 4) + (row & 7) * 2) =
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
                            const uint64_t b = dp0 + (uint64_t)(((kt >> 2) * 2048 + (kt & 3) * 32) >> 4);
                            if constexpr (NP == 8) wgmma_m64n8k16_ss<T, 1, 0>(acc[mb], a, b, 1);
                            else wgmma_m64n16k16_ss<T, 1, 0>(acc[mb], a, b, 1);
                        }
                    wgmma_commit();
                    wgmma_wait<0>();
                }
                mbar_arrive(smem_u32(&bars->v_empty[vs]));
            }
            n++;

            // ---- finalise the item: l = sum over the 128 token rows, out[h][d] = acc / l
            float* rp = red + 128;
#pragma unroll
            for (int c = 0; c < NH; c++) {
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) l_part[c] += __shfl_xor_sync(0xffffffffu, l_part[c], o);
                if (lane < 4) rp[warp * 16 + hc[c]] = l_part[c];
            }
            named_bar_sync(1, 128);
            float L[NH];
#pragma unroll
            for (int c = 0; c < NH; c++) {
                const int h = hc[c];
                L[c] = (rp[h] + rp[16 + h]) + (rp[32 + h] + rp[48 + h]);
            }
            named_bar_sync(1, 128);          // rp is rewritten by the next item
#pragma unroll
            for (int mb = 0; mb < 2; mb++)
#pragma unroll
                for (int e = 0; e < NR; e++) {
                    const int c = (e & 1) + 2 * (e >> 2);
                    const int h = hc[c];
                    if (h < g) {
                        const int d = mb * 64 + r0 + 8 * ((e >> 1) & 1);
                        const float val = acc[mb][e] / L[c];
                        const int head = it.kvh * g + h;
                        if (p.num_splits == 1) {
                            out[((int64_t)it.seq * p.nq + head) * TC_D + d] = Traits<T>::from_f(val);
                        } else {
                            const int64_t pi = ((int64_t)it.seq * p.nq + head) * p.num_splits + it.split;
                            p.part_o[pi * TC_D + d] = val;
                            if (d == 0) p.part_lse[pi] = log2f(L[c]) + m_run[c];
                        }
                    }
                }
        }
    }
}

// ====================================================================================================================
// Speculative verification (sllm_paged_attention_verify): entry i holds rows j < rows_i (query tokens at positions
// prefix_i + j); row j attends causally to positions [0, prefix_i + j].  Same pipeline as paged_attn_tc_kernel, but the wgmma N
// dimension holds (row j, head h) pairs as column j * g + h, so each (entry, kv head, split) item streams its K/V pages once for
// every row and head of the entry.  Q is one TMA box (64 d, g heads, qrows rows) per d-half over the row-strided packed q:
// columns of rows past the entry's count hold whatever the box read (the next entry's rows, or zero fill) and are never written.
struct TcVerifyParams {
    const int32_t* block_table; const int32_t* seq_ids; const int32_t* start_locs; const int32_t* row_counts;
    const int32_t* prefix_lens;
    void* o; float* part_o; float* part_lse; int32_t* row_lens;
    float scale_log2e;
    int split_tokens, num_splits, cur_layer, num_layers, nq, nkv, max_blocks_per_seq, num_items, qrows;
    int page_stride, half_stride, k_sbo, v_lbo, v_sbo, tma_4d;
};

struct VerifyItem { int seq, kvh, split, split_start, split_len, ntiles, start, rows, prefix; };

__device__ __forceinline__ bool get_verify_item(const TcVerifyParams& p, int idx, VerifyItem& it) {
    it.split = idx % p.num_splits;
    it.kvh = (idx / p.num_splits) % p.nkv;
    it.seq = idx / (p.num_splits * p.nkv);
    // converged warps only: the broadcasts make the item provably warp-uniform
    it.rows = __shfl_sync(0xffffffffu, p.row_counts[it.seq], 0);
    it.prefix = __shfl_sync(0xffffffffu, p.prefix_lens[it.seq], 0);
    it.start = __shfl_sync(0xffffffffu, p.start_locs[it.seq], 0);
    const int len = it.prefix + it.rows;                   // the last row sees every stored position
    it.split_start = it.split * p.split_tokens;
    if (it.rows <= 0 || it.split_start >= len) return false;
    it.split_len = min(p.split_tokens, len - it.split_start);
    it.ntiles = (it.split_len + TC_TILE - 1) / TC_TILE;
    return true;
}

template <bool IS_K>
__device__ __forceinline__ void verify_producer_loop(const TcVerifyParams& p, const CUtensorMap* map, const CUtensorMap* qmap,
                                                     uint8_t* ring, uint64_t* full, uint64_t* empty, int nstages, Barriers* bars,
                                                     uint8_t* q_sm, int q_bytes, int g, int lane) {
    uint32_t t = 0, n = 0;
    for (int idx = blockIdx.x; idx < p.num_items; idx += gridDim.x) {
        VerifyItem it;
        if (!get_verify_item(p, idx, it)) continue;
        if (IS_K) {       // Q of this item: heads [kvh*g, +g) of rows [start, +qrows), 128 d as two 64-wide boxes
            const int qb = n & 1;
            if (lane == 0) {
                mbar_wait(smem_u32(&bars->q_empty[qb]), ((n >> 1) & 1) ^ 1);
                const uint32_t qbar = smem_u32(&bars->q_full[qb]);
                mbar_arrive_expect_tx(qbar, (uint32_t)(256 * g * p.qrows));
                tma_load_3d(smem_u32(q_sm + qb * q_bytes), qmap, qbar, 0, it.kvh * g, it.start);
                tma_load_3d(smem_u32(q_sm + qb * q_bytes + q_bytes / 2), qmap, qbar, 64, it.kvh * g, it.start);
            }
        }
        const int first_page = it.split_start / TC_BS;
        const int npages = (it.split_len + TC_BS - 1) / TC_BS;
        const int32_t* bt = p.block_table + (int64_t)p.seq_ids[it.seq] * p.max_blocks_per_seq + first_page;
        int next_blk = lane < npages ? bt[lane] : 0;
        for (int tile0 = 0; tile0 < it.ntiles; tile0 += 4) {
            const int my_blk = next_blk;
            const int npg = (tile0 + 4) * 8 + lane;
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

template <int NP>
struct VerifyShape {
    static constexpr int Q_BYTES = 2 * NP * 128;               // [d half][NP columns][128 B]
    static constexpr int P_BYTES = 2 * NP * 128;               // [token half][NP columns][128 B]
    static constexpr int SMEM_BYTES = (TC_KSTAGES + TC_VSTAGES) * TC_K_BYTES + 2 * Q_BYTES + P_BYTES + 2048;
};

template <typename T, int NP>
__device__ __forceinline__ void wgmma_verify(float (&d)[NP / 2], uint64_t a, uint64_t b, uint32_t scale_d, bool v_operand) {
    if (v_operand) {
        if constexpr (NP == 8) wgmma_m64n8k16_ss<T, 1, 0>(d, a, b, scale_d);
        else if constexpr (NP == 16) wgmma_m64n16k16_ss<T, 1, 0>(d, a, b, scale_d);
        else wgmma_m64n32k16_ss<T, 1, 0>(d, a, b, scale_d);
    } else {
        if constexpr (NP == 8) wgmma_m64n8k16_ss<T, 0, 0>(d, a, b, scale_d);
        else if constexpr (NP == 16) wgmma_m64n16k16_ss<T, 0, 0>(d, a, b, scale_d);
        else wgmma_m64n32k16_ss<T, 0, 0>(d, a, b, scale_d);
    }
}

template <typename T, int NP>      // NP = wgmma N: g * qrows padded to 8, 16 or 32
__global__ void __launch_bounds__(TC_THREADS, 1) paged_attn_verify_kernel(const __grid_constant__ CUtensorMap kmap,
                                                                          const __grid_constant__ CUtensorMap vmap,
                                                                          const __grid_constant__ CUtensorMap qmap,
                                                                          const TcVerifyParams p) {
    constexpr int NR = NP / 2;                 // accumulator registers per m64 block
    constexpr int NH = NP / 4;                 // columns owned by one thread
    constexpr int QB = VerifyShape<NP>::Q_BYTES, HALF = NP * 128;
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* k_sm = smem;
    uint8_t* v_sm = smem + TC_KSTAGES * TC_K_BYTES;
    uint8_t* q_sm = v_sm + TC_VSTAGES * TC_K_BYTES;                  // [2][QB]
    uint8_t* p_sm = q_sm + 2 * QB;                                   // [P_BYTES]
    uint8_t* misc = p_sm + VerifyShape<NP>::P_BYTES;
    Barriers* bars = reinterpret_cast<Barriers*>(misc);
    float* red = reinterpret_cast<float*>(misc + 256);               // [2 parity][4 warps][NP] maxima, [4 warps][NP] sums

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = p.nq / p.nkv;
    const int ncols = g * p.qrows;             // columns the Q box fills; the rest of the NP stay zero

    {   // zero the K/V rings (short tail tiles leave page slots unloaded) and the Q buffers (columns >= ncols are never loaded)
        uint4* z = reinterpret_cast<uint4*>(smem);
        for (int i = tid; i < ((TC_KSTAGES + TC_VSTAGES) * TC_K_BYTES + 2 * QB) / 16; i += TC_THREADS) z[i] = make_uint4(0, 0, 0, 0);
    }
    if (tid == 0) {
        for (int i = 0; i < TC_KSTAGES; i++) { mbar_init(smem_u32(&bars->k_full[i]), 1); mbar_init(smem_u32(&bars->k_empty[i]), 128); }
        for (int i = 0; i < TC_VSTAGES; i++) { mbar_init(smem_u32(&bars->v_full[i]), 1); mbar_init(smem_u32(&bars->v_empty[i]), 128); }
        for (int i = 0; i < 2; i++) { mbar_init(smem_u32(&bars->q_full[i]), 1); mbar_init(smem_u32(&bars->q_empty[i]), 128); }
        mbar_fence_init();
        tma_prefetch_desc(&kmap); tma_prefetch_desc(&vmap); tma_prefetch_desc(&qmap);
    }
    fence_proxy_async();
    __syncthreads();

    if (warp == 4) {
        verify_producer_loop<true>(p, &kmap, &qmap, k_sm, bars->k_full, bars->k_empty, TC_KSTAGES, bars, q_sm, QB, g, lane);
    } else if (warp == 5) {
        verify_producer_loop<false>(p, &vmap, &qmap, v_sm, bars->v_full, bars->v_empty, TC_VSTAGES, bars, q_sm, QB, g, lane);
    } else {
        // Thread (warp w, lane l) owns token rows / d rows r = 16 w + l / 4 + 8 hi + 64 mb and the columns
        // hc(c) = 2 (l % 4) + (c & 1) + 8 (c >> 1), c < NH, of the S^T and O^T tiles; column hc is (row hc / g, head hc % g).
        const uint64_t dk0 = make_smem_desc(smem_u32(k_sm), 16, p.k_sbo);
        const uint64_t dq0 = make_smem_desc(smem_u32(q_sm), 16, 1024);
        const uint64_t dv0 = make_smem_desc(smem_u32(v_sm), p.v_lbo, p.v_sbo);
        const uint64_t dp0 = make_smem_desc(smem_u32(p_sm), 16, 1024);
        const int r0 = 16 * warp + (lane >> 2);
        int hc[NH], crow[NH];
#pragma unroll
        for (int c = 0; c < NH; c++) { hc[c] = 2 * (lane & 3) + (c & 1) + 8 * (c >> 1); crow[c] = hc[c] / g; }
        uint32_t t = 0, n = 0;
        T* const out = reinterpret_cast<T*>(p.o);
        for (int idx = blockIdx.x; idx < p.num_items; idx += gridDim.x) {
            VerifyItem it;
            if (!get_verify_item(p, idx, it)) continue;
            if (p.num_splits > 1 && it.kvh == 0 && it.split == 0 && tid < it.rows)
                p.row_lens[it.start + tid] = it.prefix + tid + 1;     // visible length of each row: the merge's seq_lens
            // tokens of this split that column c may see: [0, lim); <= 0 for a column whose row sees none of the split.
            // Columns of rows past the entry's count see the whole split (finite values) and are never written.
            int lim[NH];
            bool live[NH];
#pragma unroll
            for (int c = 0; c < NH; c++) {
                live[c] = hc[c] < ncols && crow[c] < it.rows;
                lim[c] = live[c] ? min(it.split_len, it.prefix + crow[c] + 1 - it.split_start) : it.split_len;
            }
            const int qb = n & 1;
            mbar_wait(smem_u32(&bars->q_full[qb]), (n >> 1) & 1);
            float m_run[NH], m_use[NH], l_part[NH];
            float acc[2][NR];
#pragma unroll
            for (int c = 0; c < NH; c++) { m_run[c] = -INFINITY; m_use[c] = 0.f; l_part[c] = 0.f; }
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
                        for (int kk = 0; kk < 8; kk++) {
                            const uint64_t a = kd + (uint64_t)((mb * 8 * p.k_sbo + (kk >> 2) * p.half_stride + (kk & 3) * 32) >> 4);
                            const uint64_t b = qd + (uint64_t)(((kk >> 2) * HALF + (kk & 3) * 32) >> 4);
                            wgmma_verify<T, NP>(s[mb], a, b, kk > 0, false);
                        }
                    wgmma_commit();
                    wgmma_wait<0>();
                }
                mbar_arrive(smem_u32(&bars->k_empty[ks_]));
                if (j == it.ntiles - 1) mbar_arrive(smem_u32(&bars->q_empty[qb]));

                // ---- scale + causal mask per column, tile max per column across the warpgroup
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
                float* rp = red + (t & 1) * 4 * NP;
#pragma unroll
                for (int c = 0; c < NH; c++) {
#pragma unroll
                    for (int o = 4; o < 32; o <<= 1) mx[c] = fmaxf(mx[c], __shfl_xor_sync(0xffffffffu, mx[c], o));
                    if (lane < 4) rp[warp * NP + hc[c]] = mx[c];
                }
                named_bar_sync(1, 128);
                float alpha[NH];
#pragma unroll
                for (int c = 0; c < NH; c++) {
                    const int h = hc[c];
                    const float mt = fmaxf(fmaxf(rp[h], rp[NP + h]), fmaxf(rp[2 * NP + h], rp[3 * NP + h]));
                    const float mn = fmaxf(m_run[c], mt);
                    // a column with no visible token yet keeps max -inf: exponentiate against 0 instead, so its p and alpha
                    // are exactly 0 (never -inf - -inf = NaN); every other column is untouched by it
                    m_use[c] = mn == -INFINITY ? 0.f : mn;
                    alpha[c] = fast_exp2_tc(m_run[c] - m_use[c]);
                    l_part[c] *= alpha[c];
                    m_run[c] = mn;
                }
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
                        for (int kt = 0; kt < 8; kt++) {
                            const uint64_t a = vd + (uint64_t)((mb * p.half_stride + kt * p.page_stride) >> 4);
                            const uint64_t b = dp0 + (uint64_t)(((kt >> 2) * HALF + (kt & 3) * 32) >> 4);
                            wgmma_verify<T, NP>(acc[mb], a, b, 1, true);
                        }
                    wgmma_commit();
                    wgmma_wait<0>();
                }
                mbar_arrive(smem_u32(&bars->v_empty[vs]));
            }
            n++;

            // ---- finalise the item: l = sum over the token rows, out = acc / l for live columns that saw a token
            float* rp = red + 8 * NP;
#pragma unroll
            for (int c = 0; c < NH; c++) {
#pragma unroll
                for (int o = 4; o < 32; o <<= 1) l_part[c] += __shfl_xor_sync(0xffffffffu, l_part[c], o);
                if (lane < 4) rp[warp * NP + hc[c]] = l_part[c];
            }
            named_bar_sync(1, 128);
            float L[NH];
#pragma unroll
            for (int c = 0; c < NH; c++) {
                const int h = hc[c];
                L[c] = (rp[h] + rp[NP + h]) + (rp[2 * NP + h] + rp[3 * NP + h]);
            }
            named_bar_sync(1, 128);
#pragma unroll
            for (int mb = 0; mb < 2; mb++)
#pragma unroll
                for (int e = 0; e < NR; e++) {
                    const int c = (e & 1) + 2 * (e >> 2);
                    if (live[c] && lim[c] > 0) {
                        const int d = mb * 64 + r0 + 8 * ((e >> 1) & 1);
                        const float val = acc[mb][e] / L[c];
                        const int head = it.kvh * g + (hc[c] - crow[c] * g);
                        const int64_t row = it.start + crow[c];
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

}  // namespace sllm

namespace sllm {

// ------------------------------------------------------------------ host side
namespace {

struct MapKey {
    const void* ptr; uint64_t rows; int kind; uint64_t aux;
    bool operator==(const MapKey& o) const { return ptr == o.ptr && rows == o.rows && kind == o.kind && aux == o.aux; }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        return std::hash<const void*>()(k.ptr) ^ (std::hash<uint64_t>()(k.rows) * 1315423911u) ^ (size_t)k.kind ^ (std::hash<uint64_t>()(k.aux) << 1);
    }
};
std::mutex g_map_mutex;
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;
int g_kv_4d_ok = -1;            // -1 unknown, 0 the driver rejected the permuted-stride 4-D map, 1 usable (a property of the
                                // driver's tensor-map encoder, identical for every device of the process)

CUtensorMapDataType map_dtype(sllm_dtype_t dt) { return dt == SLLM_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16; }

// kind 0: 2-D [rows, 128] map with (64 x 16) boxes; kind 1: 4-D page map (64 d | 8 tok | 2 halves | rows/8), box (64,8,2,2);
// kind 2: q as (128 d | nq heads | rows sequences) with sequence stride aux>>16 elements and nq = aux & 0xffff, box (64,16,1)
bool encode_map(CUtensorMap* out, const void* ptr, uint64_t rows, int kind, sllm_dtype_t dt, uint64_t aux) {
    TensorMapEncodeFn enc = get_tensor_map_encoder();
    if (!enc) return false;
    CUresult r;
    if (kind == 0) {
        cuuint64_t dims[2] = {128, rows};
        cuuint64_t strides[1] = {256};
        cuuint32_t box[2] = {64, 16}, es[2] = {1, 1};
        r = enc(out, map_dtype(dt), 2, const_cast<void*>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    } else if (kind == 2) {
        cuuint64_t dims[3] = {128, aux & 0xffff, rows};
        cuuint64_t strides[2] = {256, (aux >> 16) * 2};
        cuuint32_t box[3] = {64, 16, 1}, es[3] = {1, 1, 1};
        r = enc(out, map_dtype(dt), 3, const_cast<void*>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    } else {
        cuuint64_t dims[4] = {64, 8, 2, rows / 8};
        cuuint64_t strides[3] = {256, 128, 2048};
        cuuint32_t box[4] = {64, 8, 2, 2}, es[4] = {1, 1, 1, 1};
        r = enc(out, map_dtype(dt), 4, const_cast<void*>(ptr), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    return r == CUDA_SUCCESS;
}

bool get_map(CUtensorMap* out, const void* ptr, uint64_t rows, int kind, sllm_dtype_t dt, bool cache, uint64_t aux = 0) {
    MapKey key{ptr, rows, kind * 2 + (int)dt, aux};
    if (cache) {
        std::lock_guard<std::mutex> lk(g_map_mutex);
        auto it = g_maps.find(key);
        if (it != g_maps.end()) { *out = it->second; return true; }
    }
    if (!encode_map(out, ptr, rows, kind, dt, aux)) return false;
    if (cache) {
        std::lock_guard<std::mutex> lk(g_map_mutex);
        if (g_maps.size() > 4096) g_maps.clear();
        g_maps[key] = *out;
    }
    return true;
}

}  // namespace

bool tc_paged_supported(int head_dim, int block_size, int nq, int nkv, int64_t num_blocks, int num_layers) {
    if (head_dim != TC_D || block_size != TC_BS) return false;
    if (nkv <= 0 || nq % nkv != 0 || nq / nkv > TC_NPAD) return false;
    if ((int64_t)num_blocks * num_layers * nkv * TC_BS >= (1LL << 31)) return false;     // TMA coordinates are int32
    return get_tensor_map_encoder() != nullptr;
}

// Launches the persistent kernel; returns 0 / error like the other entry points.  `split_tokens`/`num_splits` come from
// the shared planner in paged_attn.cu.
int launch_paged_tc(const void* q, const void* k_cache, const void* v_cache, const int32_t* block_table, const int32_t* seq_ids,
                    const int32_t* seq_lens, void* o, float* part_o, float* part_lse, float scale_log2e, int num_seqs,
                    int split_tokens, int num_splits, int cur_layer, int num_layers, int nq, int nkv, int max_blocks_per_seq,
                    int64_t num_blocks, int64_t q_row_stride, sllm_dtype_t dtype, int num_sms, cudaStream_t stream) {
    const uint64_t rows = (uint64_t)num_blocks * num_layers * nkv * TC_BS;
    CUtensorMap kmap, vmap, qmap;
    if (g_kv_4d_ok != 0) {
        bool ok = get_map(&kmap, k_cache, rows, 1, dtype, true) && get_map(&vmap, v_cache, rows, 1, dtype, true);
        if (g_kv_4d_ok < 0) g_kv_4d_ok = ok ? 1 : 0;
    }
    if (g_kv_4d_ok == 0) {
        SLLM_REQUIRE(get_map(&kmap, k_cache, rows, 0, dtype, true) && get_map(&vmap, v_cache, rows, 0, dtype, true),
                     "paged_attention: cuTensorMapEncodeTiled failed for the KV cache");
    }
    // q is a transient activation (its address changes from call to call): encoded per launch (host-only, ~1 us), never cached
    SLLM_REQUIRE(get_map(&qmap, q, (uint64_t)num_seqs, 2, dtype, false, ((uint64_t)q_row_stride << 16) | (uint64_t)nq),
                 "paged_attention: cuTensorMapEncodeTiled failed for q");

    TcParams p;
    p.block_table = block_table; p.seq_ids = seq_ids; p.seq_lens = seq_lens; p.o = o; p.part_o = part_o; p.part_lse = part_lse;
    p.scale_log2e = scale_log2e; p.split_tokens = split_tokens; p.num_splits = num_splits; p.cur_layer = cur_layer;
    p.num_layers = num_layers; p.nq = nq; p.nkv = nkv; p.max_blocks_per_seq = max_blocks_per_seq; p.num_seqs = num_seqs;
    p.num_items = num_seqs * nkv * num_splits;
    p.tma_4d = g_kv_4d_ok == 1;
    if (p.tma_4d) { p.page_stride = 4096; p.tg_stride = 2048; p.half_stride = 1024; p.k_sbo = 2048; p.v_lbo = 1024; p.v_sbo = 2048; }
    else          { p.page_stride = 2048; p.tg_stride = 1024; p.half_stride = 16384; p.k_sbo = 1024; p.v_lbo = 16384; p.v_sbo = 1024; }
    const int grid = p.num_items < num_sms ? p.num_items : num_sms;
    const int g = nq / nkv;

#define SLLM_TC_LAUNCH(TT, GG)                                                                                          \
    do {                                                                                                                 \
        static unsigned long long configured = 0;                                                                        \
        if (first_use_on_this_device(configured))                                                                        \
            cudaFuncSetAttribute(paged_attn_tc_kernel<TT, GG>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES); \
        paged_attn_tc_kernel<TT, GG><<<grid, TC_THREADS, TC_SMEM_BYTES, stream>>>(kmap, vmap, qmap, p);                  \
    } while (0)
    if (dtype == SLLM_F16) {
        if (g <= 8) SLLM_TC_LAUNCH(__half, 8); else SLLM_TC_LAUNCH(__half, 16);
    } else {
        if (g <= 8) SLLM_TC_LAUNCH(__nv_bfloat16, 8); else SLLM_TC_LAUNCH(__nv_bfloat16, 16);
    }
#undef SLLM_TC_LAUNCH
    return check_launch("paged_attention(wgmma)");
}

// The verify kernel serves head_dim 128, block_size 16 and at most 32 (row, head) columns per item.
bool tc_verify_supported(int head_dim, int block_size, int nq, int nkv, int max_rows, int64_t num_blocks, int num_layers,
                         int64_t num_tokens) {
    return tc_paged_supported(head_dim, block_size, nq, nkv, num_blocks, num_layers) && (nq / nkv) * max_rows <= 32 &&
           num_tokens < (1LL << 31);
}

int launch_paged_verify_tc(const void* q, const void* k_cache, const void* v_cache, const int32_t* block_table,
                           const int32_t* seq_ids, const int32_t* start_locs, const int32_t* row_counts,
                           const int32_t* prefix_lens, void* o, float* part_o, float* part_lse, int32_t* row_lens,
                           float scale_log2e, int num_seqs, int max_rows, int64_t num_tokens, int split_tokens, int num_splits,
                           int cur_layer, int num_layers, int nq, int nkv, int max_blocks_per_seq, int64_t num_blocks,
                           int64_t q_row_stride, sllm_dtype_t dtype, int num_sms, cudaStream_t stream) {
    const uint64_t rows = (uint64_t)num_blocks * num_layers * nkv * TC_BS;
    const int g = nq / nkv;
    CUtensorMap kmap, vmap, qmap;
    if (g_kv_4d_ok != 0) {
        bool ok = get_map(&kmap, k_cache, rows, 1, dtype, true) && get_map(&vmap, v_cache, rows, 1, dtype, true);
        if (g_kv_4d_ok < 0) g_kv_4d_ok = ok ? 1 : 0;
    }
    if (g_kv_4d_ok == 0) {
        SLLM_REQUIRE(get_map(&kmap, k_cache, rows, 0, dtype, true) && get_map(&vmap, v_cache, rows, 0, dtype, true),
                     "paged_attention_verify: cuTensorMapEncodeTiled failed for the KV cache");
    }
    {   // q as (128 d | nq heads | num_tokens rows), box (64 d, g heads, max_rows rows): encoded per launch
        TensorMapEncodeFn enc = get_tensor_map_encoder();
        cuuint64_t dims[3] = {128, (cuuint64_t)nq, (cuuint64_t)num_tokens};
        cuuint64_t strides[2] = {256, (cuuint64_t)q_row_stride * 2};
        cuuint32_t box[3] = {64, (cuuint32_t)g, (cuuint32_t)max_rows}, es[3] = {1, 1, 1};
        SLLM_REQUIRE(enc && enc(&qmap, map_dtype(dtype), 3, const_cast<void*>(q), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS,
                     "paged_attention_verify: cuTensorMapEncodeTiled failed for q");
    }
    TcVerifyParams p;
    p.block_table = block_table; p.seq_ids = seq_ids; p.start_locs = start_locs; p.row_counts = row_counts;
    p.prefix_lens = prefix_lens; p.o = o; p.part_o = part_o; p.part_lse = part_lse; p.row_lens = row_lens;
    p.scale_log2e = scale_log2e; p.split_tokens = split_tokens; p.num_splits = num_splits; p.cur_layer = cur_layer;
    p.num_layers = num_layers; p.nq = nq; p.nkv = nkv; p.max_blocks_per_seq = max_blocks_per_seq;
    p.num_items = num_seqs * nkv * num_splits; p.qrows = max_rows;
    p.tma_4d = g_kv_4d_ok == 1;
    if (p.tma_4d) { p.page_stride = 4096; p.half_stride = 1024; p.k_sbo = 2048; p.v_lbo = 1024; p.v_sbo = 2048; }
    else          { p.page_stride = 2048; p.half_stride = 16384; p.k_sbo = 1024; p.v_lbo = 16384; p.v_sbo = 1024; }
    const int grid = p.num_items < num_sms ? p.num_items : num_sms;
    const int cols = g * max_rows;

#define SLLM_TCV_LAUNCH(TT, NP)                                                                                          \
    do {                                                                                                                 \
        static unsigned long long configured = 0;                                                                        \
        if (first_use_on_this_device(configured))                                                                        \
            cudaFuncSetAttribute(paged_attn_verify_kernel<TT, NP>, cudaFuncAttributeMaxDynamicSharedMemorySize,          \
                                 VerifyShape<NP>::SMEM_BYTES);                                                           \
        paged_attn_verify_kernel<TT, NP><<<grid, TC_THREADS, VerifyShape<NP>::SMEM_BYTES, stream>>>(kmap, vmap, qmap, p); \
    } while (0)
    if (dtype == SLLM_F16) {
        if (cols <= 8) SLLM_TCV_LAUNCH(__half, 8); else if (cols <= 16) SLLM_TCV_LAUNCH(__half, 16); else SLLM_TCV_LAUNCH(__half, 32);
    } else {
        if (cols <= 8) SLLM_TCV_LAUNCH(__nv_bfloat16, 8); else if (cols <= 16) SLLM_TCV_LAUNCH(__nv_bfloat16, 16);
        else SLLM_TCV_LAUNCH(__nv_bfloat16, 32);
    }
#undef SLLM_TCV_LAUNCH
    return check_launch("paged_attention_verify(wgmma)");
}

}  // namespace sllm
