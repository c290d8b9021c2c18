// Causal varlen prefill attention, generation 2 kernel: TMA + wgmma, two consumer warpgroups per CTA (sm_90a).
// Launched by prefill_attn.cu for packed k/v of the batch (PAGED = false) and for chunked prefill (PAGED = true: K/V pages
// gathered from the KV cache through the block table).
//
// Reference being replaced: swiftllm/worker/kernels/prefill_attn.py:9-139 and the flash_attn_varlen_func call at
// swiftllm/worker/layers/transformer_layer.py:86-96.  head_dim 128, fp16/bf16; numerics per SURVEY.md Appendix A6
// (fp32 scores, exp2 online softmax in fp32, P rounded to the storage dtype before P.V, o = h(acc / l)).
//
// CTA = (sequence, q head, 128 query rows).  384 threads:
//   warp 0 / 1  TMA producers: warp 0 loads Q (2 boxes of 128 rows x 64 d) once and then the K tiles, warp 1 the V tiles
//               (2 boxes of 64 x 64 per 64-token step) into separate 3-stage rings with their own mbarriers.
//   warpgroups 1 and 2  query rows 0-63 and 64-127: S[64 x 64] = Q . K_j^T   (8 wgmma m64n64k16, both operands in shared
//               memory), online softmax on the register tile (row max / sum over the 4 lanes of a quad), P rounded to
//               the storage dtype as register A operands of O[64 x 128] += P . V_j   (4 wgmma m64n128k16, V MN-major).
//               O is rescaled only when the running max grew by more than 2^8 ("lazy rescale": the reference point m_ref
//               trails the true max, exact in the end because l uses the same reference).
// Roofline: tensor-bound; FLOPs = 4 * nq * D * sum_i L_i (L_i + 1) / 2.
#pragma once
#include "tc_helpers.cuh"

namespace sllm {

using namespace tc;

constexpr int PT_D = 128;
constexpr int PT_BQ = 128;                // query rows per CTA (64 per consumer warpgroup)
constexpr int PT_BK = 64;                 // kv tokens per pipeline step
constexpr int PT_STAGES = 3;               // K and V rings (separate producers): two steps of prefetch ahead of the MMA
constexpr int PT_THREADS = 384;            // warpgroup 0: warp 0 Q+K producer, warp 1 V producer; warpgroups 1, 2: MMA + softmax
constexpr int PT_Q_BYTES = PT_BQ * PT_D * 2;          // 32 KiB ([half][128 rows][128 B])
constexpr int PT_KV_BYTES = PT_BK * PT_D * 2;         // 16 KiB per K (or V) tile ([half][64 rows][128 B])
constexpr int PT_SMEM_BYTES = PT_Q_BYTES + 2 * PT_STAGES * PT_KV_BYTES + 1024;
constexpr float PT_RESCALE_THRESHOLD = 8.0f;          // log2 units

struct PtBarriers {
    uint64_t q_full;
    uint64_t k_full[PT_STAGES], k_empty[PT_STAGES], v_full[PT_STAGES], v_empty[PT_STAGES];
    uint64_t v_tail;                      // packed only: the TMA of a last V step that ends past the sequence completes here
};

struct PtParams {
    void* o;
    const int32_t* start_locs; const int32_t* seq_lens;
    float scale_log2e;
    int nq, nkv;
};
// PAGED launches (chunked prefill): where the keys / values live.  kmap / vmap then describe the paged caches as
// [num_blocks * L * nkv * 16 rows, 128] with boxes of (64 d x 16 tokens) = one d-half of one page.
struct PtPaged {
    const int32_t* block_table; const int32_t* seq_ids; const int32_t* prefix_lens;
    int cur_layer, num_layers, max_blocks_per_seq;
};
constexpr int PT_PAGE = 16;               // tokens per KV page (PAGED only)

// PAGED = false: K/V tiles come from the packed k/v rows of the batch (the reference's contract).
// PAGED = true (chunked prefill, SURVEY.md §8 f-1): the chunk's queries sit at positions prefix .. prefix + len - 1 of
// their sequence; every 64-token K/V step is gathered from four 16-token pages of the KV cache through the block
// table (lanes 0-3 of the producer warp issue the two d-half boxes of one page each), landing in the SAME
// [half][64 rows][128 B] layout, so the consumer warpgroups and their descriptors are shared by both variants.
template <typename T, bool PAGED>
__global__ void __launch_bounds__(PT_THREADS, 1) prefill_attn_tc_kernel(const __grid_constant__ CUtensorMap qmap,
                                                                        const __grid_constant__ CUtensorMap kmap,
                                                                        const __grid_constant__ CUtensorMap vmap,
                                                                        const PtParams p, const PtPaged pg) {
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* q_sm = smem;                                       // [2 halves][128 rows][128 B]
    uint8_t* k_sm = q_sm + PT_Q_BYTES;                          // [stage][2 halves][64 rows][128 B]
    uint8_t* v_sm = k_sm + PT_STAGES * PT_KV_BYTES;
    PtBarriers* bars = reinterpret_cast<PtBarriers*>(v_sm + PT_STAGES * PT_KV_BYTES);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int qblk = gridDim.x - 1 - blockIdx.x;                // latest (heaviest) query blocks first
    const int head = blockIdx.y, seq = blockIdx.z;
    const int len = p.seq_lens[seq];                            // query rows of this sequence in the batch
    const int q0 = qblk * PT_BQ;
    if (q0 >= len) return;
    const int tok0 = p.start_locs[seq];
    const int kvh = head / (p.nq / p.nkv);
    const int pre = PAGED ? pg.prefix_lens[seq] : 0;            // position of query row 0 within its sequence
    const int kvlen = pre + len;
    // kv steps of the CTA; both warpgroups run all of them (the last one may be fully masked for warpgroup 1's rows)
    const int nkt = (min(kvlen, pre + q0 + PT_BQ) + PT_BK - 1) / PT_BK;

    if constexpr (PAGED) {
        // page slots that a tail step never loads must hold finite data (their P columns are exactly 0)
        uint4* z = reinterpret_cast<uint4*>(k_sm);
        for (int i = tid; i < 2 * PT_STAGES * PT_KV_BYTES / 16; i += PT_THREADS) z[i] = make_uint4(0, 0, 0, 0);
        fence_proxy_async();
    }
    if (tid == 0) {
        mbar_init(smem_u32(&bars->q_full), 1);
        for (int i = 0; i < PT_STAGES; i++) {
            mbar_init(smem_u32(&bars->k_full[i]), 1); mbar_init(smem_u32(&bars->k_empty[i]), 256);
            mbar_init(smem_u32(&bars->v_full[i]), 1); mbar_init(smem_u32(&bars->v_empty[i]), 256);
        }
        if constexpr (!PAGED) mbar_init(smem_u32(&bars->v_tail), 1);
        mbar_fence_init();
        tma_prefetch_desc(&qmap); tma_prefetch_desc(&kmap); tma_prefetch_desc(&vmap);
    }
    __syncthreads();

    // PAGED producer (one whole warp per ring): step j = pages 4j .. 4j+3 of the sequence.  The four block-table
    // entries of the NEXT step are fetched before this step's stage is waited for; lane 0 arms the mbarrier with the
    // bytes of the pages that exist, then lanes 0..3 issue the two (64 d x 16 token) boxes of one page each.
    auto paged_producer = [&](const CUtensorMap& map, uint8_t* ring, uint64_t* full, uint64_t* empty) {
        const int32_t* bt = pg.block_table + (int64_t)pg.seq_ids[seq] * pg.max_blocks_per_seq;
        const int npages = (kvlen + PT_PAGE - 1) / PT_PAGE;
        constexpr int PPS = PT_BK / PT_PAGE;                  // pages per step
        int nxt = (lane < PPS && lane < npages) ? bt[lane] : 0;
        for (int j = 0; j < nkt; j++) {
            const int st = j % PT_STAGES;
            const int blk = nxt;
            const int npg = (j + 1) * PPS + lane;
            nxt = (j + 1 < nkt && lane < PPS && npg < npages) ? bt[npg] : 0;
            const int valid = min(PPS, npages - j * PPS);      // >= 1: step j exists because page 4j does
            const uint32_t bar = smem_u32(&full[st]);
            if (lane == 0) {
                mbar_wait(smem_u32(&empty[st]), ((j / PT_STAGES) & 1) ^ 1);
                mbar_arrive_expect_tx(bar, (uint32_t)valid * PT_PAGE * PT_D * 2);
            }
            __syncwarp();
            if (lane < valid) {
                // row of the cache viewed as [num_blocks * L * nkv * 16 rows, 128]: first token row of this page
                const int64_t row = (((int64_t)blk * pg.num_layers + pg.cur_layer) * p.nkv + kvh) * PT_PAGE;
                const uint32_t dst = smem_u32(ring + st * PT_KV_BYTES) + lane * (PT_PAGE * 128);
                tma_load_2d(dst, &map, bar, 0, (int)row);
                tma_load_2d(dst + PT_KV_BYTES / 2, &map, bar, 64, (int)row);
            }
        }
    };

    if (warp == 0) {
        // =========================================================== TMA producer: Q once, then the K tiles
        if (lane == 0) {
            const uint32_t qbar = smem_u32(&bars->q_full);
            mbar_arrive_expect_tx(qbar, PT_Q_BYTES);
            for (int h = 0; h < 2; h++)
                tma_load_2d(smem_u32(q_sm + h * (PT_Q_BYTES / 2)), &qmap, qbar, head * PT_D + h * 64, tok0 + q0);
            if constexpr (!PAGED) {
                for (int j = 0; j < nkt; j++) {
                    const int st = j % PT_STAGES;
                    mbar_wait(smem_u32(&bars->k_empty[st]), ((j / PT_STAGES) & 1) ^ 1);
                    const uint32_t kb = smem_u32(&bars->k_full[st]);
                    mbar_arrive_expect_tx(kb, PT_KV_BYTES);
                    tma_load_2d(smem_u32(k_sm + st * PT_KV_BYTES), &kmap, kb, kvh * PT_D, tok0 + j * PT_BK);
                    tma_load_2d(smem_u32(k_sm + st * PT_KV_BYTES + PT_KV_BYTES / 2), &kmap, kb, kvh * PT_D + 64, tok0 + j * PT_BK);
                }
            }
        }
        if constexpr (PAGED) paged_producer(kmap, k_sm, bars->k_full, bars->k_empty);
    } else if (warp == 1) {
        // =========================================================== TMA producer: the V tiles (independent of K's progress)
        if constexpr (PAGED) {
            paged_producer(vmap, v_sm, bars->v_full, bars->v_empty);
        } else {
            // The tail step's box runs past the sequence into the next prompt's rows (or rows past the batch).  Their P is
            // exactly 0, but 0 x Inf and 0 x NaN are NaN, so a non-finite V there would leak into this prompt.  That step's
            // TMA therefore completes on v_tail instead; the warp zeroes rows valid..63 and only then completes v_full with a
            // plain arrive, so the consumers are unchanged.  Row r of a d-half is the 128-byte line r (SWIZZLE_128B only
            // permutes the 16-byte chunks within a line).
            const int valid = kvlen - (nkt - 1) * PT_BK;        // rows of the last step inside the sequence
            if (lane == 0) {
                for (int j = 0; j < nkt; j++) {
                    const int st = j % PT_STAGES;
                    mbar_wait(smem_u32(&bars->v_empty[st]), ((j / PT_STAGES) & 1) ^ 1);
                    const uint32_t vb = smem_u32(j == nkt - 1 && valid < PT_BK ? &bars->v_tail : &bars->v_full[st]);
                    mbar_arrive_expect_tx(vb, PT_KV_BYTES);
                    tma_load_2d(smem_u32(v_sm + st * PT_KV_BYTES), &vmap, vb, kvh * PT_D, tok0 + j * PT_BK);
                    tma_load_2d(smem_u32(v_sm + st * PT_KV_BYTES + PT_KV_BYTES / 2), &vmap, vb, kvh * PT_D + 64, tok0 + j * PT_BK);
                }
            }
            if (valid < PT_BK) {
                const int st = (nkt - 1) % PT_STAGES;
                __syncwarp();                                      // lanes 1-31 sleep here while lane 0 streams
                mbar_wait(smem_u32(&bars->v_tail), 0);            // used once per CTA
                uint8_t* tile = v_sm + st * PT_KV_BYTES;
                for (int i = lane; i < 2 * (PT_BK - valid) * 8; i += 32) {         // 8 chunks of 16 B per row and d-half
                    const int h = i / ((PT_BK - valid) * 8), r = valid + (i >> 3) % (PT_BK - valid);
                    *reinterpret_cast<uint4*>(tile + h * (PT_KV_BYTES / 2) + r * 128 + (i & 7) * 16) = make_uint4(0, 0, 0, 0);
                }
                fence_proxy_async();
                __syncwarp();
                if (lane == 0) mbar_arrive(smem_u32(&bars->v_full[st]));
            }
        }
    } else if (warp >= 4) {
        // =========================================================== consumer warpgroup x: query rows 64 x .. 64 x + 63
        // Thread (warp w of the group, lane l) owns rows rr = 16 w + l / 4 + 8 hi (hi in {0, 1}) and, of every 8-column
        // group i, columns 8 i + 2 (l % 4) + {0, 1} of the S and O tiles (see tc_helpers.cuh).
        const int x = (warp >> 2) - 1;
        const int rbase = 16 * (warp & 3) + (lane >> 2);
        const int qi0 = q0 + 64 * x + rbase;              // query index (within the sequence) of the thread's row hi = 0
        const int cb = 2 * (lane & 3);
        // descriptor bases (all tiles live below 256 KiB, so adding 16-byte units to the low word never carries)
        const uint64_t dq0 = make_smem_desc(smem_u32(q_sm + x * 64 * 128), 16, 1024);
        const uint64_t dk0 = make_smem_desc(smem_u32(k_sm), 16, 1024);
        const uint64_t dv0 = make_smem_desc(smem_u32(v_sm), PT_KV_BYTES / 2, 1024);      // MN-major: LBO = d-half stride
        float o[64];
#pragma unroll
        for (int i = 0; i < 64; i++) o[i] = 0.f;
        float m_ref[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
        const float c = p.scale_log2e;
        mbar_wait(smem_u32(&bars->q_full), 0);
        for (int j = 0; j < nkt; j++) {
            const int st = j % PT_STAGES;
            // ---- S = Q . K_j^T
            mbar_wait(smem_u32(&bars->k_full[st]), (j / PT_STAGES) & 1);
            float sc[32];
            {
                const uint64_t kd = dk0 + (uint64_t)((st * PT_KV_BYTES) >> 4);
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < 8; ks++)      // 16 d per wgmma; d-half = ks / 4
                    wgmma_m64n64k16_ss<T, 0, 0>(sc, dq0 + (uint64_t)(((ks >> 2) * (PT_Q_BYTES / 2) + (ks & 3) * 32) >> 4),
                                                kd + (uint64_t)(((ks >> 2) * (PT_KV_BYTES / 2) + (ks & 3) * 32) >> 4), ks > 0);
                wgmma_commit();
                wgmma_wait<0>();
            }
            mbar_arrive(smem_u32(&bars->k_empty[st]));

            // ---- mask, row max over the quad, lazy rescale
            const int c0 = j * PT_BK;
            const bool need_mask = c0 + PT_BK - 1 > pre + q0 + 64 * x || c0 + PT_BK > kvlen;
            float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int hi = 0; hi < 2; hi++) {
                // column c0+i is visible iff c0+i <= pre+qi and c0+i < kvlen  <=>  i <= lim   (branch-free selects)
                const int lim = min(pre + qi0 + 8 * hi, kvlen - 1) - c0;
#pragma unroll
                for (int i = 0; i < 8; i++)
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        float& v = sc[4 * i + 2 * hi + e];
                        if (need_mask && 8 * i + cb + e > lim) v = -INFINITY;
                        mx[hi] = fmaxf(mx[hi], v);
                    }
                mx[hi] = fmaxf(mx[hi], __shfl_xor_sync(0xffffffffu, mx[hi], 1));
                mx[hi] = fmaxf(mx[hi], __shfl_xor_sync(0xffffffffu, mx[hi], 2));
                const float m_new = fmaxf(m_ref[hi], mx[hi] * c);       // max of the RAW scores (scale > 0 commutes with max)
                if (m_new > m_ref[hi] + PT_RESCALE_THRESHOLD) {         // always true on the first step (m_ref = -inf)
                    const float alpha = fast_exp2_tc(m_ref[hi] - m_new);
                    l[hi] *= alpha;
#pragma unroll
                    for (int i = 0; i < 16; i++) { o[4 * i + 2 * hi] *= alpha; o[4 * i + 2 * hi + 1] *= alpha; }
                    m_ref[hi] = m_new;
                }
            }
            // ---- p = exp2(s*c - m_ref) (<= 2^8), row sums in fp32, P -> register A fragments (storage dtype)
            uint32_t pa[4][4];
#pragma unroll
            for (int i = 0; i < 8; i++)
#pragma unroll
                for (int hi = 0; hi < 2; hi++) {
                    const float a = fast_exp2_tc(fmaf(sc[4 * i + 2 * hi], c, -m_ref[hi]));
                    const float b = fast_exp2_tc(fmaf(sc[4 * i + 2 * hi + 1], c, -m_ref[hi]));
                    l[hi] += a + b;
                    typename Traits<T>::T2 v2 = Traits<T>::from_f2(make_float2(a, b));
                    pa[i >> 1][(i & 1) * 2 + hi] = *reinterpret_cast<uint32_t*>(&v2);
                }
            // ---- O += P . V_j
            mbar_wait(smem_u32(&bars->v_full[st]), (j / PT_STAGES) & 1);
            {
                const uint64_t vd = dv0 + (uint64_t)((st * PT_KV_BYTES) >> 4);
                wgmma_fence();
#pragma unroll
                for (int kt = 0; kt < 4; kt++)       // 16 tokens per wgmma
                    wgmma_m64n128k16_rs<T, 1>(o, pa[kt], vd + (uint64_t)((kt * 2048) >> 4), 1);
                wgmma_commit();
                wgmma_wait<0>();
            }
            mbar_arrive(smem_u32(&bars->v_empty[st]));
        }
        // ---- epilogue: O / l -> global (rows inside the sequence)
#pragma unroll
        for (int hi = 0; hi < 2; hi++) {
            l[hi] += __shfl_xor_sync(0xffffffffu, l[hi], 1);
            l[hi] += __shfl_xor_sync(0xffffffffu, l[hi], 2);
            const int qi = qi0 + 8 * hi;
            if (qi < len) {
                const float inv = 1.0f / l[hi];
                T* orow = reinterpret_cast<T*>(p.o) + ((int64_t)(tok0 + qi) * p.nq + head) * PT_D;
#pragma unroll
                for (int i = 0; i < 16; i++) {
                    typename Traits<T>::T2 v2 = Traits<T>::from_f2(make_float2(o[4 * i + 2 * hi] * inv, o[4 * i + 2 * hi + 1] * inv));
                    *reinterpret_cast<typename Traits<T>::T2*>(orow + 8 * i + cb) = v2;
                }
            }
        }
    }
}

}  // namespace sllm
