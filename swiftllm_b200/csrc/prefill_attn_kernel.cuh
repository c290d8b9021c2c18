// Causal varlen prefill attention, generation 1 kernel (cp.async double buffering + mma.sync).  Launched by
// prefill_attn.cu for packed k/v of the batch (PAGED = false: the reference's contract) and for chunked prefill
// (PAGED = true: k/v gathered from the paged KV cache through the block table).
//
// Reference: swiftllm/worker/kernels/prefill_attn.py:9-139 (the Triton kernel) and the flash_attn_varlen_func
// call that stands in for it at swiftllm/worker/layers/transformer_layer.py:86-96.  Numerics follow
// SURVEY.md Appendix A6: S = f32(QK^T) * (scale*log2e); online softmax in fp32 with exp2; P rounded to the
// storage dtype before P.V; o = h(acc / l).
// The sequence END is taken from prefill_seq_lens (never from a cu_seqlens array that includes decode tokens:
// the reference's mixed-batch quirk, SURVEY.md §3.1).
// Roofline: tensor-bound; FLOPs = 4 * nq * D * sum_i L_i (L_i + 1) / 2  (+ 4 * nq * D * sum_i prefix_i * L_i when PAGED).
#pragma once
#include "mma_helpers.cuh"

namespace sllm {

constexpr int PF_BQ = 128;       // query rows per CTA (8 warps x 16 rows)
constexpr int PF_BK = 64;        // kv tokens per stage
constexpr int PF_THREADS = 256;

// Where the keys / values of a PAGED launch live (chunked prefill): the paged KV cache, through the block table.
struct PfPagedKV {
    const int32_t* block_table; const int32_t* seq_ids; const int32_t* prefix_lens;
    int cur_layer, num_layers, block_size, max_blocks_per_seq;
};

// PAGED = false: k, v are the packed [T, nkv, D] rows of this very batch (the reference's contract).
// PAGED = true (chunked prefill, SURVEY.md §8 f-1): k, v are the paged caches [num_blocks, L, nkv, bs, D]; the chunk's
// queries sit at positions prefix .. prefix + len - 1 of their sequence and attend to positions <= their own.
template <typename T, int D, bool PAGED>
__global__ void __launch_bounds__(PF_THREADS, 1) prefill_attn_kernel(
    const T* __restrict__ q, const T* __restrict__ k, const T* __restrict__ v, T* __restrict__ o,
    const int32_t* __restrict__ start_locs, const int32_t* __restrict__ seq_lens, float scale_log2e, int nq, int nkv,
    int64_t qs, int64_t ks, int64_t vs,        // row strides (elements) of q, k, v; o is contiguous [T, nq, D]
    const PfPagedKV pk) {
    constexpr int CPR = D / 8;
    constexpr int Q_BYTES = PF_BQ * D * 2;
    constexpr int KV_BYTES = PF_BK * D * 2;
    extern __shared__ __align__(128) uint8_t pf_smem[];   // [Q tile][stage0: K,V][stage1: K,V]

    const int qb = gridDim.x - 1 - blockIdx.x;          // heaviest (latest) query blocks first
    const int head = blockIdx.y, seq = blockIdx.z;
    const int len = seq_lens[seq];                      // query rows of this sequence in the batch
    const int q0 = qb * PF_BQ;
    if (q0 >= len) return;
    const int pre = PAGED ? pk.prefix_lens[seq] : 0;    // position of query row 0
    const int kvlen = pre + len;
    const int64_t tok0 = start_locs[seq];
    const int kvh = head / (nq / nkv);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    const T* qg = q + tok0 * qs + (int64_t)head * D;
    const T* kg = PAGED ? k : k + tok0 * ks + (int64_t)kvh * D;
    const T* vg = PAGED ? v : v + tok0 * vs + (int64_t)kvh * D;
    const int32_t* bt = PAGED ? pk.block_table + (int64_t)pk.seq_ids[seq] * pk.max_blocks_per_seq : nullptr;
    const int64_t os = (int64_t)nq * D;

    const uint32_t q_sm = smem_u32(pf_smem);
    auto kv_sm = [&](int stage) { return smem_u32(pf_smem + Q_BYTES + stage * 2 * KV_BYTES); };

    // Q tile -> smem (rows past the sequence end are zero-filled)
#pragma unroll
    for (int it = 0; it < PF_BQ * CPR / PF_THREADS; it++) {
        const int idx = tid + it * PF_THREADS, r = idx / CPR, c = idx % CPR;
        const bool valid = q0 + r < len;
        cp_async16(q_sm + tile_off<D>(r, c), qg + (int64_t)(valid ? q0 + r : 0) * qs + c * 8, valid ? 16 : 0);
    }
    cp_async_commit();

    const int kv_end = min(kvlen, pre + q0 + PF_BQ);     // causal: keys < kv_end
    const int ntiles = (kv_end + PF_BK - 1) / PF_BK;
    auto issue_kv = [&](int tile) {
        const uint32_t ksm = kv_sm(tile & 1), vsm = ksm + KV_BYTES;
#pragma unroll
        for (int it = 0; it < PF_BK * CPR / PF_THREADS; it++) {
            const int idx = tid + it * PF_THREADS, r = idx / CPR, c = idx % CPR;
            const int t = tile * PF_BK + r;
            const bool valid = t < kvlen;
            const int64_t tr = valid ? t : 0;
            if constexpr (PAGED) {
                const int64_t blk = bt[tr / pk.block_size];
                const int64_t off = (((blk * pk.num_layers + pk.cur_layer) * nkv + kvh) * pk.block_size + tr % pk.block_size) * D + c * 8;
                cp_async16(ksm + tile_off<D>(r, c), kg + off, valid ? 16 : 0);
                cp_async16(vsm + tile_off<D>(r, c), vg + off, valid ? 16 : 0);
            } else {
                cp_async16(ksm + tile_off<D>(r, c), kg + tr * ks + c * 8, valid ? 16 : 0);
                cp_async16(vsm + tile_off<D>(r, c), vg + tr * vs + c * 8, valid ? 16 : 0);
            }
        }
    };
    issue_kv(0);
    cp_async_commit();

    // Q fragments for this warp's 16 rows
    cp_async_wait<1>();
    __syncthreads();
    uint32_t qa[D / 16][4];
    {
        const int mid = lane >> 3, r8 = lane & 7;
        const int row = warp * 16 + (mid & 1) * 8 + r8;           // matrices: (rows 0-7,k lo) (rows 8-15,k lo) (rows 0-7,k hi) (rows 8-15,k hi)
#pragma unroll
        for (int ks = 0; ks < D / 16; ks++)
            ldmatrix_x4(q_sm + tile_off<D>(row, 2 * ks + (mid >> 1)), qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3]);
    }

    float o_acc[D / 8][4];
#pragma unroll
    for (int j = 0; j < D / 8; j++) { o_acc[j][0] = o_acc[j][1] = o_acc[j][2] = o_acc[j][3] = 0.f; }
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    const int row0 = pre + q0 + warp * 16 + (lane >> 2), row1 = row0 + 8;     // absolute (in-sequence) positions of this thread's query rows

    for (int tile = 0; tile < ntiles; tile++) {
        if (tile + 1 < ntiles) issue_kv(tile + 1);
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();                                   // tile landed
        const uint32_t ks_base = kv_sm(tile & 1), vs_base = ks_base + KV_BYTES;
        const int kt0 = tile * PF_BK;
        const int mid = lane >> 3, r8 = lane & 7;
        // warp-uniform skip: this tile is entirely above the diagonal for all 16 rows of the warp
        const bool skip = kt0 > pre + q0 + warp * 16 + 15;
        if (!skip) {
            float s[PF_BK / 8][4];
#pragma unroll
            for (int nb = 0; nb < PF_BK / 8; nb++) { s[nb][0] = s[nb][1] = s[nb][2] = s[nb][3] = 0.f; }
#pragma unroll
            for (int ks = 0; ks < D / 16; ks++) {
#pragma unroll
                for (int np = 0; np < PF_BK / 16; np++) {
                    uint32_t b0, b1, b2, b3;
                    const int krow = np * 16 + (mid >> 1) * 8 + r8;
                    ldmatrix_x4(ks_base + tile_off<D>(krow, 2 * ks + (mid & 1)), b0, b1, b2, b3);
                    mma_16816<T>(s[2 * np], qa[ks], b0, b1);
                    mma_16816<T>(s[2 * np + 1], qa[ks], b2, b3);
                }
            }
            const bool need_mask = kt0 + PF_BK - 1 > pre + q0 + warp * 16 || kt0 + PF_BK > kvlen;
            float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
            for (int nb = 0; nb < PF_BK / 8; nb++) {
                const int col = kt0 + nb * 8 + (lane & 3) * 2;
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const int cc = col + (e & 1), rr = (e < 2) ? row0 : row1;
                    float x = s[nb][e] * scale_log2e;
                    if (need_mask && (cc > rr || cc >= kvlen)) x = -INFINITY;
                    s[nb][e] = x;
                }
                mx0 = fmaxf(mx0, fmaxf(s[nb][0], s[nb][1]));
                mx1 = fmaxf(mx1, fmaxf(s[nb][2], s[nb][3]));
            }
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
            // a row can still be fully masked here only if it lies past the sequence end: keep it finite
            const float mn0 = fmaxf(fmaxf(m0, mx0), -1e30f), mn1 = fmaxf(fmaxf(m1, mx1), -1e30f);
            const float a0 = fast_exp2(m0 - mn0), a1 = fast_exp2(m1 - mn1);
            m0 = mn0; m1 = mn1;
            float ps0 = 0.f, ps1 = 0.f;
            uint32_t pa[PF_BK / 16][4];
#pragma unroll
            for (int np = 0; np < PF_BK / 16; np++) {
                const float p00 = fast_exp2(s[2 * np][0] - mn0), p01 = fast_exp2(s[2 * np][1] - mn0);
                const float p02 = fast_exp2(s[2 * np][2] - mn1), p03 = fast_exp2(s[2 * np][3] - mn1);
                const float p10 = fast_exp2(s[2 * np + 1][0] - mn0), p11 = fast_exp2(s[2 * np + 1][1] - mn0);
                const float p12 = fast_exp2(s[2 * np + 1][2] - mn1), p13 = fast_exp2(s[2 * np + 1][3] - mn1);
                ps0 += (p00 + p01) + (p10 + p11);
                ps1 += (p02 + p03) + (p12 + p13);
                pa[np][0] = pack2<T>(p00, p01); pa[np][1] = pack2<T>(p02, p03);
                pa[np][2] = pack2<T>(p10, p11); pa[np][3] = pack2<T>(p12, p13);
            }
            l0 = l0 * a0 + ps0;
            l1 = l1 * a1 + ps1;
#pragma unroll
            for (int j = 0; j < D / 8; j++) { o_acc[j][0] *= a0; o_acc[j][1] *= a0; o_acc[j][2] *= a1; o_acc[j][3] *= a1; }
#pragma unroll
            for (int np = 0; np < PF_BK / 16; np++) {
                const int vrow = np * 16 + (mid & 1) * 8 + r8;
#pragma unroll
                for (int jp = 0; jp < D / 16; jp++) {
                    uint32_t b0, b1, b2, b3;
                    ldmatrix_x4_trans(vs_base + tile_off<D>(vrow, 2 * jp + (mid >> 1)), b0, b1, b2, b3);
                    mma_16816<T>(o_acc[2 * jp], pa[np], b0, b1);
                    mma_16816<T>(o_acc[2 * jp + 1], pa[np], b2, b3);
                }
            }
        }
        __syncthreads();                                   // everyone done with this stage before it is refilled
    }

    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.f / l0, i1 = 1.f / l1;
    T* og = o + (tok0 * nq + head) * D;
    const int c0 = (lane & 3) * 2;
#pragma unroll
    for (int j = 0; j < D / 8; j++) {
        if (row0 < kvlen) *reinterpret_cast<uint32_t*>(og + (int64_t)(row0 - pre) * os + j * 8 + c0) = pack2<T>(o_acc[j][0] * i0, o_acc[j][1] * i0);
        if (row1 < kvlen) *reinterpret_cast<uint32_t*>(og + (int64_t)(row1 - pre) * os + j * 8 + c0) = pack2<T>(o_acc[j][2] * i1, o_acc[j][3] * i1);
    }
}

}  // namespace sllm
