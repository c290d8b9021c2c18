// Paged (decode) attention, generation 1: cp.async page gather + mma.sync tiles.
//
// Reference: swiftllm/worker/kernels/paged_attn.py (phase 1 :9-108, phase 2 :111-149, wrapper :152-222).
// What is different by design:
//   * one CTA serves the WHOLE GQA group of a (sequence, kv head[, split]): K/V pages are read from HBM once,
//     not once per q head (the reference launches one program per q head and leans on L2);
//   * QK^T and PV run on tensor cores with fp32 accumulation (the reference accumulates q.k in the storage
//     dtype on CUDA cores, paged_attn.py:72,92);
//   * pages are gathered through the block table with a 3-stage cp.async pipeline (64 tokens per stage);
//   * v1 (single pass, writes o directly) when the batch alone fills the GPU, v2 (flash-decoding split +
//     merge kernel, same (normalised o, log2-sum-exp) partial format as the reference) otherwise.
// HBM roofline: algorithmic bytes per launch = sum_i len_i * nkv * D * 2 (K and V) * sizeof(T)
//               + 2 * Bd * nq * D * sizeof(T)  (SURVEY.md §8d).
#include "mma_helpers.cuh"
#include "paged_attn_tc.cuh"      // generation 2

namespace sllm {

constexpr int PA_TILE = 64;          // tokens per pipeline stage
constexpr int PA_STAGES = 3;
constexpr int PA_THREADS = 128;      // 4 warps, warp w owns tokens [16w, 16w+16) of every tile
constexpr int PA_MAX_SPLIT_TOKENS = 16384;

struct PagedAttnParams {
    const void* q; const void* k_cache; const void* v_cache;
    const int32_t* block_table; const int32_t* seq_ids; const int32_t* seq_lens;
    void* o; float* part_o; float* part_lse;
    float scale_log2e;
    int split_tokens, num_splits, cur_layer, num_layers, nq, nkv, block_size, max_blocks_per_seq;
    int64_t q_stride;                 // elements between consecutive q rows (sequences)
};

template <typename T, int D>
__global__ void __launch_bounds__(PA_THREADS, 2) paged_attn_kernel(const PagedAttnParams p) {
    constexpr int CPR = D / 8;                        // 16-byte chunks per row
    constexpr int TILE_BYTES = PA_TILE * D * 2;
    extern __shared__ __align__(128) uint8_t smem[];
    // layout: [stage][K tile | V tile] then page-id table
    int32_t* page_ids = reinterpret_cast<int32_t*>(smem + PA_STAGES * 2 * TILE_BYTES);

    const int split = blockIdx.x, kvh = blockIdx.y, seq = blockIdx.z;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = p.nq / p.nkv;                       // GQA group size (<= 16)
    const int seq_len = p.seq_lens[seq];
    const int split_start = split * p.split_tokens;
    if (split_start >= seq_len) return;               // this split does not exist for this sequence
    const int split_len = min(p.split_tokens, seq_len - split_start);
    const int ntiles = (split_len + PA_TILE - 1) / PA_TILE;
    const int bs = p.block_size;

    // ---- page ids of this split -> shared memory
    {
        const int first_page = split_start / bs;
        const int npages = (split_start + split_len + bs - 1) / bs - first_page;
        const int32_t* row = p.block_table + (int64_t)p.seq_ids[seq] * p.max_blocks_per_seq + first_page;
        for (int i = tid; i < npages; i += PA_THREADS) page_ids[i] = row[i];
    }
    __syncthreads();

    const T* kc = reinterpret_cast<const T*>(p.k_cache);
    const T* vc = reinterpret_cast<const T*>(p.v_cache);
    const int64_t page_stride = (int64_t)p.num_layers * p.nkv * bs * D;            // elements per block
    const int64_t head_off = ((int64_t)p.cur_layer * p.nkv + kvh) * bs * D;
    const int page_base_tok = (split_start / bs) * bs;                              // token index of page_ids[0]

    auto issue_tile = [&](int tile) {
        const int stage = tile % PA_STAGES;
        const uint32_t ks = smem_u32(smem + stage * 2 * TILE_BYTES);
        const uint32_t vs = ks + TILE_BYTES;
        const int tok0 = tile * PA_TILE;
#pragma unroll
        for (int it = 0; it < PA_TILE * CPR / PA_THREADS; it++) {
            const int idx = tid + it * PA_THREADS;
            const int r = idx / CPR, c = idx % CPR;
            const int tok = tok0 + r;                                               // token within the split
            const bool valid = tok < split_len;
            const int gtok = split_start + (valid ? tok : 0) - page_base_tok;       // token relative to page_ids[0]
            const int64_t off = (int64_t)page_ids[gtok / bs] * page_stride + head_off + (int64_t)(gtok % bs) * D + c * 8;
            const uint32_t so = tile_off<D>(r, c);
            cp_async16(ks + so, kc + off, valid ? 16 : 0);
            cp_async16(vs + so, vc + off, valid ? 16 : 0);
        }
    };

    // ---- Q fragments (A operand, 16 x D, rows >= g are zero)
    uint32_t qa[D / 16][4];
    {
        const T* qb = reinterpret_cast<const T*>(p.q) + (int64_t)seq * p.q_stride + (int64_t)kvh * g * D;
        const int r0 = lane >> 2, r1 = r0 + 8, c0 = (lane & 3) * 2;
#pragma unroll
        for (int ks = 0; ks < D / 16; ks++) {
            const int col = ks * 16 + c0;
            qa[ks][0] = r0 < g ? *reinterpret_cast<const uint32_t*>(qb + (int64_t)r0 * D + col) : 0u;
            qa[ks][1] = r1 < g ? *reinterpret_cast<const uint32_t*>(qb + (int64_t)r1 * D + col) : 0u;
            qa[ks][2] = r0 < g ? *reinterpret_cast<const uint32_t*>(qb + (int64_t)r0 * D + col + 8) : 0u;
            qa[ks][3] = r1 < g ? *reinterpret_cast<const uint32_t*>(qb + (int64_t)r1 * D + col + 8) : 0u;
        }
    }

    float o_acc[D / 8][4];
#pragma unroll
    for (int j = 0; j < D / 8; j++) { o_acc[j][0] = o_acc[j][1] = o_acc[j][2] = o_acc[j][3] = 0.f; }
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;     // running max (scaled, log2 domain) / partial sums
    const float c_scale = p.scale_log2e;

    // ---- pipeline prologue
#pragma unroll
    for (int s = 0; s < PA_STAGES - 1; s++) {
        if (s < ntiles) issue_tile(s);
        cp_async_commit();
    }

    for (int tile = 0; tile < ntiles; tile++) {
        cp_async_wait<PA_STAGES - 2>();
        __syncthreads();                      // tile `tile` landed for everyone; stage (tile-1)%S is free again
        if (tile + PA_STAGES - 1 < ntiles) issue_tile(tile + PA_STAGES - 1);
        cp_async_commit();

        const int wtok0 = tile * PA_TILE + warp * 16;            // first token (within split) of this warp's slice
        if (wtok0 >= split_len) continue;                        // warp-uniform
        const int stage = tile % PA_STAGES;
        const uint32_t ks_base = smem_u32(smem + stage * 2 * TILE_BYTES);
        const uint32_t vs_base = ks_base + TILE_BYTES;
        const int mid = lane >> 3, r8 = lane & 7;

        // S = Q K^T for 16 tokens: two n-blocks of 8 tokens
        float s[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
        {
            const int krow = warp * 16 + (mid >> 1) * 8 + r8;
#pragma unroll
            for (int ks = 0; ks < D / 16; ks++) {
                uint32_t b0, b1, b2, b3;
                ldmatrix_x4(ks_base + tile_off<D>(krow, 2 * ks + (mid & 1)), b0, b1, b2, b3);
                mma_16816<T>(s[0], qa[ks], b0, b1);
                mma_16816<T>(s[1], qa[ks], b2, b3);
            }
        }
        // scale + mask the tail, row max
        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int nb = 0; nb < 2; nb++) {
            const int tok = wtok0 + nb * 8 + (lane & 3) * 2;
            const bool v0 = tok < split_len, v1 = tok + 1 < split_len;
            s[nb][0] = v0 ? s[nb][0] * c_scale : -INFINITY;
            s[nb][1] = v1 ? s[nb][1] * c_scale : -INFINITY;
            s[nb][2] = v0 ? s[nb][2] * c_scale : -INFINITY;
            s[nb][3] = v1 ? s[nb][3] * c_scale : -INFINITY;
            mx0 = fmaxf(mx0, fmaxf(s[nb][0], s[nb][1]));
            mx1 = fmaxf(mx1, fmaxf(s[nb][2], s[nb][3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);     // finite: token wtok0 is valid
        const float a0 = fast_exp2(m0 - mn0), a1 = fast_exp2(m1 - mn1);
        m0 = mn0; m1 = mn1;
        uint32_t pa[4];
        {
            const float p00 = fast_exp2(s[0][0] - mn0), p01 = fast_exp2(s[0][1] - mn0);
            const float p02 = fast_exp2(s[0][2] - mn1), p03 = fast_exp2(s[0][3] - mn1);
            const float p10 = fast_exp2(s[1][0] - mn0), p11 = fast_exp2(s[1][1] - mn0);
            const float p12 = fast_exp2(s[1][2] - mn1), p13 = fast_exp2(s[1][3] - mn1);
            l0 = l0 * a0 + (p00 + p01 + p10 + p11);
            l1 = l1 * a1 + (p02 + p03 + p12 + p13);
            pa[0] = pack2<T>(p00, p01); pa[1] = pack2<T>(p02, p03);
            pa[2] = pack2<T>(p10, p11); pa[3] = pack2<T>(p12, p13);
        }
        // O = O*alpha + P V
        {
            const int vrow = warp * 16 + (mid & 1) * 8 + r8;
#pragma unroll
            for (int jp = 0; jp < D / 16; jp++) {
                uint32_t b0, b1, b2, b3;
                ldmatrix_x4_trans(vs_base + tile_off<D>(vrow, 2 * jp + (mid >> 1)), b0, b1, b2, b3);
                float (&oa)[4] = o_acc[2 * jp];
                float (&ob)[4] = o_acc[2 * jp + 1];
                oa[0] *= a0; oa[1] *= a0; oa[2] *= a1; oa[3] *= a1;
                ob[0] *= a0; ob[1] *= a0; ob[2] *= a1; ob[3] *= a1;
                mma_16816<T>(oa, pa, b0, b1);
                mma_16816<T>(ob, pa, b2, b3);
            }
        }
    }
    cp_async_wait<0>();
    __syncthreads();                               // all tiles consumed: the stage memory can be reused

    // ---- merge the four warps (each saw a disjoint token subset) through shared memory
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    float* sm_o = reinterpret_cast<float*>(smem);                 // [4 warps][16 rows][D]
    float* sm_m = sm_o + 4 * 16 * D;                              // [4][16]
    float* sm_l = sm_m + 4 * 16;                                  // [4][16]
    {
        const int r0 = lane >> 2, r1 = r0 + 8, c0 = (lane & 3) * 2;
        if ((lane & 3) == 0) {
            sm_m[warp * 16 + r0] = m0; sm_l[warp * 16 + r0] = l0;
            sm_m[warp * 16 + r1] = m1; sm_l[warp * 16 + r1] = l1;
        }
#pragma unroll
        for (int j = 0; j < D / 8; j++) {
            if (r0 < g) *reinterpret_cast<float2*>(&sm_o[(warp * 16 + r0) * D + j * 8 + c0]) = make_float2(o_acc[j][0], o_acc[j][1]);
            if (r1 < g) *reinterpret_cast<float2*>(&sm_o[(warp * 16 + r1) * D + j * 8 + c0]) = make_float2(o_acc[j][2], o_acc[j][3]);
        }
    }
    __syncthreads();
    for (int idx = tid; idx < g * D; idx += PA_THREADS) {
        const int r = idx / D, d = idx % D;
        float mw[4], mstar = -INFINITY;
#pragma unroll
        for (int w = 0; w < 4; w++) { mw[w] = sm_m[w * 16 + r]; mstar = fmaxf(mstar, mw[w]); }
        float L = 0.f, O = 0.f;
#pragma unroll
        for (int w = 0; w < 4; w++) {
            const float e = fast_exp2(mw[w] - mstar);              // exp2(-inf) = 0 for warps that saw no token
            L += sm_l[w * 16 + r] * e;
            O += sm_o[(w * 16 + r) * D + d] * e;
        }
        const float out = O / L;
        const int head = kvh * g + r;
        if (p.num_splits == 1) {
            reinterpret_cast<T*>(p.o)[((int64_t)seq * p.nq + head) * D + d] = Traits<T>::from_f(out);
        } else {
            const int64_t pi = ((int64_t)seq * p.nq + head) * p.num_splits + split;
            p.part_o[pi * D + d] = out;
            if (d == 0) p.part_lse[pi] = log2f(L) + mstar;         // same partial format as paged_attn.py:105-108
        }
    }
}

// Phase 2 (paged_attn.py:111-149): exp2-weighted merge of the valid splits.  grid (nq, Bd), D threads.
template <typename T>
__global__ void paged_attn_merge_kernel(const float* __restrict__ part_o, const float* __restrict__ part_lse,
                                        T* __restrict__ o, const int32_t* __restrict__ seq_lens, int nq, int D,
                                        int num_splits, int split_tokens) {
    const int head = blockIdx.x, seq = blockIdx.y, d = threadIdx.x;
    const int n = (seq_lens[seq] + split_tokens - 1) / split_tokens;
    const int64_t base = ((int64_t)seq * nq + head) * num_splits;
    float m = -INFINITY;
    for (int s = 0; s < n; s++) m = fmaxf(m, part_lse[base + s]);
    float L = 0.f, O = 0.f;
    for (int s = 0; s < n; s++) {
        const float e = fast_exp2(part_lse[base + s] - m);
        L += e;
        O += e * part_o[(base + s) * D + d];
    }
    o[((int64_t)seq * nq + head) * D + d] = Traits<T>::from_f(O / L);
}

// `lens`: the visible length of each of the `rows` rows of o
template <typename T>
static int launch_merge(const float* part_o, const float* part_lse, void* o, const int32_t* lens, int nq, int64_t rows, int head_dim,
                        int num_splits, int split_tokens, cudaStream_t stream, const char* what) {
    dim3 grid(nq, (unsigned)rows);
    paged_attn_merge_kernel<T><<<grid, head_dim, 0, stream>>>(part_o, part_lse, (T*)o, lens, nq, head_dim, num_splits, split_tokens);
    return check_launch(what);
}

// bytes of the fp32 partials (normalised o + log2-sum-exp) of `rows` rows of o split `num_splits` ways
static int64_t partial_bytes(int64_t rows, int nq, int64_t num_splits, int head_dim) {
    return rows * nq * num_splits * (head_dim + 1) * (int64_t)sizeof(float);
}

// ---- host-side split policy (v1 vs v2)
// Tokens per flash-decoding split (a multiple of 128), shared by both kernel generations so the workspace size
// does not depend on which one runs.  Fixed by the caller when seq_block_size > 0.
static int choose_split_tokens(int num_seqs, int nkv, int max_seq_len, int seq_block_size) {
    if (seq_block_size > 0) return seq_block_size;
    const int64_t pairs = (int64_t)num_seqs * nkv;
    const int64_t want = (6LL * num_sms() + pairs - 1) / pairs;    // aim for >= 6 work items per SM
    if (want <= 1) return PA_MAX_SPLIT_TOKENS;                     // v1: one item per (sequence, kv head)
    int64_t st = (max_seq_len + want - 1) / want;
    st = ((st + 127) / 128) * 128;
    if (st < 256) st = 256;
    if (st > PA_MAX_SPLIT_TOKENS) st = PA_MAX_SPLIT_TOKENS;
    return (int)st;
}

template <typename T, int D>
static int launch_paged(const PagedAttnParams& p, int num_seqs, int max_seq_len, cudaStream_t stream) {
    const size_t smem = (size_t)PA_STAGES * 2 * PA_TILE * D * 2 + (size_t)(p.split_tokens / p.block_size + 2) * sizeof(int32_t);
    SLLM_REQUIRE(smem <= 110 * 1024, "paged_attention: split too long for shared memory (%zu bytes)", smem);
    if (int e = fit_dynamic_smem<paged_attn_kernel<T, D>>(smem, "paged_attention(phase 1)")) return e;
    dim3 grid(p.num_splits, p.nkv, num_seqs);
    paged_attn_kernel<T, D><<<grid, PA_THREADS, smem, stream>>>(p);
    int e = check_launch("paged_attention(phase 1)");
    if (e) return e;
    if (p.num_splits > 1)
        return launch_merge<T>(p.part_o, p.part_lse, p.o, p.seq_lens, p.nq, num_seqs, D, p.num_splits, p.split_tokens, stream,
                               "paged_attention(phase 2)");
    return 0;
}

}  // namespace sllm

using namespace sllm;

extern "C" {

int64_t sllm_paged_attention_workspace_bytes(int num_decoding_seqs, int nq, int head_dim, int max_seq_len,
                                             int seq_block_size, int nkv) {
    if (num_decoding_seqs <= 0 || max_seq_len <= 0) return 0;
    const int st = choose_split_tokens(num_decoding_seqs, nkv, max_seq_len, seq_block_size);
    const int64_t ns = (max_seq_len + st - 1) / st;
    if (ns <= 1) return 0;
    return partial_bytes(num_decoding_seqs, nq, ns, head_dim);
}

int sllm_paged_attention(const void* q, const void* k_cache, const void* v_cache, const int32_t* block_table,
                         const int32_t* seq_ids, const int32_t* seq_lens, void* o, void* workspace,
                         int64_t workspace_bytes, float softmax_scale, int num_decoding_seqs, int max_seq_len,
                         int seq_block_size, int cur_layer, int num_layers, int nq, int nkv, int block_size,
                         int head_dim, int max_blocks_per_seq, int64_t num_blocks, int64_t q_row_stride,
                         sllm_dtype_t dtype, sllm_stream_t stream) {
    SLLM_REQUIRE(num_decoding_seqs >= 0, "paged_attention: negative batch");
    if (num_decoding_seqs == 0) return 0;
    SLLM_REQUIRE(q && k_cache && v_cache && block_table && seq_ids && seq_lens && o, "paged_attention: null pointer");
    SLLM_REQUIRE(head_dim == 64 || head_dim == 128, "paged_attention: head_dim %d not supported (64, 128)", head_dim);
    SLLM_REQUIRE(nkv > 0 && nq % nkv == 0 && nq / nkv <= 16, "paged_attention: GQA group %d/%d not supported (<=16)", nq, nkv);
    SLLM_REQUIRE(block_size > 0 && max_seq_len > 0 && cur_layer >= 0 && cur_layer < num_layers, "paged_attention: bad geometry");
    SLLM_REQUIRE(seq_block_size >= 0 && seq_block_size % block_size == 0,
                 "paged_attention: seq_block_size (%d) must be a multiple of block_size (%d)", seq_block_size, block_size);
    SLLM_REQUIRE(q_row_stride >= (int64_t)nq * head_dim && q_row_stride % 8 == 0, "paged_attention: bad q row stride %lld", (long long)q_row_stride);
    SLLM_REQUIRE(seq_block_size <= PA_MAX_SPLIT_TOKENS, "paged_attention: seq_block_size %d > %d", seq_block_size, PA_MAX_SPLIT_TOKENS);
    PagedAttnParams p;
    p.q = q; p.k_cache = k_cache; p.v_cache = v_cache; p.block_table = block_table; p.seq_ids = seq_ids; p.seq_lens = seq_lens;
    p.o = o;
    p.scale_log2e = softmax_scale * 1.4426950408889634f;
    p.split_tokens = choose_split_tokens(num_decoding_seqs, nkv, max_seq_len, seq_block_size);
    p.num_splits = (max_seq_len + p.split_tokens - 1) / p.split_tokens;
    p.cur_layer = cur_layer; p.num_layers = num_layers; p.nq = nq; p.nkv = nkv; p.block_size = block_size;
    p.max_blocks_per_seq = max_blocks_per_seq; p.q_stride = q_row_stride;
    p.part_o = nullptr; p.part_lse = nullptr;
    if (p.num_splits > 1) {
        const int64_t need = partial_bytes(num_decoding_seqs, nq, p.num_splits, head_dim);
        SLLM_REQUIRE(workspace && workspace_bytes >= need, "paged_attention: workspace too small (%lld < %lld bytes)",
                     (long long)workspace_bytes, (long long)need);
        p.part_o = (float*)workspace;
        p.part_lse = p.part_o + (int64_t)num_decoding_seqs * nq * p.num_splits * head_dim;
    }
    cudaStream_t st = (cudaStream_t)stream;
    // SLLM_PAGED_ATTN_GEN=1 forces the cp.async/mma.sync kernel; default: TMA/wgmma whenever the shape is covered (head_dim 128,
    // block_size 16)
    const int gen = forced_generation("SLLM_PAGED_ATTN_GEN");
    if (gen != 1 && tc_paged_supported(head_dim, block_size, nq, nkv, num_blocks, num_layers) && dtype <= SLLM_BF16) {
        TcLaunch a = {};
        a.p.block_table = block_table; a.p.seq_ids = seq_ids; a.p.seq_lens = seq_lens;
        a.p.o = o; a.p.part_o = p.part_o; a.p.part_lse = p.part_lse; a.p.scale_log2e = p.scale_log2e;
        a.p.split_tokens = p.split_tokens; a.p.num_splits = p.num_splits; a.p.cur_layer = cur_layer; a.p.num_layers = num_layers;
        a.p.nq = nq; a.p.nkv = nkv; a.p.max_blocks_per_seq = max_blocks_per_seq;
        a.q = q; a.k_cache = k_cache; a.v_cache = v_cache; a.num_blocks = num_blocks; a.q_row_stride = q_row_stride;
        a.num_tokens = num_decoding_seqs; a.num_seqs = num_decoding_seqs; a.dtype = dtype; a.num_sms = num_sms(); a.stream = st;
        int e = launch_paged_tc(a);
        if (e) return e;
        if (p.num_splits > 1)
            SLLM_DISPATCH_DTYPE(dtype, return (launch_merge<T>(p.part_o, p.part_lse, o, seq_lens, nq, num_decoding_seqs, head_dim,
                                                               p.num_splits, p.split_tokens, st, "paged_attention(phase 2)")));
        return 0;
    }
    SLLM_REQUIRE(gen != 2, "paged_attention: SLLM_PAGED_ATTN_GEN=2 but the shape is not covered by the wgmma kernel");
    if (head_dim == 128) { SLLM_DISPATCH_DTYPE(dtype, return (launch_paged<T, 128>(p, num_decoding_seqs, max_seq_len, st))); }
    else { SLLM_DISPATCH_DTYPE(dtype, return (launch_paged<T, 64>(p, num_decoding_seqs, max_seq_len, st))); }
    return 0;
}

// ---- speculative verification: splits are planned over (entries x kv heads) with the longest visible length, partials are
// [rows, nq, num_splits] + per-row visible lengths (int32 [num_tokens]), merged by paged_attn_merge_kernel
int64_t sllm_paged_attention_verify_workspace_bytes(int num_seqs, int64_t num_tokens, int nq, int nkv, int head_dim,
                                                    int max_seq_len) {
    if (num_seqs <= 0 || num_tokens <= 0 || max_seq_len <= 0 || nkv <= 0) return 0;
    const int st = choose_split_tokens(num_seqs, nkv, max_seq_len, 0);
    const int64_t ns = (max_seq_len + st - 1) / st;
    if (ns <= 1) return 0;
    return partial_bytes(num_tokens, nq, ns, head_dim) + num_tokens * (int64_t)sizeof(int32_t);
}

int sllm_paged_attention_verify(const void* q, const void* k_cache, const void* v_cache, void* o, const int32_t* block_table,
                                const int32_t* seq_ids, const int32_t* start_locs, const int32_t* row_counts,
                                const int32_t* prefix_lens, void* workspace, int64_t workspace_bytes, float softmax_scale,
                                int num_seqs, int max_rows, int max_seq_len, int64_t num_tokens, int cur_layer, int num_layers,
                                int nq, int nkv, int block_size, int head_dim, int max_blocks_per_seq, int64_t num_blocks,
                                int64_t q_row_stride, sllm_dtype_t dtype, sllm_stream_t stream) {
    SLLM_REQUIRE(num_seqs >= 0 && num_tokens >= 0, "paged_attention_verify: negative sizes");
    if (num_seqs == 0) return 0;
    SLLM_REQUIRE(q && k_cache && v_cache && o && block_table && seq_ids && start_locs && row_counts && prefix_lens,
                 "paged_attention_verify: null pointer");
    SLLM_REQUIRE(max_rows >= 1 && max_rows <= 8, "paged_attention_verify: max_rows %d outside [1, 8]", max_rows);
    SLLM_REQUIRE(num_tokens >= max_rows && max_seq_len >= max_rows, "paged_attention_verify: num_tokens / max_seq_len below max_rows");
    SLLM_REQUIRE(head_dim == 64 || head_dim == 128, "paged_attention_verify: head_dim %d not supported (64, 128)", head_dim);
    SLLM_REQUIRE(nkv > 0 && nq % nkv == 0, "paged_attention_verify: nq %d not a multiple of nkv %d", nq, nkv);
    SLLM_REQUIRE(q_row_stride >= (int64_t)nq * head_dim && q_row_stride % 8 == 0, "paged_attention_verify: bad q row stride");
    SLLM_REQUIRE(block_size > 0 && num_layers > 0 && cur_layer >= 0 && cur_layer < num_layers && max_blocks_per_seq > 0 && num_blocks > 0,
                 "paged_attention_verify: bad cache geometry (layer %d of %d)", cur_layer, num_layers);
    cudaStream_t st = (cudaStream_t)stream;
    // SLLM_PAGED_ATTN_GEN=1 forces the paged-prefill kernel below, =2 makes a shape the verify kernel does not serve an error
    const int gen = forced_generation("SLLM_PAGED_ATTN_GEN");
    if (gen != 1 && dtype <= SLLM_BF16 &&
        tc_verify_supported(head_dim, block_size, nq, nkv, max_rows, num_blocks, num_layers, num_tokens)) {
        const int split_tokens = choose_split_tokens(num_seqs, nkv, max_seq_len, 0);
        const int num_splits = (max_seq_len + split_tokens - 1) / split_tokens;
        float *part_o = nullptr, *part_lse = nullptr;
        int32_t* row_lens = nullptr;
        if (num_splits > 1) {
            const int64_t need = sllm_paged_attention_verify_workspace_bytes(num_seqs, num_tokens, nq, nkv, head_dim, max_seq_len);
            SLLM_REQUIRE(workspace && workspace_bytes >= need, "paged_attention_verify: workspace too small (%lld < %lld bytes)",
                         (long long)workspace_bytes, (long long)need);
            part_o = (float*)workspace;
            part_lse = part_o + num_tokens * nq * num_splits * head_dim;
            row_lens = (int32_t*)(part_lse + num_tokens * nq * num_splits);
        }
        TcLaunch a = {};
        a.p.block_table = block_table; a.p.seq_ids = seq_ids; a.p.start_locs = start_locs; a.p.row_counts = row_counts;
        a.p.prefix_lens = prefix_lens; a.p.o = o; a.p.part_o = part_o; a.p.part_lse = part_lse; a.p.row_lens = row_lens;
        a.p.scale_log2e = softmax_scale * 1.4426950408889634f; a.p.split_tokens = split_tokens; a.p.num_splits = num_splits;
        a.p.cur_layer = cur_layer; a.p.num_layers = num_layers; a.p.nq = nq; a.p.nkv = nkv;
        a.p.max_blocks_per_seq = max_blocks_per_seq; a.p.qrows = max_rows;
        a.q = q; a.k_cache = k_cache; a.v_cache = v_cache; a.num_blocks = num_blocks; a.q_row_stride = q_row_stride;
        a.num_tokens = num_tokens; a.num_seqs = num_seqs; a.dtype = dtype; a.num_sms = num_sms(); a.stream = st;
        int e = launch_paged_verify_tc(a);
        if (e) return e;
        if (num_splits > 1)
            SLLM_DISPATCH_DTYPE(dtype, return (launch_merge<T>(part_o, part_lse, o, row_lens, nq, num_tokens, head_dim, num_splits,
                                                               split_tokens, st, "paged_attention_verify(merge)")));
        return 0;
    }
    SLLM_REQUIRE(gen != 2, "paged_attention_verify: SLLM_PAGED_ATTN_GEN=2 but the shape is not covered by the wgmma verify kernel");
    // shapes the verify kernel does not serve: the chunked-prefill kernel computes the same function (rows = chunk tokens)
    return sllm_prefill_attention_paged(q, k_cache, v_cache, o, block_table, seq_ids, start_locs, row_counts, prefix_lens,
                                        softmax_scale, num_seqs, max_rows, num_tokens, cur_layer, num_layers, nq, nkv, block_size,
                                        head_dim, max_blocks_per_seq, num_blocks, q_row_stride, dtype, stream);
}

}  // extern "C"
