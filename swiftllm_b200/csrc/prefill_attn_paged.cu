// Chunked ("prefix-aware") prefill attention: the queries of a prompt CHUNK attend to the whole prefix + chunk through
// the paged KV cache.  SURVEY.md §8 f-1: the reference's forward cannot express a partial prompt (its prefill attention,
// swiftllm/worker/kernels/prefill_attn.py:102-139 / transformer_layer.py:86-96, only ever sees the packed k/v of the
// batch), which is what SARATHI-style piggybacking (BASELINE.json configs[2]) needs.  Definition = the one that makes
// a prompt processed in chunks equal to the same prompt processed at once (oracle/kernels.py:
// prefix_prefill_attention_exact).  Both generations of the prefill kernel are instantiated with PAGED = true:
//   gen 2 (prefill_attn_tc_kernel.cuh): TMA page gather + wgmma, head_dim 128, block_size 16
//   gen 1 (prefill_attn_kernel.cuh):    cp.async page gather + mma.sync, head_dim 64 / 128, any block_size
// Roofline: tensor-bound; FLOPs = 4 * nq * D * sum_i (prefix_i * L_i + L_i (L_i + 1) / 2).
#include <stdlib.h>

#include "prefill_attn_kernel.cuh"
#include "prefill_attn_tc_kernel.cuh"

namespace sllm {

template <typename T, int D>
static int launch_prefill_paged(const void* q, const void* k_cache, const void* v_cache, void* o, const int32_t* start_locs,
                                const int32_t* chunk_lens, float scale, int num_seqs, int max_chunk_len, int nq, int nkv,
                                int64_t qs, const PfPagedKV& pk, cudaStream_t stream) {
    const size_t smem = (size_t)PF_BQ * D * 2 + 2 * 2 * (size_t)PF_BK * D * 2;
    static unsigned long long configured = 0;
    if (first_use_on_this_device(configured)) {
        cudaFuncSetAttribute(prefill_attn_kernel<T, D, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    }
    dim3 grid(cdiv(max_chunk_len, PF_BQ), nq, num_seqs);
    prefill_attn_kernel<T, D, true><<<grid, PF_THREADS, smem, stream>>>((const T*)q, (const T*)k_cache, (const T*)v_cache, (T*)o,
                                                                       start_locs, chunk_lens, scale * 1.4426950408889634f, nq,
                                                                       nkv, qs, 0, 0, pk);
    return check_launch("prefill_attention_paged");
}

static bool tc_prefill_paged_supported(int head_dim, int block_size, int64_t num_tokens, int64_t cache_rows) {
    return head_dim == PT_D && block_size == PT_PAGE && num_tokens > 0 && num_tokens < (1LL << 31) &&
           cache_rows < (1LL << 31) && get_tensor_map_encoder() != nullptr;      // TMA coordinates are int32
}

static int launch_prefill_paged_tc(const void* q, const void* k_cache, const void* v_cache, void* o, const int32_t* start_locs,
                                   const int32_t* chunk_lens, float scale_log2e, int num_seqs, int max_chunk_len,
                                   int64_t num_tokens, int nq, int nkv, int64_t qs, int64_t cache_rows, const PtPaged& pg,
                                   sllm_dtype_t dtype, cudaStream_t stream) {
    CUtensorMap qmap, kmap, vmap;
    SLLM_REQUIRE(pt_map(&qmap, q, (uint64_t)num_tokens, nq * PT_D, qs, PT_BQ, dtype) &&
                 pt_map(&kmap, k_cache, (uint64_t)cache_rows, PT_D, PT_D, PT_PAGE, dtype) &&
                 pt_map(&vmap, v_cache, (uint64_t)cache_rows, PT_D, PT_D, PT_PAGE, dtype),
                 "prefill_attention_paged: cuTensorMapEncodeTiled failed");
    PtParams p;
    p.o = o; p.start_locs = start_locs; p.seq_lens = chunk_lens; p.scale_log2e = scale_log2e; p.nq = nq; p.nkv = nkv;
    dim3 grid((max_chunk_len + PT_BQ - 1) / PT_BQ, nq, num_seqs);
    if (dtype == SLLM_F16) {
        static unsigned long long c = 0;
        if (first_use_on_this_device(c)) cudaFuncSetAttribute(prefill_attn_tc_kernel<__half, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, PT_SMEM_BYTES);
        prefill_attn_tc_kernel<__half, true><<<grid, PT_THREADS, PT_SMEM_BYTES, stream>>>(qmap, kmap, vmap, p, pg);
    } else {
        static unsigned long long c = 0;
        if (first_use_on_this_device(c)) cudaFuncSetAttribute(prefill_attn_tc_kernel<__nv_bfloat16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, PT_SMEM_BYTES);
        prefill_attn_tc_kernel<__nv_bfloat16, true><<<grid, PT_THREADS, PT_SMEM_BYTES, stream>>>(qmap, kmap, vmap, p, pg);
    }
    return check_launch("prefill_attention_paged(wgmma)");
}

}  // namespace sllm

using namespace sllm;

extern "C" int sllm_prefill_attention_paged(const void* q, const void* k_cache, const void* v_cache, void* o,
                                            const int32_t* block_table, const int32_t* seq_ids,
                                            const int32_t* prefill_seq_start_locs, const int32_t* prefill_seq_lens,
                                            const int32_t* prefill_prefix_lens, float softmax_scale, int num_prefill_seqs,
                                            int max_prefill_len, int64_t num_prefill_tokens, int cur_layer, int num_layers,
                                            int nq, int nkv, int block_size, int head_dim, int max_blocks_per_seq,
                                            int64_t num_blocks, int64_t q_row_stride, sllm_dtype_t dtype, sllm_stream_t stream) {
    SLLM_REQUIRE(num_prefill_seqs >= 0 && max_prefill_len >= 0, "prefill_attention_paged: negative sizes");
    if (num_prefill_seqs == 0 || max_prefill_len == 0) return 0;
    SLLM_REQUIRE(q && k_cache && v_cache && o && block_table && seq_ids && prefill_seq_start_locs && prefill_seq_lens &&
                 prefill_prefix_lens, "prefill_attention_paged: null pointer");
    SLLM_REQUIRE(head_dim == 64 || head_dim == 128, "prefill_attention_paged: head_dim %d not supported (64, 128)", head_dim);
    SLLM_REQUIRE(nkv > 0 && nq % nkv == 0, "prefill_attention_paged: nq %d not a multiple of nkv %d", nq, nkv);
    SLLM_REQUIRE(q_row_stride >= (int64_t)nq * head_dim && q_row_stride % 8 == 0, "prefill_attention_paged: bad q row stride");
    SLLM_REQUIRE(block_size > 0 && num_layers > 0 && cur_layer >= 0 && cur_layer < num_layers && max_blocks_per_seq > 0 && num_blocks > 0,
                 "prefill_attention_paged: bad cache geometry (layer %d of %d)", cur_layer, num_layers);
    cudaStream_t st = (cudaStream_t)stream;
    // SLLM_PREFILL_ATTN_GEN=1 forces the cp.async/mma.sync kernel (A/B measurements), like sllm_prefill_attention
    const char* gen_env = getenv("SLLM_PREFILL_ATTN_GEN");
    const int gen = (gen_env && gen_env[0] == '1') ? 1 : (gen_env && gen_env[0] == '2') ? 2 : 0;
    const int64_t cache_rows = num_blocks * num_layers * nkv * block_size;
    if (gen != 1 && dtype <= SLLM_BF16 && tc_prefill_paged_supported(head_dim, block_size, num_prefill_tokens, cache_rows)) {
        PtPaged pg{block_table, seq_ids, prefill_prefix_lens, cur_layer, num_layers, max_blocks_per_seq};
        return launch_prefill_paged_tc(q, k_cache, v_cache, o, prefill_seq_start_locs, prefill_seq_lens,
                                       softmax_scale * 1.4426950408889634f, num_prefill_seqs, max_prefill_len, num_prefill_tokens,
                                       nq, nkv, q_row_stride, cache_rows, pg, dtype, st);
    }
    SLLM_REQUIRE(gen != 2, "prefill_attention_paged: SLLM_PREFILL_ATTN_GEN=2 but the shape is not covered by the wgmma kernel");
    PfPagedKV pk{block_table, seq_ids, prefill_prefix_lens, cur_layer, num_layers, block_size, max_blocks_per_seq};
    if (head_dim == 128) { SLLM_DISPATCH_DTYPE(dtype, return (launch_prefill_paged<T, 128>(q, k_cache, v_cache, o, prefill_seq_start_locs, prefill_seq_lens, softmax_scale, num_prefill_seqs, max_prefill_len, nq, nkv, q_row_stride, pk, st))); }
    else { SLLM_DISPATCH_DTYPE(dtype, return (launch_prefill_paged<T, 64>(q, k_cache, v_cache, o, prefill_seq_start_locs, prefill_seq_lens, softmax_scale, num_prefill_seqs, max_prefill_len, nq, nkv, q_row_stride, pk, st))); }
    return 0;
}
