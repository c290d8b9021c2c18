// Causal varlen prefill attention: both C entries and the host side of both kernel generations.
//   sllm_prefill_attention         packed q/k/v of the batch (the reference's contract)
//   sllm_prefill_attention_paged   chunked ("prefix-aware") prefill, PAGED = true: the queries of a prompt CHUNK attend to the
//                                  whole prefix + chunk through the paged KV cache
// gen 2 (prefill_attn_tc_kernel.cuh): TMA + wgmma, head_dim 128 (PAGED: block_size 16), fp16/bf16
// gen 1 (prefill_attn_kernel.cuh):    cp.async + mma.sync, head_dim 64 / 128, any block_size; SLLM_PREFILL_ATTN_GEN=1 forces it
//
// Reference: swiftllm/worker/kernels/prefill_attn.py:9-139 (the Triton kernel) and the flash_attn_varlen_func call that stands
// in for it at swiftllm/worker/layers/transformer_layer.py:86-96.  Numerics follow SURVEY.md Appendix A6: S = f32(QK^T) *
// (scale*log2e); online softmax in fp32 with exp2; P rounded to the storage dtype before P.V; o = h(acc / l).
// The sequence END is taken from prefill_seq_lens (never from a cu_seqlens array that includes decode tokens: the reference's
// mixed-batch quirk, SURVEY.md §3.1).
// The reference cannot express a partial prompt (SURVEY.md §8 f-1: its prefill attention only ever sees the packed k/v of the
// batch), which is what SARATHI-style piggybacking (BASELINE.json configs[2]) needs.  The paged definition is the one that
// makes a prompt processed in chunks equal to the same prompt processed at once (oracle/kernels.py:
// prefix_prefill_attention_exact).
// Roofline: tensor-bound; FLOPs = 4 * nq * D * sum_i (prefix_i * L_i + L_i (L_i + 1) / 2)  (prefix_i = 0 when packed).
#include "prefill_attn_kernel.cuh"
#include "prefill_attn_tc_kernel.cuh"

namespace sllm {

// One launch of either entry, filled after its argument checks.
struct PrefillLaunch {
    const void* q; const void* k; const void* v; void* o;        // PAGED: k / v are the paged caches
    const int32_t* start_locs; const int32_t* seq_lens;
    float scale_log2e;
    int num_seqs, max_len;
    int64_t num_tokens;
    int nq, nkv, head_dim;
    int64_t qs;                       // q row stride (elements)
    sllm_dtype_t dtype;
    cudaStream_t stream;
    int64_t ks = 0, vs = 0;           // packed: k / v row strides (elements)
    PfPagedKV paged = {};             // PAGED: where the pages of a sequence are
    int64_t cache_rows = 0;           // PAGED: rows of a cache viewed as [num_blocks * L * nkv * block_size, head_dim]
};

template <bool PAGED> constexpr const char* entry_name =PAGED ? "prefill_attention_paged" : "prefill_attention";

// generation 2: (Q, K, V) tensor maps, cached per (pointer, geometry)
template <typename T, bool PAGED>
static int launch_gen2(const PrefillLaunch& a) {
    CUtensorMap qmap, kmap, vmap;
    bool ok = cached_rows_map(&qmap, a.q, a.dtype, a.num_tokens, a.nq * PT_D, a.qs, PT_BQ);
    if (PAGED)      // the caches as [cache_rows, 128]: one (64 d x 16 token) box per d-half of a page
        ok = ok && cached_rows_map(&kmap, a.k, a.dtype, a.cache_rows, PT_D, PT_D, PT_PAGE) &&
             cached_rows_map(&vmap, a.v, a.dtype, a.cache_rows, PT_D, PT_D, PT_PAGE);
    else            // the packed [tokens, nkv * 128] rows, (64 d x 64 token) boxes
        ok = ok && cached_rows_map(&kmap, a.k, a.dtype, a.num_tokens, a.nkv * PT_D, a.ks, PT_BK) &&
             cached_rows_map(&vmap, a.v, a.dtype, a.num_tokens, a.nkv * PT_D, a.vs, PT_BK);
    SLLM_REQUIRE(ok, "%s: cuTensorMapEncodeTiled failed", entry_name<PAGED>);
    PtParams p;
    p.o = a.o; p.start_locs = a.start_locs; p.seq_lens = a.seq_lens; p.scale_log2e = a.scale_log2e; p.nq = a.nq; p.nkv = a.nkv;
    const PfPagedKV& pk = a.paged;
    const PtPaged pg = PAGED ? PtPaged{pk.block_table, pk.seq_ids, pk.prefix_lens, pk.cur_layer, pk.num_layers, pk.max_blocks_per_seq}
                             : PtPaged{};
    if (int e = fit_dynamic_smem<prefill_attn_tc_kernel<T, PAGED>>(PT_SMEM_BYTES, entry_name<PAGED>)) return e;
    dim3 grid(cdiv(a.max_len, PT_BQ), a.nq, a.num_seqs);
    prefill_attn_tc_kernel<T, PAGED><<<grid, PT_THREADS, PT_SMEM_BYTES, a.stream>>>(qmap, kmap, vmap, p, pg);
    return check_launch(PAGED ? "prefill_attention_paged(wgmma)" : "prefill_attention(wgmma)");
}

template <typename T, int D, bool PAGED>
static int launch_gen1(const PrefillLaunch& a) {
    const size_t smem = (size_t)PF_BQ * D * 2 + 2 * 2 * (size_t)PF_BK * D * 2;
    if (int e = fit_dynamic_smem<prefill_attn_kernel<T, D, PAGED>>(smem, entry_name<PAGED>)) return e;
    dim3 grid(cdiv(a.max_len, PF_BQ), a.nq, a.num_seqs);
    prefill_attn_kernel<T, D, PAGED><<<grid, PF_THREADS, smem, a.stream>>>((const T*)a.q, (const T*)a.k, (const T*)a.v, (T*)a.o,
                                                                           a.start_locs, a.seq_lens, a.scale_log2e, a.nq, a.nkv,
                                                                           a.qs, a.ks, a.vs, a.paged);
    return check_launch(entry_name<PAGED>);
}

template <bool PAGED>
static bool gen2_serves(const PrefillLaunch& a) {
    return a.head_dim == PT_D && (!PAGED || a.paged.block_size == PT_PAGE) && a.num_tokens > 0 && a.num_tokens < (1LL << 31) &&
           (!PAGED || a.cache_rows < (1LL << 31)) && get_tensor_map_encoder() != nullptr;      // TMA coordinates are int32
}

template <bool PAGED>
static int launch_prefill(const PrefillLaunch& a) {
    const int gen = forced_generation("SLLM_PREFILL_ATTN_GEN");
    if (gen != 1 && a.dtype <= SLLM_BF16 && gen2_serves<PAGED>(a))
        return a.dtype == SLLM_F16 ? launch_gen2<__half, PAGED>(a) : launch_gen2<__nv_bfloat16, PAGED>(a);
    SLLM_REQUIRE(gen != 2, "%s: SLLM_PREFILL_ATTN_GEN=2 but the shape is not covered by the wgmma kernel", entry_name<PAGED>);
    if (a.head_dim == 128) { SLLM_DISPATCH_DTYPE(a.dtype, return (launch_gen1<T, 128, PAGED>(a))); }
    else { SLLM_DISPATCH_DTYPE(a.dtype, return (launch_gen1<T, 64, PAGED>(a))); }
    return 0;
}

}  // namespace sllm

using namespace sllm;

extern "C" int sllm_prefill_attention(const void* q, const void* k, const void* v, void* o, const int32_t* start_locs,
                                      const int32_t* seq_lens, float softmax_scale, int num_prefill_seqs,
                                      int max_prefill_len, int64_t num_prefill_tokens, int nq, int nkv, int head_dim,
                                      int64_t q_row_stride, int64_t k_row_stride, int64_t v_row_stride,
                                      sllm_dtype_t dtype, sllm_stream_t stream) {
    SLLM_REQUIRE(num_prefill_seqs >= 0 && max_prefill_len >= 0, "prefill_attention: negative sizes");
    if (num_prefill_seqs == 0 || max_prefill_len == 0) return 0;
    SLLM_REQUIRE(q && k && v && o && start_locs && seq_lens, "prefill_attention: null pointer");
    SLLM_REQUIRE(head_dim == 64 || head_dim == 128, "prefill_attention: head_dim %d not supported (64, 128)", head_dim);
    SLLM_REQUIRE(nkv > 0 && nq % nkv == 0, "prefill_attention: nq %d not a multiple of nkv %d", nq, nkv);
    SLLM_REQUIRE(q_row_stride >= (int64_t)nq * head_dim && k_row_stride >= (int64_t)nkv * head_dim && v_row_stride >= (int64_t)nkv * head_dim &&
                 q_row_stride % 8 == 0 && k_row_stride % 8 == 0 && v_row_stride % 8 == 0, "prefill_attention: bad row strides");
    PrefillLaunch a{q, k, v, o, start_locs, seq_lens, softmax_scale * 1.4426950408889634f, num_prefill_seqs, max_prefill_len,
                    num_prefill_tokens, nq, nkv, head_dim, q_row_stride, dtype, (cudaStream_t)stream};
    a.ks = k_row_stride; a.vs = v_row_stride;
    return launch_prefill<false>(a);
}

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
    PrefillLaunch a{q, k_cache, v_cache, o, prefill_seq_start_locs, prefill_seq_lens, softmax_scale * 1.4426950408889634f,
                    num_prefill_seqs, max_prefill_len, num_prefill_tokens, nq, nkv, head_dim, q_row_stride, dtype, (cudaStream_t)stream};
    a.paged = PfPagedKV{block_table, seq_ids, prefill_prefix_lens, cur_layer, num_layers, block_size, max_blocks_per_seq};
    a.cache_rows = num_blocks * num_layers * nkv * block_size;
    return launch_prefill<true>(a);
}
