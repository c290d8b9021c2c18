// Causal varlen prefill attention over packed q/k/v: C-ABI entry + launch of the generation 1 kernel
// (prefill_attn_kernel.cuh: cp.async double buffering + mma.sync); generation 2 lives in prefill_attn_tc.cu.
//
// Reference: swiftllm/worker/kernels/prefill_attn.py:9-139 (the Triton kernel) and the flash_attn_varlen_func
// call that stands in for it at swiftllm/worker/layers/transformer_layer.py:86-96.  Numerics follow
// SURVEY.md Appendix A6: S = f32(QK^T) * (scale*log2e); online softmax in fp32 with exp2; P rounded to the
// storage dtype before P.V; o = h(acc / l).
// The sequence END is taken from prefill_seq_lens (never from a cu_seqlens array that includes decode tokens:
// the reference's mixed-batch quirk, SURVEY.md §3.1).
// Roofline: tensor-bound; FLOPs = 4 * nq * D * sum_i L_i (L_i + 1) / 2.
#include <stdlib.h>

#include "prefill_attn_kernel.cuh"

namespace sllm {

template <typename T, int D>
static int launch_prefill(const void* q, const void* k, const void* v, void* o, const int32_t* start_locs,
                          const int32_t* seq_lens, float scale, int num_seqs, int max_len, int nq, int nkv,
                          int64_t qs, int64_t ks, int64_t vs, cudaStream_t stream) {
    const size_t smem = (size_t)PF_BQ * D * 2 + 2 * 2 * (size_t)PF_BK * D * 2;
    static unsigned long long configured = 0;
    if (first_use_on_this_device(configured)) {
        cudaFuncSetAttribute(prefill_attn_kernel<T, D, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    }
    dim3 grid(cdiv(max_len, PF_BQ), nq, num_seqs);
    prefill_attn_kernel<T, D, false><<<grid, PF_THREADS, smem, stream>>>((const T*)q, (const T*)k, (const T*)v, (T*)o, start_locs,
                                                                        seq_lens, scale * 1.4426950408889634f, nq, nkv, qs, ks, vs,
                                                                        PfPagedKV{});
    return check_launch("prefill_attention");
}

// generation 2 (prefill_attn_tc.cu)
bool tc_prefill_supported(int head_dim, int64_t num_tokens);
int launch_prefill_tc(const void* q, const void* k, const void* v, void* o, const int32_t* start_locs, const int32_t* seq_lens,
                      float scale_log2e, int num_seqs, int max_len, int64_t num_tokens, int nq, int nkv, int64_t qs, int64_t ks,
                      int64_t vs, sllm_dtype_t dtype, cudaStream_t stream);

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
    cudaStream_t st = (cudaStream_t)stream;
    // SLLM_PREFILL_ATTN_GEN=1 forces the cp.async/mma.sync kernel (A/B measurements); default: TMA/wgmma for head_dim 128
    const char* gen_env = getenv("SLLM_PREFILL_ATTN_GEN");
    const int gen = (gen_env && gen_env[0] == '1') ? 1 : (gen_env && gen_env[0] == '2') ? 2 : 0;
    if (gen != 1 && dtype <= SLLM_BF16 && tc_prefill_supported(head_dim, num_prefill_tokens))
        return launch_prefill_tc(q, k, v, o, start_locs, seq_lens, softmax_scale * 1.4426950408889634f, num_prefill_seqs,
                                 max_prefill_len, num_prefill_tokens, nq, nkv, q_row_stride, k_row_stride, v_row_stride, dtype, st);
    SLLM_REQUIRE(gen != 2, "prefill_attention: SLLM_PREFILL_ATTN_GEN=2 but the shape is not covered by the wgmma kernel");
    if (head_dim == 128) { SLLM_DISPATCH_DTYPE(dtype, return (launch_prefill<T, 128>(q, k, v, o, start_locs, seq_lens, softmax_scale, num_prefill_seqs, max_prefill_len, nq, nkv, q_row_stride, k_row_stride, v_row_stride, st))); }
    else { SLLM_DISPATCH_DTYPE(dtype, return (launch_prefill<T, 64>(q, k, v, o, start_locs, seq_lens, softmax_scale, num_prefill_seqs, max_prefill_len, nq, nkv, q_row_stride, k_row_stride, v_row_stride, st))); }
    return 0;
}
