// Decode-step fusion of two latency-bound launches: rotary embedding (swiftllm/worker/kernels/rotary_emb.py:44-58) and the
// decode part of the KV-cache store (swiftllm/worker/kernels/kvcache_mgmt.py:50-79), which the reference (and the unfused
// path here) run back to back on the same [Bd, (nq + 2 nkv) * D] rows, 2 x 32 launches per decode step.
// One thread per (token, head, 8-wide chunk of the first half of the head):
//   q heads: rotated in place;   k heads: rotated, written in place AND to their cache slot;   v heads: copied to the cache.
// Same arithmetic as rotary_kernel (elementwise.cu), rotate8 (common.cuh): every product and sum individually rounded
// (bit-exact with the reference's interpreter and the oracle).  Bytes: 2*T*(nq+nkv)*D*s (rotary) + 4*T*nkv*D*s (store) + T*D*s (cos/sin).
#include "common.cuh"

namespace sllm {

template <typename T>
__global__ void __launch_bounds__(256) rotary_store_decode_kernel(
    T* __restrict__ q, T* __restrict__ k, const T* __restrict__ v, const T* __restrict__ cosb, const T* __restrict__ sinb,
    T* __restrict__ k_cache, T* __restrict__ v_cache, const int32_t* __restrict__ block_table,
    const int32_t* __restrict__ seq_ids, const int32_t* __restrict__ seq_lens, int64_t total, int nq, int nkv, int head_dim,
    int64_t q_stride, int64_t k_stride, int64_t v_stride, int cur_layer, int num_layers, int bs, int max_blocks_per_seq) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int chunks = head_dim >> 4;             // 8-wide chunks in half a head
    const int heads = nq + 2 * nkv;
    const int c = (int)(idx % chunks);
    const int hh = (int)((idx / chunks) % heads);
    const int64_t t = idx / ((int64_t)chunks * heads);
    const int half = head_dim >> 1;
    if (hh < nq) {                                // ---- q head: rotate in place
        T* base = q + t * q_stride + hh * head_dim;
        Vec8<T> x0 = ld_vec8(base + 8 * c), x1 = ld_vec8(base + half + 8 * c);
        Vec8<T> cv = ld_vec8(cosb + t * half + 8 * c), sv = ld_vec8(sinb + t * half + 8 * c);
        Vec8<T> o0, o1;
        rotate8(o0, o1, x0, x1, cv, sv);
        st_vec8(base + 8 * c, o0);
        st_vec8(base + half + 8 * c, o1);
        return;
    }
    // ---- k / v head: the new token's slot in the paged cache (kvcache_mgmt.py:63-70: position len - 1)
    const int pos = seq_lens[t] - 1;
    const int64_t blk = block_table[(int64_t)seq_ids[t] * max_blocks_per_seq + pos / bs];
    const bool is_k = hh < nq + nkv;
    const int h = is_k ? hh - nq : hh - nq - nkv;
    const int64_t dst = ((((blk * num_layers + cur_layer) * nkv + h) * bs) + pos % bs) * (int64_t)head_dim;
    if (is_k) {
        T* base = k + t * k_stride + h * head_dim;
        Vec8<T> x0 = ld_vec8(base + 8 * c), x1 = ld_vec8(base + half + 8 * c);
        Vec8<T> cv = ld_vec8(cosb + t * half + 8 * c), sv = ld_vec8(sinb + t * half + 8 * c);
        Vec8<T> o0, o1;
        rotate8(o0, o1, x0, x1, cv, sv);
        st_vec8(base + 8 * c, o0);
        st_vec8(base + half + 8 * c, o1);
        st_vec8(k_cache + dst + 8 * c, o0);
        st_vec8(k_cache + dst + half + 8 * c, o1);
    } else {
        const T* base = v + t * v_stride + h * head_dim;
        st_vec8(v_cache + dst + 8 * c, ld_vec8(base + 8 * c));
        st_vec8(v_cache + dst + half + 8 * c, ld_vec8(base + half + 8 * c));
    }
}

}  // namespace sllm

using namespace sllm;

extern "C" int sllm_rotary_store_kvcache_decode(void* q, void* k, const void* v, const void* cosb, const void* sinb, void* k_cache,
                                                void* v_cache, const int32_t* block_table, const int32_t* seq_ids,
                                                const int32_t* decoding_seq_lens, int num_decoding_seqs, int cur_layer,
                                                int num_layers, int num_q_heads, int num_kv_heads, int block_size, int head_dim,
                                                int max_blocks_per_seq, int64_t q_row_stride, int64_t k_row_stride,
                                                int64_t v_row_stride, sllm_dtype_t dtype, sllm_stream_t stream) {
    SLLM_REQUIRE(head_dim > 0 && head_dim % 16 == 0, "rotary_store: head_dim (%d) must be a multiple of 16", head_dim);
    SLLM_REQUIRE(num_q_heads > 0 && num_kv_heads > 0 && num_decoding_seqs >= 0, "rotary_store: bad shape");
    SLLM_REQUIRE(q_row_stride >= (int64_t)num_q_heads * head_dim && k_row_stride >= (int64_t)num_kv_heads * head_dim &&
                 v_row_stride >= (int64_t)num_kv_heads * head_dim && q_row_stride % 8 == 0 && k_row_stride % 8 == 0 &&
                 v_row_stride % 8 == 0, "rotary_store: bad row strides (%lld, %lld, %lld)", (long long)q_row_stride,
                 (long long)k_row_stride, (long long)v_row_stride);
    SLLM_REQUIRE(block_size > 0 && num_layers > 0 && cur_layer >= 0 && cur_layer < num_layers && max_blocks_per_seq > 0,
                 "rotary_store: bad cache geometry (layer %d of %d)", cur_layer, num_layers);
    if (num_decoding_seqs == 0) return 0;
    SLLM_REQUIRE(q && k && v && cosb && sinb && k_cache && v_cache && block_table && seq_ids && decoding_seq_lens,
                 "rotary_store: null pointer");
    const int64_t total = (int64_t)num_decoding_seqs * (num_q_heads + 2 * num_kv_heads) * (head_dim / 16);
    const int threads = 256;
    const unsigned blocks = (unsigned)((total + threads - 1) / threads);
    SLLM_DISPATCH_DTYPE(dtype, (rotary_store_decode_kernel<T><<<blocks, threads, 0, (cudaStream_t)stream>>>(
                                   (T*)q, (T*)k, (const T*)v, (const T*)cosb, (const T*)sinb, (T*)k_cache, (T*)v_cache, block_table,
                                   seq_ids, decoding_seq_lens, total, num_q_heads, num_kv_heads, head_dim, q_row_stride,
                                   k_row_stride, v_row_stride, cur_layer, num_layers, block_size, max_blocks_per_seq)));
    return check_launch("rotary_store_kvcache_decode");
}
