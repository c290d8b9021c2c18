// Causal varlen prefill attention, generation 2 (TMA + wgmma): host side of the packed-k/v variant.  The kernel is
// prefill_attn_tc_kernel.cuh; reference being replaced: swiftllm/worker/kernels/prefill_attn.py:9-139 and the
// flash_attn_varlen_func call at swiftllm/worker/layers/transformer_layer.py:86-96.
#include <mutex>
#include <unordered_map>

#include "prefill_attn_tc_kernel.cuh"

namespace sllm {

// ------------------------------------------------------------------ host side
namespace {
std::mutex g_pt_mutex;
struct PtKey {
    const void* ptr; uint64_t rows; int cols; int dt; int64_t stride;
    bool operator==(const PtKey& o) const { return ptr == o.ptr && rows == o.rows && cols == o.cols && dt == o.dt && stride == o.stride; }
};
struct PtKeyHash { size_t operator()(const PtKey& k) const { return std::hash<const void*>()(k.ptr) ^ (k.rows * 1315423911u) ^ (size_t)(k.cols * 31 + k.dt) ^ ((size_t)k.stride << 7); } };
std::unordered_map<PtKey, CUtensorMap, PtKeyHash> g_pt_maps;
}  // namespace

// 2-D map over a [rows, cols] 16-bit tensor with `row_stride` elements between rows, boxes of (64 cols x box_rows), SWIZZLE_128B
// (cached per (pointer, geometry); also used by prefill_attn_paged.cu for the paged caches)
bool pt_map(CUtensorMap* out, const void* ptr, uint64_t rows, int cols, int64_t row_stride, int box_rows, sllm_dtype_t dt) {
    PtKey key{ptr, rows, cols * 1024 + box_rows, (int)dt, row_stride};
    {
        std::lock_guard<std::mutex> lk(g_pt_mutex);
        auto it = g_pt_maps.find(key);
        if (it != g_pt_maps.end()) { *out = it->second; return true; }
    }
    TensorMapEncodeFn enc = get_tensor_map_encoder();
    if (!enc) return false;
    cuuint64_t dims[2] = {(cuuint64_t)cols, rows};
    cuuint64_t strides[1] = {(cuuint64_t)row_stride * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)box_rows}, es[2] = {1, 1};
    CUresult r = enc(out, dt == SLLM_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr),
                     dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return false;
    std::lock_guard<std::mutex> lk(g_pt_mutex);
    if (g_pt_maps.size() > 4096) g_pt_maps.clear();
    g_pt_maps[key] = *out;
    return true;
}

bool tc_prefill_supported(int head_dim, int64_t num_tokens) {
    return head_dim == PT_D && num_tokens > 0 && num_tokens < (1LL << 31) && get_tensor_map_encoder() != nullptr;
}

int launch_prefill_tc(const void* q, const void* k, const void* v, void* o, const int32_t* start_locs, const int32_t* seq_lens,
                      float scale_log2e, int num_seqs, int max_len, int64_t num_tokens, int nq, int nkv, int64_t qs, int64_t ks,
                      int64_t vs, sllm_dtype_t dtype, cudaStream_t stream) {
    CUtensorMap qmap, kmap, vmap;
    SLLM_REQUIRE(pt_map(&qmap, q, (uint64_t)num_tokens, nq * PT_D, qs, PT_BQ, dtype) &&
                 pt_map(&kmap, k, (uint64_t)num_tokens, nkv * PT_D, ks, PT_BK, dtype) &&
                 pt_map(&vmap, v, (uint64_t)num_tokens, nkv * PT_D, vs, PT_BK, dtype),
                 "prefill_attention: cuTensorMapEncodeTiled failed");
    PtParams p;
    p.o = o; p.start_locs = start_locs; p.seq_lens = seq_lens; p.scale_log2e = scale_log2e; p.nq = nq; p.nkv = nkv;
    dim3 grid((max_len + PT_BQ - 1) / PT_BQ, nq, num_seqs);
    if (dtype == SLLM_F16) {
        static unsigned long long c = 0;
        if (first_use_on_this_device(c)) cudaFuncSetAttribute(prefill_attn_tc_kernel<__half, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, PT_SMEM_BYTES);
        prefill_attn_tc_kernel<__half, false><<<grid, PT_THREADS, PT_SMEM_BYTES, stream>>>(qmap, kmap, vmap, p, PtPaged{});
    } else {
        static unsigned long long c = 0;
        if (first_use_on_this_device(c)) cudaFuncSetAttribute(prefill_attn_tc_kernel<__nv_bfloat16, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, PT_SMEM_BYTES);
        prefill_attn_tc_kernel<__nv_bfloat16, false><<<grid, PT_THREADS, PT_SMEM_BYTES, stream>>>(qmap, kmap, vmap, p, PtPaged{});
    }
    return check_launch("prefill_attention(wgmma)");
}

}  // namespace sllm
