// Library plumbing (errors, device check, kernel-generation switch, tensor maps) and the host-side block swapper.
#include <stdarg.h>
#include <stdlib.h>

#include <mutex>
#include <string_view>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "tc_helpers.cuh"

namespace sllm {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_error("%s: %s", what, cudaGetErrorString(e));
        return (int)e;
    }
    return 0;
}

int forced_generation(const char* env_var) {
    const char* e = getenv(env_var);
    return (e && e[0] == '1') ? 1 : (e && e[0] == '2') ? 2 : 0;
}

int num_sms() {
    static int sms[64] = {0};
    const int dev = current_device() & 63;
    if (sms[dev] == 0) {
        int n = 0;
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        sms[dev] = n > 0 ? n : 132;
    }
    return sms[dev];
}

int raise_dynamic_smem(const void* kernel, size_t bytes, int& covered, const char* who) {
    static std::mutex m;             // two threads raising one kernel's limit: the larger value must be the one that stays
    std::lock_guard<std::mutex> lk(m);
    int limit = covered;
    cudaError_t e = cudaSuccess;
    if (limit == 0) {
        cudaFuncAttributes fa;
        e = cudaFuncGetAttributes(&fa, kernel);
        limit = 48 * 1024 - (int)fa.sharedSizeBytes;
    }
    if (e == cudaSuccess && (int64_t)bytes > limit) {
        e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
        limit = (int)bytes;
    }
    if (e != cudaSuccess) {
        cudaGetLastError();          // reported here, not by the next launch's check_launch
        set_error("%s: cannot allow %zu bytes of dynamic shared memory: %s", who, bytes, cudaGetErrorString(e));
        return (int)e;
    }
    __atomic_store_n(&covered, limit, __ATOMIC_RELAXED);
    return 0;
}

namespace tc {
// cuTensorMapEncodeTiled through the runtime (no link-time dependency on libcuda)
TensorMapEncodeFn get_tensor_map_encoder() {
    static TensorMapEncodeFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (TensorMapEncodeFn)p;
        cudaGetLastError();
    }
    return fn;
}

bool encode_tma_map(CUtensorMap* out, const void* ptr, sllm_dtype_t dt, int rank, const cuuint64_t* dims,
                    const cuuint64_t* byte_strides, const cuuint32_t* box) {
    TensorMapEncodeFn enc = get_tensor_map_encoder();
    if (!enc) return false;
    const cuuint32_t es[5] = {1, 1, 1, 1, 1};
    return enc(out, dt == SLLM_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr),
               dims, byte_strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

namespace {
struct MapKey {         // every argument of cached_tma_map, unused dimensions zero; compared and hashed as bytes
    const void* ptr; int dt, rank; cuuint64_t dims[5], strides[4]; cuuint32_t box[5], unused;
    std::string_view bytes() const { return std::string_view(reinterpret_cast<const char*>(this), sizeof(*this)); }
    bool operator==(const MapKey& o) const { return bytes() == o.bytes(); }
};
static_assert(std::has_unique_object_representations_v<MapKey>, "MapKey must have no padding bytes");
struct MapKeyHash { size_t operator()(const MapKey& k) const { return std::hash<std::string_view>()(k.bytes()); } };
std::mutex g_map_mutex;
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;
}  // namespace

bool cached_tma_map(CUtensorMap* out, const void* ptr, sllm_dtype_t dt, int rank, const cuuint64_t* dims,
                    const cuuint64_t* byte_strides, const cuuint32_t* box) {
    if (rank < 1 || rank > 5) return false;
    MapKey key{};
    key.ptr = ptr; key.dt = (int)dt; key.rank = rank;
    for (int i = 0; i < rank; i++) {
        key.dims[i] = dims[i]; key.box[i] = box[i];
        if (i > 0) key.strides[i - 1] = byte_strides[i - 1];
    }
    {
        std::lock_guard<std::mutex> lk(g_map_mutex);
        auto it = g_maps.find(key);
        if (it != g_maps.end()) { *out = it->second; return true; }
    }
    if (!encode_tma_map(out, ptr, dt, rank, dims, byte_strides, box)) return false;
    std::lock_guard<std::mutex> lk(g_map_mutex);
    if (g_maps.size() > 4096) g_maps.clear();
    g_maps[key] = *out;
    return true;
}
}  // namespace tc

}  // namespace sllm

extern "C" {

int sllm_abi_version(void) { return SLLM_ABI_VERSION; }

const char* sllm_last_error(void) { return sllm::g_err; }

int sllm_device_check(int device) {
    cudaDeviceProp p;
    cudaError_t e = cudaGetDeviceProperties(&p, device);
    if (e != cudaSuccess) {
        sllm::set_error("cudaGetDeviceProperties(%d): %s", device, cudaGetErrorString(e));
        return (int)e;
    }
    if (p.major != 9) {
        sllm::set_error("device %d is sm_%d%d; this library contains sm_90a code only (no fallback path)",
                        device, p.major, p.minor);
        return 1;
    }
    return 0;
}

// Reference: csrc/src/block_swapping.cpp:22-85.  Same run-coalescing rule (:33-44): a run continues while
// both the source and the target id advance by exactly one.  Differences from the reference, on purpose:
// every cudaMemcpyAsync return code is checked (the reference ignores them, :51-80).
int sllm_swap_blocks(const int64_t* src, const int64_t* dst, int64_t n, int is_swap_in, void* k_cache,
                     void* v_cache, void* k_swap, void* v_swap, int64_t block_bytes, sllm_stream_t stream_) {
    SLLM_REQUIRE(n >= 0 && block_bytes > 0, "swap_blocks: bad sizes n=%lld block_bytes=%lld", (long long)n,
                 (long long)block_bytes);
    SLLM_REQUIRE(n == 0 || (src && dst && k_cache && v_cache && k_swap && v_swap), "swap_blocks: null pointer");
    cudaStream_t stream = (cudaStream_t)stream_;
    int64_t i = 0;
    while (i < n) {
        int64_t j = i + 1;
        while (j < n && src[j] == src[j - 1] + 1 && dst[j] == dst[j - 1] + 1) j++;
        size_t bytes = (size_t)(j - i) * (size_t)block_bytes;
        size_t so = (size_t)src[i] * (size_t)block_bytes, dof = (size_t)dst[i] * (size_t)block_bytes;
        cudaError_t e1, e2;
        if (is_swap_in) {   // CPU swap space -> GPU cache
            e1 = cudaMemcpyAsync((char*)k_cache + dof, (const char*)k_swap + so, bytes, cudaMemcpyHostToDevice, stream);
            e2 = cudaMemcpyAsync((char*)v_cache + dof, (const char*)v_swap + so, bytes, cudaMemcpyHostToDevice, stream);
        } else {            // GPU cache -> CPU swap space
            e1 = cudaMemcpyAsync((char*)k_swap + dof, (const char*)k_cache + so, bytes, cudaMemcpyDeviceToHost, stream);
            e2 = cudaMemcpyAsync((char*)v_swap + dof, (const char*)v_cache + so, bytes, cudaMemcpyDeviceToHost, stream);
        }
        if (e1 != cudaSuccess || e2 != cudaSuccess) {
            sllm::set_error("swap_blocks: cudaMemcpyAsync failed: %s",
                            cudaGetErrorString(e1 != cudaSuccess ? e1 : e2));
            return (int)(e1 != cudaSuccess ? e1 : e2);
        }
        i = j;
    }
    return 0;
}

}  // extern "C"
