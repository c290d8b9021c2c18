// Library plumbing (errors, device check) and the host-side block swapper.
#include <stdarg.h>

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
