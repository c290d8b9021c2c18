// Shared helpers for the sm_90a data-plane kernels.
#pragma once

#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/swiftllm_b200.h"

namespace sllm {

// ---------------------------------------------------------------- errors
void set_error(const char* fmt, ...);
int check_launch(const char* what);   // cudaGetLastError -> error code + message
// Kernel generation forced by the environment variable `env_var`: "1" forces generation 1 (A/B measurements, debugging), "2"
// makes a shape generation 2 does not serve an error, anything else 0 (generation 2 wherever it serves the shape).  Re-read on
// every call, so tests can toggle it.
int forced_generation(const char* env_var);

#define SLLM_REQUIRE(cond, ...)            \
    do {                                   \
        if (!(cond)) {                     \
            ::sllm::set_error(__VA_ARGS__); \
            return 1;                      \
        }                                  \
    } while (0)

// ---------------------------------------------------------------- dtype traits
template <typename T> struct Traits;
template <> struct Traits<__half> {
    using T2 = __half2;
    static __device__ __forceinline__ float2 to_f2(T2 v) { return __half22float2(v); }
    static __device__ __forceinline__ T2 from_f2(float2 v) { return __float22half2_rn(v); }
    static __device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
    static __device__ __forceinline__ __half from_f(float v) { return __float2half_rn(v); }
};
template <> struct Traits<__nv_bfloat16> {
    using T2 = __nv_bfloat162;
    static __device__ __forceinline__ float2 to_f2(T2 v) { return __bfloat1622float2(v); }
    static __device__ __forceinline__ T2 from_f2(float2 v) { return __float22bfloat162_rn(v); }
    static __device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }
    static __device__ __forceinline__ __nv_bfloat16 from_f(float v) { return __float2bfloat16_rn(v); }
};

// 16-byte vector of 8 half/bf16 values
template <typename T> struct alignas(16) Vec8 {
    typename Traits<T>::T2 v[4];
};

template <typename T> __device__ __forceinline__ Vec8<T> ld_vec8(const T* p) {
    uint4 u = *reinterpret_cast<const uint4*>(p);
    return *reinterpret_cast<Vec8<T>*>(&u);
}
template <typename T> __device__ __forceinline__ void st_vec8(T* p, const Vec8<T>& v) {
    *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(&v);
}
// streaming (read-once) 16-byte load that does not allocate in L1
template <typename T> __device__ __forceinline__ Vec8<T> ld_vec8_stream(const T* p) {
    uint4 u;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(p));
    return *reinterpret_cast<Vec8<T>*>(&u);
}

// shared-memory address of a generic pointer (operand of cp.async / ldmatrix / mbarrier / TMA / wgmma descriptors)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---------------------------------------------------------------- add + RMSNorm row epilogue
// One CTA per token row of `nvec` 16-byte vectors (row_threads threads), the rounding order of rmsnorm.py:39-65.  rmsnorm_kernel
// and the three exchange kernels build their rows from these, which is what keeps x_out bit-identical across them.

template <typename T> __device__ __forceinline__ void add_sum_sq(float& ss, const Vec8<T>& a) {
#pragma unroll
    for (int j = 0; j < 4; j++) { float2 f = Traits<T>::to_f2(a.v[j]); ss += f.x * f.x + f.y * f.y; }
}
// a = h(sum + r) for one vector: stored back to the residual at rr, stashed for the normalise pass, added to the sum of squares
template <typename T> __device__ __forceinline__ void add_residual(const Vec8<T>& sum, T* rr, uint4* stash, float& ss) {
    Vec8<T> a, b = ld_vec8(rr);
#pragma unroll
    for (int j = 0; j < 4; j++) a.v[j] = __hadd2_rn(sum.v[j], b.v[j]);
    st_vec8(rr, a);
    *stash = *reinterpret_cast<uint4*>(&a);
    add_sum_sq(ss, a);
}
// 1 / rms of the row from every thread's warp_sum of its sum of squares.  red[] holds one float per warp; every thread adds it in
// the same order -> identical rstd.  A caller that reuses red[] for another row synchronises before calling again.  hidden and eps
// by reference: an exchange kernel then reads them from its parameter struct after the barrier, which keeps its schedule.
__device__ __forceinline__ float row_rstd(float warp_ss, float* red, const int& hidden, const float& eps) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    if (lane == 0) red[warp] = warp_ss;
    __syncthreads();
    float total = 0.f;
    for (int w = 0; w < nwarps; w++) total += red[w];
    return 1.0f / sqrtf(total / (float)hidden + eps);
}
// o = (a * rstd) * w, one rounding.  `a` may live in shared memory (read after w is loaded); o is an out-parameter because a
// returned Vec8 compiles rmsnorm_kernel to a different schedule.
template <typename T> __device__ __forceinline__ void rms_scale(Vec8<T>& o, const Vec8<T>& a, float rstd, const T* w) {
    using TT = Traits<T>;
    Vec8<T> g8 = ld_vec8(w);
#pragma unroll
    for (int j = 0; j < 4; j++) {
        float2 f = TT::to_f2(a.v[j]), g = TT::to_f2(g8.v[j]);
        o.v[j] = TT::from_f2(make_float2((f.x * rstd) * g.x, (f.y * rstd) * g.y));
    }
}
// threads per row of nvec vectors: one vector per thread up to 512, whole warps
static inline int row_threads(int nvec) {
    const int threads = nvec >= 512 ? 512 : (nvec >= 256 ? 256 : ((nvec + 31) / 32) * 32);
    return threads < 32 ? 32 : threads;
}

static inline int cdiv(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// ---------------------------------------------------------------- elementwise formulas
// h(up * h(silu(f(gate)))) of 8 values: silu in fp32 (IEEE division), rounded to the storage dtype before the product
template <typename T> __device__ __forceinline__ Vec8<T> silu_mul8(const Vec8<T>& up, const Vec8<T>& gate) {
    using TT = Traits<T>;
    Vec8<T> o;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        float2 g = TT::to_f2(gate.v[j]);
        g.x = g.x / (1.0f + expf(-g.x));
        g.y = g.y / (1.0f + expf(-g.y));
        o.v[j] = __hmul2_rn(up.v[j], TT::from_f2(g));
    }
    return o;
}
// Rotary embedding of one 8-wide chunk x0 of a head's first half and its partner x1 in the second half:
// o0 = x0·c − x1·s, o1 = x0·s + x1·c, every product and sum rounded to the storage dtype (the *_rn intrinsics forbid FMA
// contraction), as rotary_emb.py:32-41 evaluates under the Triton interpreter.
template <typename T>
__device__ __forceinline__ void rotate8(Vec8<T>& o0, Vec8<T>& o1, const Vec8<T>& x0, const Vec8<T>& x1, const Vec8<T>& c,
                                        const Vec8<T>& s) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
        o0.v[j] = __hsub2_rn(__hmul2_rn(x0.v[j], c.v[j]), __hmul2_rn(x1.v[j], s.v[j]));
        o1.v[j] = __hadd2_rn(__hmul2_rn(x0.v[j], s.v[j]), __hmul2_rn(x1.v[j], c.v[j]));
    }
}

// ---------------------------------------------------------------- per-device one-time state (a process may drive several GPUs)
static inline int current_device() {
    int d = 0;
    cudaGetDevice(&d);
    return d;
}
int num_sms();   // multiprocessors of the current device, cached

// ---------------------------------------------------------------- dynamic shared-memory limit
// A kernel's launches may use 48 KB of shared memory, static and dynamic together; past that the kernel's dynamic shared-memory
// limit, a per-device attribute, must first be raised.  Every launcher with dynamic shared memory calls
// fit_dynamic_smem<Kernel>(bytes, its name) before the launch.  `covered` is, per kernel and device, the dynamic size its launches
// may use as things stand: 0 until the slow path (host.cu) has read the kernel's static size from the compiled kernel, then 48 KB
// minus that, and after a raise the raised limit.  It only grows, so a launch it covers costs no driver call and no lock.  The
// slow path must not run under stream capture: the decode graphs' warm-up launches every kernel of their shapes eagerly first.
int raise_dynamic_smem(const void* kernel, size_t bytes, int& covered, const char* who);
template <auto Kernel> inline int fit_dynamic_smem(size_t bytes, const char* who) {
    static int covered[64];
    int& c = covered[current_device() & 63];
    if ((int64_t)bytes <= __atomic_load_n(&c, __ATOMIC_RELAXED)) return 0;
    return raise_dynamic_smem(reinterpret_cast<const void*>(Kernel), bytes, c, who);
}

// dispatch on the dtype tag
#define SLLM_DISPATCH_DTYPE(dtype, ...)                                     \
    do {                                                                    \
        if ((dtype) == SLLM_F16) { using T = __half; __VA_ARGS__; }         \
        else if ((dtype) == SLLM_BF16) { using T = __nv_bfloat16; __VA_ARGS__; } \
        else { ::sllm::set_error("unknown dtype tag %d", (int)(dtype)); return 1; } \
    } while (0)

}  // namespace sllm
