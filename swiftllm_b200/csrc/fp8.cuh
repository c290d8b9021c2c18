// Per-row e4m3 quantization (DESIGN.md §8o; tests/fp8_oracle.py restates it), for one row y of the storage dtype:
//   s   = fmaxf(amax(|y|) / 448.f, 0x1p-126f)        fp32, IEEE division; an all-zero row gets s = 2^-126 and q = 0
//   q_j = e4m3_rn_satfinite(y_j / s)                   fp32 IEEE division, then cvt.rn.satfinite.e4m3x2.f32
// so y_j ~= q_j * s.  One CTA per row: the block amax is one warp_max per warp and a fixed-order pass over the warps' maxima.
// Used by rmsnorm_kernel's quantizing instances (elementwise.cu) and the kernels of fp8.cu.
#pragma once

#include <cuda_fp8.h>

#include "common.cuh"

namespace sllm {

constexpr float kE4m3Max = 448.f;

// amax of the row from every thread's local maximum; `red` holds one float per warp, read in warp order -> the same s everywhere
__device__ __forceinline__ float row_scale(float local, float* red) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    local = warp_max(local);
    if (lane == 0) red[warp] = local;
    __syncthreads();
    float m = 0.f;
    for (int w = 0; w < nwarps; w++) m = fmaxf(m, red[w]);
    return fmaxf(__fdiv_rn(m, kE4m3Max), 0x1p-126f);
}

template <typename T> __device__ __forceinline__ float vec_amax(float m, const Vec8<T>& a) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const float2 f = Traits<T>::to_f2(a.v[j]);
        m = fmaxf(m, fmaxf(fabsf(f.x), fabsf(f.y)));
    }
    return m;
}

// 8 e4m3 bytes of y / s, element j at byte j
template <typename T> __device__ __forceinline__ uint2 quant8(const Vec8<T>& a, float s) {
    uint32_t w[2];
#pragma unroll
    for (int h = 0; h < 2; h++) {
        uint32_t lo, hi;
        float2 f = Traits<T>::to_f2(a.v[2 * h]);
        lo = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(f.x, s), __fdiv_rn(f.y, s)), __NV_SATFINITE, __NV_E4M3);
        f = Traits<T>::to_f2(a.v[2 * h + 1]);
        hi = __nv_cvt_float2_to_fp8x2(make_float2(__fdiv_rn(f.x, s), __fdiv_rn(f.y, s)), __NV_SATFINITE, __NV_E4M3);
        w[h] = lo | (hi << 16);
    }
    return make_uint2(w[0], w[1]);
}

__device__ __forceinline__ void st_q8(uint8_t* p, uint2 v) { *reinterpret_cast<uint2*>(p) = v; }

static inline bool aligned(const void* p, int bytes) { return ((uintptr_t)p % bytes) == 0; }

}  // namespace sllm
