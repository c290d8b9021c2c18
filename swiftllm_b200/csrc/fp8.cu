// FP8 (e4m3) weights: per-token activation quantization fused into the kernels that produce each GEMM input.  The GEMMs stay
// library calls (torch._scaled_mm, row-wise scales); these kernels write their e4m3 operands and fp32 scales.
// Numerics (DESIGN.md §8o; tests/fp8_oracle.py restates them), for one row y of the storage dtype:
//   s   = fmaxf(amax(|y|) / 448.f, 0x1p-126f)        fp32, IEEE division; an all-zero row gets s = 2^-126 and q = 0
//   q_j = e4m3_rn_satfinite(y_j / s)                   fp32 IEEE division, then cvt.rn.satfinite.e4m3x2.f32
// so y_j ~= q_j * s.  y is exactly the row the unquantized kernel stores:
//   add_rmsnorm_quant_kernel   the fused add+RMSNorm of rmsnorm_kernel<T, true, *> (the residual update included), built from the
//                              same row epilogue (add_residual / row_rstd / rms_scale, common.cuh); the 16-bit row is not stored
//   silu_and_mul_quant_kernel  silu_and_mul_kernel's h(up * h(silu(f(gate)))) of [up | gate]
//   quant_rows_kernel          the given rows (the attention output, an exchange's normalised rows, weights at load)
// One CTA per row in all three: the block amax is one warp_max per warp and a fixed-order pass over the warps' maxima.
// Algorithmic bytes (s = 2): add_rmsnorm_quant 3*T*H*s + T*H + 4*T + H*s (x, residual read and written, e4m3 out, scales, weight);
// silu_and_mul_quant 2*T*F*s + T*F + 4*T; quant_rows R*C*s + R*C + 4*R.
#include <cuda_fp8.h>

#include "common.cuh"

namespace sllm {
namespace {

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

// ------------------------------------------------------------------ add + RMSNorm + quantize
// rmsnorm_kernel<T, true, VPT>'s row (VPT > 0: the row in registers; VPT == 0: staged in shared memory), then the quantized store.
template <typename T, int VPT>
__global__ void __launch_bounds__(512) add_rmsnorm_quant_kernel(const T* __restrict__ x, T* __restrict__ residual,
                                                                const T* __restrict__ weight, float eps, int hidden,
                                                                uint8_t* __restrict__ xq, float* __restrict__ scales) {
    extern __shared__ uint4 row_smem[];
    __shared__ float red[16], redmax[16];
    const int64_t t = blockIdx.x;
    const T* xr = x + t * hidden;
    T* rr = residual + t * hidden;
    uint8_t* qr = xq + t * hidden;
    const int nvec = hidden >> 3;
    constexpr int NV = VPT > 0 ? VPT : 1;
    Vec8<T> regs[NV];

    float ss = 0.f;
    if (VPT > 0) {
        Vec8<T> rv[NV];
#pragma unroll
        for (int v = 0; v < NV; v++) regs[v] = ld_vec8(xr + 8 * (threadIdx.x + v * blockDim.x));
#pragma unroll
        for (int v = 0; v < NV; v++) rv[v] = ld_vec8(rr + 8 * (threadIdx.x + v * blockDim.x));
#pragma unroll
        for (int v = 0; v < NV; v++) {
#pragma unroll
            for (int j = 0; j < 4; j++) regs[v].v[j] = __hadd2_rn(regs[v].v[j], rv[v].v[j]);
            st_vec8(rr + 8 * (threadIdx.x + v * blockDim.x), regs[v]);
            add_sum_sq(ss, regs[v]);
        }
    } else {
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) add_residual(ld_vec8(xr + 8 * i), rr + 8 * i, &row_smem[i], ss);
    }
    const float rstd = row_rstd(warp_sum(ss), red, hidden, eps);
    float m = 0.f;
    if (VPT > 0) {
#pragma unroll
        for (int v = 0; v < NV; v++) {
            Vec8<T> o;
            rms_scale(o, regs[v], rstd, weight + 8 * (threadIdx.x + v * blockDim.x));
            regs[v] = o;
            m = vec_amax(m, o);
        }
    } else {
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            Vec8<T> o;
            rms_scale(o, *reinterpret_cast<Vec8<T>*>(&row_smem[i]), rstd, weight + 8 * i);
            row_smem[i] = *reinterpret_cast<uint4*>(&o);
            m = vec_amax(m, o);
        }
    }
    const float s = row_scale(m, redmax);
    if (VPT > 0) {
#pragma unroll
        for (int v = 0; v < NV; v++) {
            const int i = threadIdx.x + v * blockDim.x;
            st_q8(qr + 8 * i, quant8(regs[v], s));
        }
    } else {
        for (int i = threadIdx.x; i < nvec; i += blockDim.x)
            st_q8(qr + 8 * i, quant8(*reinterpret_cast<Vec8<T>*>(&row_smem[i]), s));
    }
    if (threadIdx.x == 0) scales[t] = s;
}

// ------------------------------------------------------------------ SiLU·mul + quantize
// x [T, >= 2F] = [up | gate] (row stride ldx); out [T, F] e4m3.  The product row is staged in shared memory (F * 2 bytes).
template <typename T>
__global__ void __launch_bounds__(512) silu_and_mul_quant_kernel(const T* __restrict__ x, int64_t ldx, int F,
                                                                 uint8_t* __restrict__ out, float* __restrict__ scales) {
    using TT = Traits<T>;
    extern __shared__ uint4 row_smem[];
    __shared__ float redmax[16];
    const int64_t t = blockIdx.x;
    const T* up_r = x + t * ldx;
    const int nvec = F >> 3;
    float m = 0.f;
#pragma unroll 4
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
        const Vec8<T> up = ld_vec8_stream(up_r + 8 * i), gate = ld_vec8_stream(up_r + F + 8 * i);
        Vec8<T> o;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            float2 g = TT::to_f2(gate.v[j]);
            g.x = g.x / (1.0f + expf(-g.x));
            g.y = g.y / (1.0f + expf(-g.y));
            o.v[j] = __hmul2_rn(up.v[j], TT::from_f2(g));
        }
        row_smem[i] = *reinterpret_cast<uint4*>(&o);
        m = vec_amax(m, o);
    }
    const float s = row_scale(m, redmax);
    uint8_t* qr = out + t * F;
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) st_q8(qr + 8 * i, quant8(*reinterpret_cast<Vec8<T>*>(&row_smem[i]), s));
    if (threadIdx.x == 0) scales[t] = s;
}

// ------------------------------------------------------------------ quantize rows
// x [R, C] with row stride ldx; out [R, C] e4m3.  Two passes over the row: the amax, then the quantized store (the second read
// hits L2 / L1; rows up to a few 10 KB).
template <typename T>
__global__ void __launch_bounds__(512) quant_rows_kernel(const T* __restrict__ x, int64_t ldx, int cols, uint8_t* __restrict__ out,
                                                         float* __restrict__ scales) {
    __shared__ float redmax[16];
    const int64_t t = blockIdx.x;
    const T* xr = x + t * ldx;
    const int nvec = cols >> 3;
    float m = 0.f;
#pragma unroll 4
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) m = vec_amax(m, ld_vec8(xr + 8 * i));
    const float s = row_scale(m, redmax);
    uint8_t* qr = out + t * (int64_t)cols;
#pragma unroll 4
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) st_q8(qr + 8 * i, quant8(ld_vec8(xr + 8 * i), s));
    if (threadIdx.x == 0) scales[t] = s;
}

bool aligned(const void* p, int bytes) { return ((uintptr_t)p % bytes) == 0; }

template <typename T>
int launch_add_rmsnorm_quant(const void* x, void* residual, const void* weight, float eps, int64_t T_, int hidden, void* xq,
                             float* scales, cudaStream_t stream) {
    const int nvec = hidden / 8;
    // the register paths of launch_rmsnorm: hidden 4096 .. 8192 (4 vectors per thread), then up to 4096 (2 per thread)
    if (nvec % 4 == 0 && (nvec / 4) % 32 == 0 && nvec / 4 >= 64 && nvec / 4 <= 256) {
        add_rmsnorm_quant_kernel<T, 4><<<(unsigned)T_, nvec / 4, 0, stream>>>((const T*)x, (T*)residual, (const T*)weight, eps,
                                                                              hidden, (uint8_t*)xq, scales);
        return check_launch("fused_add_rmsnorm_quant_fp8");
    }
    if (nvec % 2 == 0 && (nvec / 2) % 32 == 0 && nvec / 2 <= 256) {
        add_rmsnorm_quant_kernel<T, 2><<<(unsigned)T_, nvec / 2, 0, stream>>>((const T*)x, (T*)residual, (const T*)weight, eps,
                                                                              hidden, (uint8_t*)xq, scales);
        return check_launch("fused_add_rmsnorm_quant_fp8");
    }
    const size_t smem = (size_t)nvec * sizeof(uint4);
    // the 48 KB a kernel may use without raising its limit include its static shared memory: red[16], redmax[16]
    if (smem + 32 * sizeof(float) > 48 * 1024)
        cudaFuncSetAttribute(add_rmsnorm_quant_kernel<T, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    add_rmsnorm_quant_kernel<T, 0><<<(unsigned)T_, row_threads(nvec), smem, stream>>>((const T*)x, (T*)residual, (const T*)weight,
                                                                                      eps, hidden, (uint8_t*)xq, scales);
    return check_launch("fused_add_rmsnorm_quant_fp8");
}

}  // namespace
}  // namespace sllm

using namespace sllm;

extern "C" {

int sllm_fused_add_rmsnorm_quant_fp8(const void* x, void* residual, const void* weight, float eps, int64_t num_tokens, int hidden,
                                     void* xq, float* scales, sllm_dtype_t dtype, sllm_stream_t stream) {
    SLLM_REQUIRE(hidden > 0 && hidden % 16 == 0 && hidden <= (1 << 16),
                 "fused_add_rmsnorm_quant_fp8: hidden (%d) must be a positive multiple of 16 up to 65536", hidden);
    SLLM_REQUIRE(num_tokens >= 0 && num_tokens <= INT32_MAX, "fused_add_rmsnorm_quant_fp8: num_tokens %lld out of range",
                 (long long)num_tokens);
    if (num_tokens == 0) return 0;
    SLLM_REQUIRE(x && residual && weight && xq && scales, "fused_add_rmsnorm_quant_fp8: null pointer");
    SLLM_REQUIRE(aligned(x, 16) && aligned(residual, 16) && aligned(weight, 16) && aligned(xq, 8),
                 "fused_add_rmsnorm_quant_fp8: x, residual and weight must be 16-byte aligned, xq 8-byte aligned");
    SLLM_DISPATCH_DTYPE(dtype, return (launch_add_rmsnorm_quant<T>(x, residual, weight, eps, num_tokens, hidden, xq, scales,
                                                                    (cudaStream_t)stream)));
    return 0;
}

int sllm_silu_and_mul_quant_fp8(const void* x, int64_t x_row_stride, int64_t num_tokens, int64_t F, void* out, float* scales,
                                sllm_dtype_t dtype, sllm_stream_t stream) {
    SLLM_REQUIRE(F > 0 && F % 16 == 0 && F <= (1 << 16), "silu_and_mul_quant_fp8: F (%lld) must be a positive multiple of 16 up to 65536",
                 (long long)F);
    SLLM_REQUIRE(x_row_stride >= 2 * F && x_row_stride % 8 == 0,
                 "silu_and_mul_quant_fp8: x_row_stride %lld must be >= 2 * F and a multiple of 8", (long long)x_row_stride);
    SLLM_REQUIRE(num_tokens >= 0 && num_tokens <= INT32_MAX, "silu_and_mul_quant_fp8: num_tokens %lld out of range",
                 (long long)num_tokens);
    if (num_tokens == 0) return 0;
    SLLM_REQUIRE(x && out && scales, "silu_and_mul_quant_fp8: null pointer");
    SLLM_REQUIRE(aligned(x, 16) && aligned(out, 8), "silu_and_mul_quant_fp8: x must be 16-byte aligned, out 8-byte aligned");
    const int nvec = (int)(F / 8);
    const size_t smem = (size_t)nvec * sizeof(uint4);
    SLLM_DISPATCH_DTYPE(dtype, {
        if (smem + 16 * sizeof(float) > 48 * 1024)     // static shared memory (redmax[16]) counts against the 48 KB
            cudaFuncSetAttribute(silu_and_mul_quant_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        silu_and_mul_quant_kernel<T><<<(unsigned)num_tokens, row_threads(nvec), smem, (cudaStream_t)stream>>>(
            (const T*)x, x_row_stride, (int)F, (uint8_t*)out, scales);
        return check_launch("silu_and_mul_quant_fp8");
    });
}

int sllm_quant_fp8_rows(const void* x, int64_t x_row_stride, int64_t num_rows, int64_t cols, void* out, float* scales,
                        sllm_dtype_t dtype, sllm_stream_t stream) {
    SLLM_REQUIRE(cols > 0 && cols % 16 == 0 && cols <= INT32_MAX, "quant_fp8_rows: cols (%lld) must be a positive multiple of 16",
                 (long long)cols);
    SLLM_REQUIRE(x_row_stride >= cols && x_row_stride % 8 == 0,
                 "quant_fp8_rows: x_row_stride %lld must be >= cols and a multiple of 8", (long long)x_row_stride);
    SLLM_REQUIRE(num_rows >= 0 && num_rows <= INT32_MAX, "quant_fp8_rows: num_rows %lld out of range", (long long)num_rows);
    if (num_rows == 0) return 0;
    SLLM_REQUIRE(x && out && scales, "quant_fp8_rows: null pointer");
    SLLM_REQUIRE(aligned(x, 16) && aligned(out, 8), "quant_fp8_rows: x must be 16-byte aligned, out 8-byte aligned");
    const int threads = row_threads((int)(cols / 8));
    SLLM_DISPATCH_DTYPE(dtype, {
        quant_rows_kernel<T><<<(unsigned)num_rows, threads, 0, (cudaStream_t)stream>>>((const T*)x, x_row_stride, (int)cols,
                                                                                       (uint8_t*)out, scales);
        return check_launch("quant_fp8_rows");
    });
}

}  // extern "C"
