// FP8 (e4m3) weights: per-token activation quantization fused into the kernels that produce each GEMM input.  The GEMMs stay
// library calls (torch._scaled_mm, row-wise scales); these kernels write their e4m3 operands and fp32 scales, by the numerics of
// fp8.cuh.  The quantized row y is exactly the row the unquantized kernel stores:
//   rmsnorm_kernel<T, true, VPT, true>  (elementwise.cu) the fused add+RMSNorm, the residual update included; the 16-bit row is
//                                       not stored
//   silu_and_mul_quant_kernel           silu_and_mul_kernel's h(up * h(silu(f(gate)))) of [up | gate]
//   quant_rows_kernel                   the given rows (the attention output, an exchange's normalised rows, weights at load)
// Algorithmic bytes (s = 2): silu_and_mul_quant 2*T*F*s + T*F + 4*T; quant_rows R*C*s + R*C + 4*R.
#include "fp8.cuh"

namespace sllm {
namespace {

// ------------------------------------------------------------------ SiLU·mul + quantize
// x [T, >= 2F] = [up | gate] (row stride ldx); out [T, F] e4m3.  The product row is staged in shared memory (F * 2 bytes).
template <typename T>
__global__ void __launch_bounds__(512) silu_and_mul_quant_kernel(const T* __restrict__ x, int64_t ldx, int F,
                                                                 uint8_t* __restrict__ out, float* __restrict__ scales) {
    extern __shared__ uint4 row_smem[];
    __shared__ float redmax[16];
    const int64_t t = blockIdx.x;
    const T* up_r = x + t * ldx;
    const int nvec = F >> 3;
    float m = 0.f;
#pragma unroll 4
    for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
        const Vec8<T> up = ld_vec8_stream(up_r + 8 * i), gate = ld_vec8_stream(up_r + F + 8 * i);
        Vec8<T> o = silu_mul8(up, gate);
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

}  // namespace
}  // namespace sllm

using namespace sllm;

extern "C" {

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
        if (int e = fit_dynamic_smem<silu_and_mul_quant_kernel<T>>(smem, "silu_and_mul_quant_fp8")) return e;
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
