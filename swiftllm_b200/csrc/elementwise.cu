// HBM-bound elementwise kernels: RMSNorm, fused add+RMSNorm (also quantizing its output to e4m3), rotary embedding,
// SiLU-and-mul.  All are 128-bit vectorised (8 half/bf16 values per load/store), coalesced, and follow the rounding
// order of the reference Triton kernels (SURVEY.md Appendix A; oracle/kernels.py restates them):
//   rmsnorm.py:5-24, :39-65   rotary_emb.py:7-41   silu_and_mul.py:5-23
// Algorithmic bytes (s = 2): rmsnorm 2*T*H*s + H*s, fused 4*T*H*s + H*s, fused + quantize 3*T*H*s + T*H + 4*T + H*s (x,
// residual read and written, e4m3 out, scales, weight), rotary 2*T*(nq+nkv)*D*s + T*D*s, silu_and_mul 3*T*F*s.
// The RMSNorm row epilogue (add_residual / row_rstd / rms_scale, common.cuh) is the exchange kernels' too.
#include <type_traits>

#include "fp8.cuh"

namespace sllm {

// ------------------------------------------------------------------ RMSNorm
// One CTA per token row.  VPT > 0: the row is exactly blockDim * VPT 16-byte vectors and every thread keeps its VPT
// vectors in registers, with all loads issued before the first use (several independent 16-byte requests in flight per
// thread: the kernel is latency-bound otherwise; a row is read from HBM exactly once).  VPT == 0: generic row length, the
// (post-add) row is staged in shared memory instead.
// QUANT (with FUSED_ADD): the normalised row is not stored in 16 bits but quantized to e4m3 (fp8.cuh) into xq, its scale into
// scales[t].  redmax is an array of its own: placed behind red[] it changes the quantizing instances' code.
template <typename T, bool FUSED_ADD, int VPT, bool QUANT>
__global__ void __launch_bounds__(512) rmsnorm_kernel(std::conditional_t<QUANT, const T*, T*> __restrict__ x,
                                                      T* __restrict__ residual, const T* __restrict__ weight, float eps,
                                                      int hidden, uint8_t* __restrict__ xq, float* __restrict__ scales) {
    extern __shared__ uint4 row_smem[];
    __shared__ float red[16], redmax[QUANT ? 16 : 1];
    const int64_t t = blockIdx.x;
    const auto xr = x + t * hidden;
    T* rr = FUSED_ADD ? residual + t * hidden : nullptr;
    const int nvec = hidden >> 3;
    constexpr int NV = VPT > 0 ? VPT : 1;
    Vec8<T> regs[NV];

    float ss = 0.f;
    if (VPT > 0) {
        Vec8<T> rv[NV];
#pragma unroll
        for (int v = 0; v < NV; v++) regs[v] = ld_vec8(xr + 8 * (threadIdx.x + v * blockDim.x));
        if (FUSED_ADD) {
#pragma unroll
            for (int v = 0; v < NV; v++) rv[v] = ld_vec8(rr + 8 * (threadIdx.x + v * blockDim.x));
        }
#pragma unroll
        for (int v = 0; v < NV; v++) {
            if (FUSED_ADD) {
#pragma unroll
                for (int j = 0; j < 4; j++) regs[v].v[j] = __hadd2_rn(regs[v].v[j], rv[v].v[j]);   // s = h(x + r): storage-dtype add
                st_vec8(rr + 8 * (threadIdx.x + v * blockDim.x), regs[v]);
            }
            add_sum_sq(ss, regs[v]);
        }
    } else {
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
            Vec8<T> a = ld_vec8(xr + 8 * i);
            if (FUSED_ADD) {
                add_residual(a, rr + 8 * i, &row_smem[i], ss);
            } else {
                row_smem[i] = *reinterpret_cast<uint4*>(&a);
                add_sum_sq(ss, a);
            }
        }
    }
    const float rstd = row_rstd(warp_sum(ss), red, hidden, eps);
    if constexpr (!QUANT) {
        if (VPT > 0) {
#pragma unroll
            for (int v = 0; v < NV; v++) {
                const int i = threadIdx.x + v * blockDim.x;
                Vec8<T> o;
                rms_scale(o, regs[v], rstd, weight + 8 * i);
                st_vec8(xr + 8 * i, o);
            }
        } else {
            for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
                Vec8<T> o;
                rms_scale(o, *reinterpret_cast<Vec8<T>*>(&row_smem[i]), rstd, weight + 8 * i);
                st_vec8(xr + 8 * i, o);
            }
        }
    } else {
        uint8_t* qr = xq + t * hidden;
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
}

// The instance of rmsnorm_kernel for a row of `hidden` elements, for all three RMSNorm entries.  xq and scales: QUANT only.
template <typename T, bool FUSED, bool QUANT>
static int launch_rmsnorm(const void* x, void* residual, const void* weight, float eps, int64_t T_, int hidden, void* xq,
                          float* scales, cudaStream_t stream) {
    if (T_ == 0) return 0;
    using X = std::conditional_t<QUANT, const T*, T*>;
    const int nvec = hidden / 8;
    const char* what = QUANT ? "fused_add_rmsnorm_quant_fp8" : (FUSED ? "fused_add_rmsnorm" : "rmsnorm");
    // rows of 4 x 128 .. 4 x 256 vectors (hidden 4096 .. 8192): 4 vectors per thread, 128 .. 256 threads, no shared-memory staging
    if (nvec % 4 == 0 && (nvec / 4) % 32 == 0 && nvec / 4 >= 64 && nvec / 4 <= 256) {
        rmsnorm_kernel<T, FUSED, 4, QUANT><<<(unsigned)T_, nvec / 4, 0, stream>>>((X)x, (T*)residual, (const T*)weight, eps, hidden,
                                                                                  (uint8_t*)xq, scales);
        return check_launch(what);
    }
    if (nvec % 2 == 0 && (nvec / 2) % 32 == 0 && nvec / 2 <= 256) {
        rmsnorm_kernel<T, FUSED, 2, QUANT><<<(unsigned)T_, nvec / 2, 0, stream>>>((X)x, (T*)residual, (const T*)weight, eps, hidden,
                                                                                  (uint8_t*)xq, scales);
        return check_launch(what);
    }
    const int threads = row_threads(nvec);
    const size_t smem = (size_t)nvec * sizeof(uint4);
    if (int e = fit_dynamic_smem<rmsnorm_kernel<T, FUSED, 0, QUANT>>(smem, what)) return e;
    rmsnorm_kernel<T, FUSED, 0, QUANT><<<(unsigned)T_, threads, smem, stream>>>((X)x, (T*)residual, (const T*)weight, eps, hidden,
                                                                                (uint8_t*)xq, scales);
    return check_launch(what);
}

// ------------------------------------------------------------------ rotary embedding
// One thread per (token, head, 8-wide chunk of the first half): rotates x[d..d+8) with x[d+D/2..d+D/2+8) (rotate8, common.cuh).
template <typename T>
__global__ void __launch_bounds__(256) rotary_kernel(T* __restrict__ q, T* __restrict__ k, const T* __restrict__ cosb,
                                                     const T* __restrict__ sinb, int64_t total, int nq, int nkv,
                                                     int head_dim, int64_t q_stride, int64_t k_stride) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int chunks = head_dim >> 4;             // 8-wide chunks in half a head
    const int heads = nq + nkv;
    const int c = (int)(idx % chunks);
    const int hh = (int)((idx / chunks) % heads);
    const int64_t t = idx / ((int64_t)chunks * heads);
    T* base = hh < nq ? q + t * q_stride + hh * head_dim : k + t * k_stride + (hh - nq) * head_dim;
    const int half = head_dim >> 1;
    Vec8<T> x0 = ld_vec8(base + 8 * c), x1 = ld_vec8(base + half + 8 * c);
    Vec8<T> cv = ld_vec8(cosb + t * half + 8 * c), sv = ld_vec8(sinb + t * half + 8 * c);
    Vec8<T> o0, o1;
    rotate8(o0, o1, x0, x1, cv, sv);
    st_vec8(base + 8 * c, o0);
    st_vec8(base + half + 8 * c, o1);
}

// ------------------------------------------------------------------ SiLU and mul
// x [T, 2F] = [up | gate]; x[:, :F] = silu_mul8(up, gate).  One thread per 2 x 8 outputs (4 independent 16-byte loads in flight).
template <typename T>
__global__ void __launch_bounds__(256) silu_and_mul_kernel(T* __restrict__ x, int64_t total_vec, int64_t F) {
    const int64_t idx0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 2;
    if (idx0 >= total_vec) return;
    const int64_t vec_per_row = F >> 3;
    const bool two = idx0 + 1 < total_vec;
    T* up_p[2]; Vec8<T> up[2], gate[2];
#pragma unroll
    for (int u = 0; u < 2; u++) {
        const int64_t idx = idx0 + (two ? u : 0);
        up_p[u] = x + (idx / vec_per_row) * 2 * F + 8 * (idx % vec_per_row);
    }
#pragma unroll
    for (int u = 0; u < 2; u++) { up[u] = ld_vec8(up_p[u]); gate[u] = ld_vec8_stream(up_p[u] + F); }
#pragma unroll
    for (int u = 0; u < 2; u++) {
        if (u == 1 && !two) break;
        st_vec8(up_p[u], silu_mul8(up[u], gate[u]));
    }
}

}  // namespace sllm

using namespace sllm;

extern "C" {

int sllm_rmsnorm_inplace(void* x, const void* weight, float eps, int64_t num_tokens, int hidden, sllm_dtype_t dtype,
                         sllm_stream_t stream) {
    SLLM_REQUIRE(num_tokens >= 0 && hidden > 0 && hidden % 8 == 0, "rmsnorm: hidden (%d) must be a positive multiple of 8", hidden);
    SLLM_REQUIRE(num_tokens == 0 || (x && weight), "rmsnorm: null pointer");
    SLLM_DISPATCH_DTYPE(dtype, return (launch_rmsnorm<T, false, false>(x, nullptr, weight, eps, num_tokens, hidden, nullptr, nullptr,
                                                                    (cudaStream_t)stream)));
    return 0;
}

int sllm_fused_add_rmsnorm_inplace(void* x, void* residual, const void* weight, float eps, int64_t num_tokens,
                                   int hidden, sllm_dtype_t dtype, sllm_stream_t stream) {
    SLLM_REQUIRE(num_tokens >= 0 && hidden > 0 && hidden % 8 == 0, "fused_add_rmsnorm: hidden (%d) must be a positive multiple of 8", hidden);
    SLLM_REQUIRE(num_tokens == 0 || (x && residual && weight), "fused_add_rmsnorm: null pointer");
    SLLM_DISPATCH_DTYPE(dtype, return (launch_rmsnorm<T, true, false>(x, residual, weight, eps, num_tokens, hidden, nullptr, nullptr,
                                                                   (cudaStream_t)stream)));
    return 0;
}

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
    SLLM_DISPATCH_DTYPE(dtype, return (launch_rmsnorm<T, true, true>(x, residual, weight, eps, num_tokens, hidden, xq, scales,
                                                                      (cudaStream_t)stream)));
    return 0;
}

int sllm_rotary_embedding_inplace(void* q, void* k, const void* cosb, const void* sinb, int64_t num_tokens,
                                  int num_q_heads, int num_kv_heads, int head_dim, int64_t q_row_stride,
                                  int64_t k_row_stride, sllm_dtype_t dtype, sllm_stream_t stream) {
    SLLM_REQUIRE(head_dim > 0 && head_dim % 16 == 0, "rotary: head_dim (%d) must be a multiple of 16", head_dim);
    SLLM_REQUIRE(q_row_stride >= (int64_t)num_q_heads * head_dim && k_row_stride >= (int64_t)num_kv_heads * head_dim &&
                 q_row_stride % 8 == 0 && k_row_stride % 8 == 0, "rotary: bad row strides (%lld, %lld)",
                 (long long)q_row_stride, (long long)k_row_stride);
    SLLM_REQUIRE(num_q_heads > 0 && num_kv_heads > 0 && num_tokens >= 0, "rotary: bad shape");
    if (num_tokens == 0) return 0;
    SLLM_REQUIRE(q && k && cosb && sinb, "rotary: null pointer");
    const int64_t total = num_tokens * (int64_t)(num_q_heads + num_kv_heads) * (head_dim / 16);
    const int threads = 256;
    const unsigned blocks = (unsigned)((total + threads - 1) / threads);
    SLLM_DISPATCH_DTYPE(dtype, (rotary_kernel<T><<<blocks, threads, 0, (cudaStream_t)stream>>>(
                                   (T*)q, (T*)k, (const T*)cosb, (const T*)sinb, total, num_q_heads, num_kv_heads, head_dim,
                                   q_row_stride, k_row_stride)));
    return check_launch("rotary_embedding");
}

int sllm_silu_and_mul_inplace(void* x, int64_t num_tokens, int64_t F, sllm_dtype_t dtype, sllm_stream_t stream) {
    SLLM_REQUIRE(F > 0 && F % 8 == 0 && num_tokens >= 0, "silu_and_mul: ffn_inter_dim (%lld) must be a positive multiple of 8", (long long)F);
    if (num_tokens == 0) return 0;
    SLLM_REQUIRE(x, "silu_and_mul: null pointer");
    const int64_t total = num_tokens * (F / 8);
    const int threads = 256;
    const unsigned blocks = (unsigned)(((total + 1) / 2 + threads - 1) / threads);
    SLLM_DISPATCH_DTYPE(dtype, (silu_and_mul_kernel<T><<<blocks, threads, 0, (cudaStream_t)stream>>>((T*)x, total, F)));
    return check_launch("silu_and_mul");
}

}  // extern "C"
