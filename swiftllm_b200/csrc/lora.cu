// Multi-LoRA: per-request low-rank adapters added to a projection's output, next to the library GEMM that computes it.
// Semantics (restated in numpy by tests/lora_oracle.py), at a site with 16-bit input x [T, K], GEMM output y [T, N], for row t
// of a tile whose slot a has A [S * R, K] (S stacked slices), B [N, R] and scale s:
//   shrink   u[t, j] = round16(sum_k x[t, k] * A[j, k]), fp32 accumulation in an order fixed by K alone (never by the tile, the
//            batch or the other rows), so u is a function of the row and the adapter only;
//   expand   y[t, n] = round16(float(y[t, n]) + s * sum_j u[t, sl(n) * R + j] * B[n, j]): the inner sum in fp32, then one fp32
//            multiply by s, one fp32 add and one rounding to nearest even.  sl(n) is the slice of column n ([0, n1), [n1, n2),
//            [n2, N)); a slice whose bit is clear in slice_mask[a] is not written, nor is any row outside every tile.
// Work list: int32 triples (first row, rows, slot) built by the host from runs of equal slot; tiles with rows outside [1, 64],
// a slot outside [0, max_loras) or rows past num_rows are skipped.  Empty tiles (rows 0) pad a CUDA graph's fixed tile count.
//
// Layout.  Both kernels are memory-bound mma.sync m16n8k16 loops that load their fragments straight from global memory: a lane
// loads 16 (shrink) or 8 (expand) contiguous bytes of one row of each operand and the two operands use the same permutation of
// k inside a 32- (16-) element chunk, so every product x[t, k] * A[j, k] meets its partner and no shared-memory staging is needed
// (each loaded fragment is consumed in registers by the warp that loaded it).
//   shrink   grid (tiles, S * R / 16): a CTA computes 16 columns of u for its tile's rows.  Its 8 warps take the 32-wide k-chunks
//            c = warp, warp + 8, ... (a split fixed by K), and the 8 fp32 partials are summed in warp order through shared memory,
//            then rounded once.  Split-K without workspace or atomics, and decode tiles still spread over S * R / 16 CTAs.
//   expand   grid (tiles, ceil(N / 128)): 4 warps of 32 columns each; the epilogue reads y, adds, rounds and writes, so every
//            element of y is written by exactly one thread.
// Algorithmic bytes per launch: shrink 2 * (rows * K + tiles * S * R * K + rows * S * R); expand 2 * (2 * rows * N + tiles * N * R
// + rows * S * R).
#include "mma_helpers.cuh"

namespace sllm {
namespace {

constexpr int kTileRows = 64;                       // TM: rows of one tile (4 m16 fragments)
constexpr int kShrinkWarps = 8;
constexpr int kShrinkCols = 16;                     // u columns per shrink CTA (two n8 fragments)
constexpr int kExpandWarps = 4;
constexpr int kExpandCols = 32 * kExpandWarps;      // y columns per expand CTA

__device__ __forceinline__ uint4 ldg16(const void* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ uint2 ldg8(const void* p) { return __ldg(reinterpret_cast<const uint2*>(p)); }

struct Tile {
    int row0, rows, slot;
};

// the tile of this CTA, or rows == 0 when it is skipped
__device__ __forceinline__ Tile load_tile(const int32_t* tiles, int64_t num_rows, const int32_t* slice_mask, int max_loras,
                                          int& mask) {
    const int32_t* t = tiles + 3 * (int64_t)blockIdx.x;
    Tile tl{t[0], t[1], t[2]};
    mask = 0;
    if (tl.rows < 1 || tl.rows > kTileRows || tl.row0 < 0 || tl.row0 + (int64_t)tl.rows > num_rows || tl.slot < 0 ||
        tl.slot >= max_loras)
        return Tile{0, 0, 0};
    mask = slice_mask[tl.slot];
    if (mask == 0) tl.rows = 0;
    return tl;
}

// MT m16 fragments of rows (1 for a tile of up to 16 rows, 4 otherwise); rows past the tile are zeros and never stored
template <typename T, int MT>
__device__ __forceinline__ void shrink_body(const T* __restrict__ x, int64_t ldx, int K, const T* __restrict__ a, const Tile& tl,
                                            float (&part)[kShrinkWarps][kTileRows][kShrinkCols]) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
    float acc[MT][2][4];
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int n = 0; n < 2; ++n)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[m][n][i] = 0.f;
    const T* a0 = a + (int64_t)g * K + 8 * c;           // n fragment 0: u column g, fragment 1: column g + 8
    const T* a1 = a0 + 8 * (int64_t)K;
    const T* xr[MT][2];
    bool ok[MT][2];
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = 16 * m + 8 * h + g;
            ok[m][h] = r < tl.rows;
            xr[m][h] = x + (int64_t)(tl.row0 + (ok[m][h] ? r : 0)) * ldx + 8 * c;
        }
    const int chunks = K / 32;
#pragma unroll 2
    for (int kc = warp; kc < chunks; kc += kShrinkWarps) {
        const int k = 32 * kc;
        const uint4 b0 = ldg16(a0 + k), b1 = ldg16(a1 + k);
        uint4 xv[MT][2];
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int h = 0; h < 2; ++h) xv[m][h] = ok[m][h] ? ldg16(xr[m][h] + k) : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int m = 0; m < MT; ++m) {
            const uint32_t lo[4] = {xv[m][0].x, xv[m][1].x, xv[m][0].y, xv[m][1].y};
            const uint32_t hi[4] = {xv[m][0].z, xv[m][1].z, xv[m][0].w, xv[m][1].w};
            mma_16816<T>(acc[m][0], lo, b0.x, b0.y);
            mma_16816<T>(acc[m][0], hi, b0.z, b0.w);
            mma_16816<T>(acc[m][1], lo, b1.x, b1.y);
            mma_16816<T>(acc[m][1], hi, b1.z, b1.w);
        }
    }
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int n = 0; n < 2; ++n) {
            const int r = 16 * m + g, col = 8 * n + 2 * c;
            part[warp][r][col] = acc[m][n][0];
            part[warp][r][col + 1] = acc[m][n][1];
            part[warp][r + 8][col] = acc[m][n][2];
            part[warp][r + 8][col + 1] = acc[m][n][3];
        }
}

template <typename T>
__global__ void __launch_bounds__(32 * kShrinkWarps) lora_shrink_kernel(
    const T* __restrict__ x, int64_t ldx, int64_t num_rows, int K, T* __restrict__ u, int64_t ldu, const T* __restrict__ lora_a,
    int64_t a_slot_stride, const int32_t* __restrict__ tiles, const int32_t* __restrict__ slice_mask, int max_loras) {
    __shared__ float part[kShrinkWarps][kTileRows][kShrinkCols];
    int mask;
    const Tile tl = load_tile(tiles, num_rows, slice_mask, max_loras, mask);
    if (tl.rows == 0) return;
    const int n0 = kShrinkCols * blockIdx.y;
    const T* a = lora_a + tl.slot * a_slot_stride + (int64_t)n0 * K;
    if (tl.rows <= 16)
        shrink_body<T, 1>(x, ldx, K, a, tl, part);
    else
        shrink_body<T, kTileRows / 16>(x, ldx, K, a, tl, part);
    __syncthreads();
    for (int i = threadIdx.x; i < tl.rows * kShrinkCols; i += blockDim.x) {
        const int r = i / kShrinkCols, col = i % kShrinkCols;
        float s = part[0][r][col];
#pragma unroll
        for (int w = 1; w < kShrinkWarps; ++w) s += part[w][r][col];
        u[(tl.row0 + r) * ldu + n0 + col] = Traits<T>::from_f(s);
    }
}

template <typename T>
__global__ void __launch_bounds__(32 * kExpandWarps) lora_expand_kernel(
    T* __restrict__ y, int64_t ldy, int64_t num_rows, int N, const T* __restrict__ u, int64_t ldu, const T* __restrict__ lora_b,
    int64_t b_slot_stride, int R, int n1, int n2, const int32_t* __restrict__ tiles, const int32_t* __restrict__ slice_mask,
    const float* __restrict__ scales, int max_loras) {
    int mask;
    const Tile tl = load_tile(tiles, num_rows, slice_mask, max_loras, mask);
    if (tl.rows == 0) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, c = lane & 3;
    const float s = scales[tl.slot];
    const T* b = lora_b + tl.slot * b_slot_stride;
    const int mt = (tl.rows + 15) / 16;
    for (int f = 0; f < 4; ++f) {
        const int n0 = kExpandCols * blockIdx.y + 32 * warp + 8 * f;
        if (n0 >= N) break;
        const int sl = n0 < n1 ? 0 : (n0 < n2 ? 1 : 2);
        if (!((mask >> sl) & 1)) continue;
        uint2 bf[4];                                        // the column's R <= 64 weights: four k16 fragments
        const T* bp = b + (int64_t)(n0 + g) * R + 4 * c;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) bf[kk] = 16 * kk < R ? ldg8(bp + 16 * kk) : make_uint2(0, 0);
        for (int m = 0; m < mt; ++m) {
            const int r0 = 16 * m + g, r1 = r0 + 8;
            const bool ok0 = r0 < tl.rows, ok1 = r1 < tl.rows;
            const T* u0 = u + (int64_t)(tl.row0 + (ok0 ? r0 : 0)) * ldu + sl * R + 4 * c;
            const T* u1 = u + (int64_t)(tl.row0 + (ok1 ? r1 : 0)) * ldu + sl * R + 4 * c;
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                if (16 * kk >= R) break;
                const uint2 x0 = ok0 ? ldg8(u0 + 16 * kk) : make_uint2(0, 0);
                const uint2 x1 = ok1 ? ldg8(u1 + 16 * kk) : make_uint2(0, 0);
                const uint32_t af[4] = {x0.x, x1.x, x0.y, x1.y};
                mma_16816<T>(acc, af, bf[kk].x, bf[kk].y);
            }
            const int col = n0 + 2 * c;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (!(h ? ok1 : ok0)) continue;
                using T2 = typename Traits<T>::T2;
                T2* p = reinterpret_cast<T2*>(y + (int64_t)(tl.row0 + (h ? r1 : r0)) * ldy + col);
                const float2 v = Traits<T>::to_f2(*p);
                *p = Traits<T>::from_f2(make_float2(__fadd_rn(v.x, __fmul_rn(s, acc[2 * h])),
                                                    __fadd_rn(v.y, __fmul_rn(s, acc[2 * h + 1]))));
            }
        }
    }
}

bool aligned(const void* p, int bytes) { return ((uintptr_t)p % bytes) == 0; }

}  // namespace
}  // namespace sllm

extern "C" int sllm_lora_shrink(const void* x, int64_t x_row_stride, int64_t num_rows, int in_features, void* u,
                                int64_t u_row_stride, const void* lora_a, int64_t a_slot_stride, int u_cols, const int32_t* tiles,
                                int64_t num_tiles, const int32_t* slice_mask, int max_loras, sllm_dtype_t dtype,
                                sllm_stream_t stream) {
    using namespace sllm;
    SLLM_REQUIRE(dtype == SLLM_F16 || dtype == SLLM_BF16, "lora_shrink: unsupported dtype tag %d", (int)dtype);
    SLLM_REQUIRE(num_rows >= 0 && num_rows <= INT32_MAX, "lora_shrink: num_rows %lld out of range", (long long)num_rows);
    SLLM_REQUIRE(in_features > 0 && in_features % 32 == 0, "lora_shrink: in_features must be a positive multiple of 32, got %d",
                 in_features);
    SLLM_REQUIRE(x_row_stride >= in_features && x_row_stride % 8 == 0,
                 "lora_shrink: x_row_stride %lld must be >= in_features %d and a multiple of 8", (long long)x_row_stride,
                 in_features);
    SLLM_REQUIRE(u_cols > 0 && u_cols % kShrinkCols == 0 && u_cols <= 3 * 64,
                 "lora_shrink: u_cols must be a multiple of 16 in [16, 192], got %d", u_cols);
    SLLM_REQUIRE(u_row_stride >= u_cols, "lora_shrink: u_row_stride %lld < u_cols %d", (long long)u_row_stride, u_cols);
    SLLM_REQUIRE(a_slot_stride >= (int64_t)u_cols * in_features && a_slot_stride % 8 == 0,
                 "lora_shrink: a_slot_stride %lld must be >= u_cols * in_features and a multiple of 8", (long long)a_slot_stride);
    SLLM_REQUIRE(max_loras > 0, "lora_shrink: max_loras must be positive, got %d", max_loras);
    SLLM_REQUIRE(num_tiles >= 0 && num_tiles <= INT32_MAX, "lora_shrink: num_tiles %lld out of range", (long long)num_tiles);
    if (num_tiles == 0) return 0;
    SLLM_REQUIRE(x && u && lora_a && tiles && slice_mask, "lora_shrink: null pointer");
    SLLM_REQUIRE(aligned(x, 16) && aligned(lora_a, 16), "lora_shrink: x and lora_a must be 16-byte aligned");
    const dim3 grid((unsigned)num_tiles, (unsigned)(u_cols / kShrinkCols));
    SLLM_DISPATCH_DTYPE(dtype, {
        lora_shrink_kernel<T><<<grid, 32 * kShrinkWarps, 0, (cudaStream_t)stream>>>(
            (const T*)x, x_row_stride, num_rows, in_features, (T*)u, u_row_stride, (const T*)lora_a, a_slot_stride, tiles,
            slice_mask, max_loras);
        return check_launch("lora_shrink");
    });
}

extern "C" int sllm_lora_expand(void* y, int64_t y_row_stride, int64_t num_rows, int out_features, const void* u,
                                int64_t u_row_stride, const void* lora_b, int64_t b_slot_stride, int rank, int slice1, int slice2,
                                const int32_t* tiles, int64_t num_tiles, const int32_t* slice_mask, const float* scales,
                                int max_loras, sllm_dtype_t dtype, sllm_stream_t stream) {
    using namespace sllm;
    SLLM_REQUIRE(dtype == SLLM_F16 || dtype == SLLM_BF16, "lora_expand: unsupported dtype tag %d", (int)dtype);
    SLLM_REQUIRE(num_rows >= 0 && num_rows <= INT32_MAX, "lora_expand: num_rows %lld out of range", (long long)num_rows);
    SLLM_REQUIRE(out_features > 0 && out_features % 8 == 0 && (out_features + kExpandCols - 1) / kExpandCols <= 65535,
                 "lora_expand: out_features must be a positive multiple of 8 below 2^23, got %d", out_features);
    SLLM_REQUIRE(y_row_stride >= out_features && y_row_stride % 2 == 0,
                 "lora_expand: y_row_stride %lld must be >= out_features %d and even", (long long)y_row_stride, out_features);
    SLLM_REQUIRE(rank > 0 && rank % 16 == 0 && rank <= 64, "lora_expand: rank must be 16, 32, 48 or 64, got %d", rank);
    SLLM_REQUIRE(slice1 >= 0 && slice1 <= slice2 && slice2 <= out_features && slice1 % 8 == 0 && slice2 % 8 == 0,
                 "lora_expand: slice ends %d, %d must be multiples of 8 with 0 <= slice1 <= slice2 <= out_features", slice1,
                 slice2);
    const int slices = 1 + (slice1 < out_features) + (slice2 < out_features);
    SLLM_REQUIRE(u_row_stride >= (int64_t)slices * rank && u_row_stride % 4 == 0,
                 "lora_expand: u_row_stride %lld must cover %d slices of rank %d and be a multiple of 4", (long long)u_row_stride,
                 slices, rank);
    SLLM_REQUIRE(b_slot_stride >= (int64_t)out_features * rank && b_slot_stride % 4 == 0,
                 "lora_expand: b_slot_stride %lld must be >= out_features * rank and a multiple of 4", (long long)b_slot_stride);
    SLLM_REQUIRE(max_loras > 0, "lora_expand: max_loras must be positive, got %d", max_loras);
    SLLM_REQUIRE(num_tiles >= 0 && num_tiles <= INT32_MAX, "lora_expand: num_tiles %lld out of range", (long long)num_tiles);
    if (num_tiles == 0) return 0;
    SLLM_REQUIRE(y && u && lora_b && tiles && slice_mask && scales, "lora_expand: null pointer");
    SLLM_REQUIRE(aligned(y, 4) && aligned(u, 8) && aligned(lora_b, 8), "lora_expand: y, u and lora_b must be 4-, 8- and 8-byte aligned");
    const dim3 grid((unsigned)num_tiles, (unsigned)((out_features + kExpandCols - 1) / kExpandCols));
    SLLM_DISPATCH_DTYPE(dtype, {
        lora_expand_kernel<T><<<grid, 32 * kExpandWarps, 0, (cudaStream_t)stream>>>(
            (T*)y, y_row_stride, num_rows, out_features, (const T*)u, u_row_stride, (const T*)lora_b, b_slot_stride, rank, slice1,
            slice2, tiles, slice_mask, scales, max_loras);
        return check_launch("lora_expand");
    });
}
