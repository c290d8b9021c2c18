// Hopper (sm_90a) primitives used by the TMA + wgmma kernels: mbarrier, TMA tensor loads, wgmma shared-memory
// descriptors and the warpgroup MMA itself (fp32 accumulators in registers).  Inline PTX only.
// Descriptor bit layouts follow the PTX ISA "warpgroup-level matrix shared memory layout" section (matrix descriptor
// format for wgmma).
#pragma once
#include <cuda.h>

#include <type_traits>

#include "common.cuh"

namespace sllm {
namespace tc {

// ------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}\n"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// non-blocking probe (try_wait may suspend the thread for a while; a poller that serves several queues must not)
__device__ __forceinline__ bool mbar_test_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile("{\n .reg .pred p;\n mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}\n"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// Spin with a watchdog: a protocol bug must surface as a trapped kernel (CUDA error), never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > (1u << 26)) { printf("sllm: mbarrier watchdog (block %d thread %d bar %u parity %u)\n", blockIdx.x, threadIdx.x, bar, parity); __trap(); }
    }
}

// ------------------------------------------------------------------ proxies / fences
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(m) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}

// ------------------------------------------------------------------ wgmma descriptors
// Shared-memory matrix descriptor, SWIZZLE_128B (1 KiB-aligned atoms).  K-major operand: rows of 128 B (64 x 16-bit
// along K), 8-row atoms `sbo` bytes apart (LBO unused); a K step of 16 elements advances the start address by 32 B.
// MN-major operand: atoms of 8 K-rows x 64 MN-elements; `lbo` = byte distance between MN-adjacent atoms, `sbo` = byte
// distance between K-adjacent atoms.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    d |= (uint64_t)1 << 62;      // layout type: SWIZZLE_128B
    return d;
}

// ------------------------------------------------------------------ wgmma (issued by all 128 threads of a warpgroup)
// Accumulator fragment of an m64nN tile, thread t = 32 w + l of the warpgroup: d[4i + e] holds row 16 w + l / 4 + 8 (e >> 1)
// and column 8 i + 2 (l % 4) + (e & 1).  The register A fragment of m64k16 uses the same (row, column) pairs for its
// four 32-bit registers (columns 0..7 then 8..15), so an accumulator tile converts to A operands register for register.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D (+)= A * B with A and B in shared memory (_ss) or A in registers (_rs); TA / TB = 1: that operand is MN-major
// (transposed), 16-bit types only
template <typename T, int TA, int TB>
__device__ __forceinline__ void wgmma_m64n8k16_ss(float (&d)[4], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    if constexpr (std::is_same<T, __half>::value)
        asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %6, 0;\n wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 "
                     "{%0,%1,%2,%3}, %4, %5, p, 1, 1, %7, %8;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB) : "memory");
    else
        asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %6, 0;\n wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 "
                     "{%0,%1,%2,%3}, %4, %5, p, 1, 1, %7, %8;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                     : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB) : "memory");
}

template <typename T, int TA, int TB>
__device__ __forceinline__ void wgmma_m64n16k16_ss(float (&d)[8], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    if constexpr (std::is_same<T, __half>::value)
        asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %10, 0;\n wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
                     "{%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                     : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB) : "memory");
    else
        asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %10, 0;\n wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
                     "{%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                     : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB) : "memory");
}

template <typename T, int TA, int TB>
__device__ __forceinline__ void wgmma_m64n32k16_ss(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    if constexpr (std::is_same<T, __half>::value)
        asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %18, 0;\n wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
                     "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                       "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                     : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB) : "memory");
    else
        asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %18, 0;\n wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
                     "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                       "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                     : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB) : "memory");
}

template <typename T, int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16_ss(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    if constexpr (std::is_same<T, __half>::value)
        asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %34, 0;\n wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
                     "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                     : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB) : "memory");
    else
        asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %34, 0;\n wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
                     "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                     : "l"(adesc), "l"(bdesc), "r"(scale_d), "n"(TA), "n"(TB) : "memory");
}

template <typename T, int TB>
__device__ __forceinline__ void wgmma_m64n128k16_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t scale_d) {
    if constexpr (std::is_same<T, __half>::value)
        asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %69, 0;\n wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
                     "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, %70;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d), "n"(TB) : "memory");
    else
        asm volatile("{\n .reg .pred p;\n setp.ne.b32 p, %69, 0;\n wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
                     "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, %70;\n}\n"
                     : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(scale_d), "n"(TB) : "memory");
}


__device__ __forceinline__ float fast_exp2_tc(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// non-blocking half of a producer / consumer named barrier: counts this thread's arrival towards `nthreads`
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ------------------------------------------------------------------ host: tensor-map encoding through the runtime's driver entry point
typedef CUresult (*TensorMapEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                      const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
TensorMapEncodeFn get_tensor_map_encoder();     // nullptr if unavailable (host.cu)

// Every tensor map of the library (host.cu): 16-bit elements, SWIZZLE_128B, L2_256B promotion, no OOB fill, unit element
// strides.  dims[0] is the contiguous dimension; byte_strides[i] is the distance between consecutive indices of dims[i + 1].
// False if the encoder is unavailable or rejects the geometry.
bool encode_tma_map(CUtensorMap* out, const void* ptr, sllm_dtype_t dt, int rank, const cuuint64_t* dims,
                    const cuuint64_t* byte_strides, const cuuint32_t* box);
// The same, memoised on all arguments (a KV cache keeps its address, so its maps are encoded once)
bool cached_tma_map(CUtensorMap* out, const void* ptr, sllm_dtype_t dt, int rank, const cuuint64_t* dims,
                    const cuuint64_t* byte_strides, const cuuint32_t* box);
// A [rows, cols] tensor with rows `row_stride` elements apart, boxes of (64 cols x box_rows), cached
inline bool cached_rows_map(CUtensorMap* out, const void* ptr, sllm_dtype_t dt, uint64_t rows, uint64_t cols, int64_t row_stride,
                            uint32_t box_rows) {
    const cuuint64_t dims[2] = {cols, rows}, strides[1] = {(cuuint64_t)row_stride * 2};
    const cuuint32_t box[2] = {64, box_rows};
    return cached_tma_map(out, ptr, dt, 2, dims, strides, box);
}

}  // namespace tc
}  // namespace sllm
