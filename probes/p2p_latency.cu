// NVLink peer-memory probe (2 GPUs of one box, one process): what the fused TP exchange (csrc/allreduce_norm.cu) is made of.
//   1. flag round trip: GPU0 release-stores an epoch into GPU1's memory, GPU1 (spinning with ld.acquire.sys) echoes it into GPU0's
//      memory -> ns per round trip = 2 x the one-way signal latency that every barrier of the exchange kernel pays;
//   2. peer read bandwidth: one kernel on GPU0 sums a buffer that lives on GPU1 with 16-byte volatile loads (the one-shot path)
//      for sizes from 256 KiB (a decode exchange at TP 8: 32 rows x 8 KiB) to 128 MiB (a prefill exchange);
//   3. peer write bandwidth: 16-byte stores into GPU1's memory (the two-shot path's all-gather half).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O2 -std=c++17 -o probes/build/p2p_latency probes/p2p_latency.cu
// Run on a machine with >= 2 GPUs: probes/build/p2p_latency
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// role 0: for i in 1..iters: store i to peer_flag, wait until my_flag == i.   role 1: wait until my_flag == i, store i to peer_flag.
__global__ void pingpong(uint32_t* my_flag, uint32_t* peer_flag, int iters, int role, long long* cycles) {
    const long long t0 = clock64();
    for (uint32_t i = 1; i <= (uint32_t)iters; i++) {
        if (role == 0) st_release_sys(peer_flag, i);
        uint32_t spins = 0;
        while (ld_acquire_sys(my_flag) < i) { if (++spins > (1u << 28)) { printf("pingpong watchdog (role %d, i %u)\n", role, i); return; } }
        if (role == 1) st_release_sys(peer_flag, i);
    }
    *cycles = clock64() - t0;
}

__global__ void peer_read(const uint4* __restrict__ src, size_t nvec, unsigned long long* sink) {
    unsigned long long acc = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
        uint4 u;
        asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(u.x), "=r"(u.y), "=r"(u.z), "=r"(u.w) : "l"(src + i) : "memory");
        acc += u.x ^ u.y ^ u.z ^ u.w;
    }
    if (acc == 0x1234567887654321ull) *sink = acc;       // keep the loads alive
}

__global__ void peer_write(uint4* __restrict__ dst, size_t nvec) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = make_uint4((unsigned)i, 1u, 2u, 3u);
}

int main() {
    int ndev = 0;
    CK(cudaGetDeviceCount(&ndev));
    if (ndev < 2) { printf("needs 2 GPUs, found %d\n", ndev); return 0; }
    int can01 = 0, can10 = 0;
    CK(cudaDeviceCanAccessPeer(&can01, 0, 1)); CK(cudaDeviceCanAccessPeer(&can10, 1, 0));
    if (!can01 || !can10) { printf("no peer access between GPU 0 and 1\n"); return 0; }
    CK(cudaSetDevice(0)); CK(cudaDeviceEnablePeerAccess(1, 0));
    CK(cudaSetDevice(1)); CK(cudaDeviceEnablePeerAccess(0, 0));

    // ---- 1. flag round trip
    uint32_t *flag0, *flag1; long long *cyc0, *cyc1;
    CK(cudaSetDevice(0)); CK(cudaMalloc(&flag0, 256)); CK(cudaMemset(flag0, 0, 256)); CK(cudaMalloc(&cyc0, 8));
    CK(cudaSetDevice(1)); CK(cudaMalloc(&flag1, 256)); CK(cudaMemset(flag1, 0, 256)); CK(cudaMalloc(&cyc1, 8));
    CK(cudaDeviceSynchronize()); CK(cudaSetDevice(0)); CK(cudaDeviceSynchronize());
    const int iters = 20000;
    cudaEvent_t e0, e1;
    CK(cudaSetDevice(0)); CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    CK(cudaSetDevice(1)); pingpong<<<1, 1>>>(flag1, flag0, iters, 1, cyc1);
    CK(cudaSetDevice(0)); CK(cudaEventRecord(e0)); pingpong<<<1, 1>>>(flag0, flag1, iters, 0, cyc0); CK(cudaEventRecord(e1));
    CK(cudaDeviceSynchronize()); CK(cudaSetDevice(1)); CK(cudaDeviceSynchronize());
    float ms = 0; CK(cudaEventElapsedTime(&ms, e0, e1));
    printf("flag round trip (release store -> acquire spin -> echo): %.0f ns (%d iterations, %.2f ms)\n", ms * 1e6 / iters, iters, ms);

    // ---- 2./3. peer read / write bandwidth from GPU 0 into memory that lives on GPU 1
    const size_t max_bytes = 128u << 20;
    uint4* remote; unsigned long long* sink;
    CK(cudaSetDevice(1)); CK(cudaMalloc(&remote, max_bytes)); CK(cudaMemset(remote, 1, max_bytes)); CK(cudaDeviceSynchronize());
    CK(cudaSetDevice(0)); CK(cudaMalloc(&sink, 8));
    int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    for (size_t bytes = 256u << 10; bytes <= max_bytes; bytes *= 8) {
        for (int mode = 0; mode < 2; mode++) {
            const int blocks = (int)((bytes / 16 + 511) / 512) < sms * 4 ? (int)((bytes / 16 + 511) / 512) : sms * 4;
            for (int w = 0; w < 3; w++) { if (mode == 0) peer_read<<<blocks, 512>>>(remote, bytes / 16, sink); else peer_write<<<blocks, 512>>>(remote, bytes / 16); }
            CK(cudaEventRecord(e0));
            const int reps = 20;
            for (int r = 0; r < reps; r++) { if (mode == 0) peer_read<<<blocks, 512>>>(remote, bytes / 16, sink); else peer_write<<<blocks, 512>>>(remote, bytes / 16); }
            CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize());
            CK(cudaEventElapsedTime(&ms, e0, e1));
            printf("peer %s %8zu KiB, %4d CTAs: %7.2f us per launch, %7.1f GB/s\n", mode == 0 ? "read " : "write", bytes >> 10, blocks,
                   ms * 1e3 / reps, (double)bytes * reps / (ms * 1e-3) / 1e9);
        }
    }
    return 0;
}
