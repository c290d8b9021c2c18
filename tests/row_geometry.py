"""TEST INFRASTRUCTURE: the host-side launch geometry of the row kernels (csrc/elementwise.cu: launch_rmsnorm, which serves
RMSNorm, add + RMSNorm and its FP8 variant; csrc/common.cuh: row_threads), restated so that tests can pick widths that run each
instance and name their cases by it.  tests/test_row_geometry_cpu.py holds this file to the sources.

The launcher chooses one of three instances of rmsnorm_kernel from the row width H alone (nvec = H / 8 16-byte vectors):
    VPT = 4   nvec / 4 threads, each keeps 4 vectors in registers     H % 1024 == 0, 2048 <= H <= 8192
    VPT = 2   nvec / 2 threads, each keeps 2 vectors in registers     H % 512 == 0, H <= 4096, not the above
    VPT = 0   row_threads(nvec) threads, the row staged in nvec * 16 bytes of dynamic shared memory; once that and the kernel's
              static shared memory pass 48 KB, the launch raises the kernel's dynamic shared-memory limit first.  The static size
              differs between the 16-bit and the FP8 instances (STATIC_SMEM): at H = 24576 (exactly 48 KB of row) both raise it,
              at H = 24544 only the FP8 instance does."""
from __future__ import annotations

SMEM_DEFAULT = 48 * 1024              # shared memory (static + dynamic) a kernel may use without cudaFuncSetAttribute
STATIC_SMEM = {"rmsnorm": 16 * 4,     # rmsnorm_kernel: red[16]
               "rmsnorm_quant": 32 * 4}       # its FP8 instances: red[16], redmax[16]
VEC = 8                               # 16-bit elements per 16-byte vector


def row_threads(nvec: int) -> int:
    """Threads per row of nvec vectors: one vector per thread up to 512, whole warps."""
    threads = 512 if nvec >= 512 else (256 if nvec >= 256 else (nvec + 31) // 32 * 32)
    return max(threads, 32)


def launch_path(H: int, kernel: str = "rmsnorm") -> tuple:
    """(vpt, threads, dynamic shared-memory bytes, sets the shared-memory attribute) of a launch at width H."""
    nvec = H // VEC
    if nvec % 4 == 0 and (nvec // 4) % 32 == 0 and 64 <= nvec // 4 <= 256:
        return 4, nvec // 4, 0, False
    if nvec % 2 == 0 and (nvec // 2) % 32 == 0 and nvec // 2 <= 256:
        return 2, nvec // 2, 0, False
    smem = nvec * 16
    return 0, row_threads(nvec), smem, smem + STATIC_SMEM[kernel] > SMEM_DEFAULT


def instance(H: int) -> str:
    vpt, _, _, attr = launch_path(H)
    return f"VPT{vpt}" if vpt else ("GEN>48K" if attr else "GEN")


def padded_width(H: int) -> int:
    """Elements the row's threads would cover if every thread handled the same number of vectors."""
    vpt, threads, _, _ = launch_path(H)
    per_thread = vpt or -(-(H // VEC) // threads)
    return threads * per_thread * VEC


# Widths the GPU tests run, each named by its instance.  VPT4 and VPT2 include both ends of their ranges; the generic path
# includes a row narrower than one warp's vectors (64), rows with idle threads (896: 112 vectors on 128 threads; 1040: 130
# on 160), several vectors per thread (8200: 1025 on 512, thread 0 takes 3), the widest row that fits the default 48 KB next to
# red[16] (24544), the row of exactly 48 KB (24576), which does not, and rows past it.
# 1536, 2560, 3584, 4096, 5120 and 8192 are model hidden sizes (Qwen2-1.5B, phi-2, Qwen2-7B, Llama-3-8B, Llama-2-13B,
# Llama-3-70B); 28672 is Llama-3-70B's MLP width.
WIDTHS = (2048, 4096, 5120, 8192,
          512, 1536, 2560, 3584,
          64, 896, 1040, 8200, 16384, 24544,
          24576, 24584, 28672)


def width_id(H: int) -> str:
    return f"{instance(H)}-H{H}"
