"""Builds the sm_90a data-plane library IN-TREE: swiftllm_b200/libswiftllm_b200.so (plain nvcc, C ABI).

    python -m swiftllm_b200.build            # incremental (per-file objects under swiftllm_b200/csrc/build/)

The .so and the objects are build products (git-ignored).  sm_90a only: no other -gencode.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
# development variants (e.g. SLLM_BUILD_VARIANT=trace SLLM_NVCC_EXTRA=-DSLLM_PT_TRACE): separate objects and library name; the
# product library is always the plain one
_VARIANT = os.environ.get("SLLM_BUILD_VARIANT", "")
OBJ = os.path.join(CSRC, "build" + ("_" + _VARIANT if _VARIANT else ""))
LIB = os.path.join(HERE, "libswiftllm_b200" + ("_" + _VARIANT if _VARIANT else "") + ".so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v"] + os.environ.get("SLLM_NVCC_EXTRA", "").split()


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale(out, deps):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(d) > t for d in deps)


def build(verbose: bool = False, force: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "swiftllm_b200.h"))
    jobs = []
    for s in sources():
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s[:-3] + ".o")
        if force or _stale(obj, [src] + headers):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        r = subprocess.run([NVCC, *FLAGS, "-c", src, "-o", obj], capture_output=True, text=True)
        log = obj[:-2] + ".ptxas.log"
        with open(log, "w") as f:
            f.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(f"[build] {os.path.basename(src)} ok")
        return obj

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    objs = [os.path.join(OBJ, s[:-3] + ".o") for s in sources()]
    if jobs or _stale(LIB, objs):
        r = subprocess.run([NVCC, "-shared", "-o", LIB, *objs, "-lcudart"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(f"[build] linked {LIB}")
    return LIB


if __name__ == "__main__":
    build(verbose=True, force="--force" in sys.argv)
