"""Build libb200grb.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m pygraphblas_b200.build [--force]

The objects and the .so live next to the sources (git-ignored build products).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200grb.so")
SOURCES = ["objects.cu", "device_ops.cu", "spmv.cu", "spmv_run.cu", "spmv_run_int.cu", "spmv_run_generic.cu", "spmv_pull.cu",
           "spgemm.cu", "vector_ops.cu", "matrix_ops.cu", "matrix_assign.cu", "dist.cu", "hyper.cu", "compat.cu",
           "positional.cu", "spmm.cu", "sddmm.cu", "gemm.cu", "spgemm_pull.cu"]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-std=c++17", "-O3"] + GENCODE + ["-lineinfo",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-diag-suppress", "186,177,550"]


def _nvcc():
    for p in ("/usr/local/cuda/bin/nvcc",):
        if os.path.exists(p):
            return p
    return "nvcc"


def _deps_mtime():
    m = 0.0
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for f in os.listdir(root):
            if f.endswith((".cuh", ".h", ".inc")):
                m = max(m, os.path.getmtime(os.path.join(root, f)))
    return m


def build_library(force=False, verbose=True):
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    dep = _deps_mtime()
    todo = []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(CSRC, s[:-3] + ".o")
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), dep):
            todo.append((src, obj))

    def compile_one(so):
        src, obj = so
        cmd = [_nvcc()] + NVCC_FLAGS + ["-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose and r.stderr.strip():
            print(r.stderr, flush=True)

    if todo:
        with ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
            list(ex.map(compile_one, todo))
    objs = [os.path.join(CSRC, s[:-3] + ".o") for s in srcs]
    if todo or not os.path.exists(LIB) or force:
        cmd = [_nvcc(), "-shared", "-o", LIB] + objs + GENCODE
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv))
