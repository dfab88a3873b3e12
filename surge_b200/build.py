"""Build libsgr.so (CUDA kernels + C ABI) in-tree for sm_90a (H100) with nvcc.

The shared object lands in surge_b200/lib/ (git-ignored build product).
nvcc cross-compiles without a GPU, so this is also the "does it build" check on a CPU box.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIB_DIR, "libsgr.so")
OBJ_DIR = os.path.join(HERE, "build")

SOURCES = ["engine.cu", "fold_kernels.cu", "fold_rows.cu", "fold_runs.cu", "fold_vruns.cu", "group_kernels.cu", "incremental.cu", "bulk_fold.cu", "dist.cu", "route_push.cu", "dingest_kernels.cu", "dingest.cu", "id_index.cu", "id_order.cu", "changes.cu", "put_batch.cu", "state_values.cu", "partitioner.cpp", "ingest.cpp"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-Wall", "-Xptxas", "-v"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build the CUDA extension (there is no CPU fallback)")


def _deps_mtime() -> float:
    m = 0.0
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in os.listdir(root):
            m = max(m, os.path.getmtime(os.path.join(root, f)))
    return max(m, os.path.getmtime(os.path.abspath(__file__)))


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _deps_mtime():
        return LIB
    nvcc = _nvcc()
    os.makedirs(OBJ_DIR, exist_ok=True)
    os.makedirs(LIB_DIR, exist_ok=True)

    def compile_one(src: str) -> str:
        obj = os.path.join(OBJ_DIR, os.path.splitext(src)[0] + ".o")
        cmd = [nvcc, *ARCH, *CFLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = r.stdout + r.stderr
        with open(obj + ".log", "w") as f:
            f.write(" ".join(cmd) + "\n" + log)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{log}")
        if verbose:
            print(log)
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    cmd = [nvcc, *ARCH, "-shared", "-o", LIB, *objs, "-Xcompiler", "-fPIC", "-ldl", "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
