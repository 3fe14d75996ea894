"""In-tree build of the sm_90a C-ABI library ``spconv_b200/lib/libspconv_b200.so``.

The reference builds its native module through pccm/ccimport JIT (``spconv/build.py:23-74``);
here it is a plain ``nvcc`` invocation per translation unit (cross-compiles without a GPU).
"""
from __future__ import annotations

import concurrent.futures
import os
import subprocess
import sys
from typing import List

_PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_PKG, "csrc")
LIB_DIR = os.path.join(_PKG, "lib")
OBJ_DIR = os.path.join(_PKG, "lib", "obj")
LIB_PATH = os.path.join(LIB_DIR, "libspconv_b200.so")

SOURCES = ["core.cu", "rulebook.cu", "sort.cu", "gemm_simt.cu", "gemm_tc.cu", "gemm_tc_wgrad.cu", "api_gemm.cu", "pool.cu", "pointops.cu", "peer.cu", "sparse_add.cu", "hash_table.cu", "batchnorm.cu", "global_pool.cu", "point_scatter.cu", "depthwise.cu", "group_norm.cu", "point_interp.cu", "fp8.cu"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    return cand if os.path.exists(cand) else "nvcc"


def _deps_mtime() -> float:
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs.append(os.path.join(os.path.dirname(_PKG), "include", "spconv_b200.h"))
    return max(os.path.getmtime(h) for h in hdrs)


def _compile_one(src: str, verbose: bool, extra: List[str]) -> str:
    obj = os.path.join(OBJ_DIR, src.replace(".cu", ".o"))
    srcp = os.path.join(CSRC, src)
    if os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(srcp), _deps_mtime()):
        return obj
    cmd = [_nvcc(), *NVCC_FLAGS, *extra, "-c", srcp, "-o", obj]
    if verbose:
        print(" ".join(cmd), flush=True)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{res.stdout}\n{res.stderr}")
    if verbose and res.stderr.strip():
        print(res.stderr)
    return obj


def build(verbose: bool = False, force: bool = False, ptxas_info: bool = False) -> str:
    os.makedirs(OBJ_DIR, exist_ok=True)
    if force:
        for f in os.listdir(OBJ_DIR):
            os.remove(os.path.join(OBJ_DIR, f))
    extra = ["-Xptxas", "-v"] if ptxas_info else []
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(lambda s: _compile_one(s, verbose or ptxas_info, extra), SOURCES))
    if (not os.path.exists(LIB_PATH)
            or os.path.getmtime(LIB_PATH) < max(os.path.getmtime(o) for o in objs)):
        cmd = [_nvcc(), "-shared", "-cudart", "static", "-gencode", "arch=compute_90a,code=sm_90a",
               "-o", LIB_PATH, *objs]
        if verbose:
            print(" ".join(cmd), flush=True)
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    print(build(verbose=True, force="--force" in sys.argv, ptxas_info="--ptxas" in sys.argv))
