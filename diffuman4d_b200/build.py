"""Build libd4d.so (sm_90a, H100) in-tree with nvcc.  No torch, no CPU fallback: the product is this library
(include/d4d.h); it reads no environment variables on the data path.

    python -m diffuman4d_b200.build          # incremental
    python -m diffuman4d_b200.build --force
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "libd4d.so")
SOURCES = ["tmap.cu", "gemm_wgmma.cu", "attention_wgmma.cu", "norm.cu", "elementwise.cu", "unet.cu", "d4d_api.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-Xcompiler", "-fPIC",
         "-diag-suppress", "177"]


def _deps_mtime() -> float:
    t = 0.0
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in os.listdir(root):
            if f.endswith((".h", ".cuh")):
                t = max(t, os.path.getmtime(os.path.join(root, f)))
    return t


def _compile(src: str, force: bool, hdr_t: float) -> str:
    obj = os.path.join(OBJ, src.replace(".cu", ".o"))
    s = os.path.join(CSRC, src)
    if not force and os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(s), hdr_t):
        return obj
    cmd = [NVCC, *FLAGS, "-I", CSRC, "-c", s, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    return obj


def _link(lib: str, objs, force: bool) -> bool:
    need_link = force or not os.path.exists(lib) or any(os.path.getmtime(o) > os.path.getmtime(lib) for o in objs)
    if need_link:
        cmd = [NVCC, "-shared", "-o", lib, *objs, "-cudart", "static", "-gencode", "arch=compute_90a,code=sm_90a",
               "-Xlinker", "--exclude-libs,ALL"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return need_link


def build(force: bool = False, verbose: bool = True) -> str:
    os.makedirs(OBJ, exist_ok=True)
    hdr_t = _deps_mtime()
    with cf.ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 4)) as ex:
        objs = list(ex.map(lambda s: _compile(s, force, hdr_t), SOURCES))
    linked = _link(LIB, objs, force)
    if verbose:
        print(f"[d4d] {'built' if linked else 'up to date'}: {LIB}")
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
