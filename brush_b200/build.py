"""Builds brush_b200/libbrush_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

nvcc cross-compiles without a GPU; the .so is a build product and stays out of git.
project.cu and project_bwd.cu are compiled with -fmad=false (see csrc/bg_math.cuh): the
per-Gaussian stage must round exactly like its specification so that culling, tile counts and
projected rows are reproducible bit for bit.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "csrc", "_obj")
LIB = os.path.join(HERE, "libbrush_b200.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
          "-Xcompiler", "-Wall", "-Xcudafe", "--diag_suppress=177"]
SOURCES = {
    "api.cu": [],
    "project.cu": ["-fmad=false"],
    "project_bwd.cu": ["-fmad=false"],
    "sort.cu": [],
    "blend_fwd.cu": [],
    "blend_bwd.cu": [],
    "loss.cu": [],
    "optim.cu": [],
    "update.cu": ["-fmad=false"],
    "dp.cu": [],
    "refine.cu": ["-fmad=false"],
    "lod.cu": ["-fmad=false"],
    "depth_loss.cu": ["-fmad=false"],
    "compress.cu": ["-fmad=false"],
    "mesh.cu": ["-fmad=false"],
    "mesh_sparse.cu": ["-fmad=false"],
    "bilagrid.cu": [],
}


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _digest() -> str:
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in sorted(os.listdir(root)):
            p = os.path.join(root, f)
            if os.path.isfile(p) and f.endswith((".cu", ".cuh", ".h")):
                h.update(f.encode())
                h.update(open(p, "rb").read())
    h.update(repr(sorted(SOURCES.items())).encode())
    h.update(repr(COMMON + ARCH).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    stamp = os.path.join(OBJ, "digest.txt")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    nvcc = _nvcc()

    def compile_one(item):
        src, extra = item
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [nvcc, *ARCH, *COMMON, *extra, "-Xptxas", "-v", "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        with open(obj + ".ptxas.txt", "w") as f:
            f.write(r.stderr)
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(compile_one, SOURCES.items()))
    cmd = [nvcc, *ARCH, "-shared", "-o", LIB, *objs, "-cudart", "static", "-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
