"""The sparse mesh export through the C++ host layer (include/brush_b200.hpp: SparseTsdfGrid, sparse_tsdf_mark /
_allocate / _integrate, extract_mesh), compiled with g++ against the C ABI: the same PLY bytes as the Python path."""
import ctypes
import os
import struct
import subprocess

import numpy as np
import pytest

import mesh_ref as mr
from test_mesh_cpu import fused_sphere_grid

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "_build", "sparse_mesh_check")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


@pytest.fixture(scope="module")
def exe():
    from brush_b200 import build
    build.build()
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpp", "sparse_mesh_check.cpp")
    hdrs = [os.path.join(ROOT, "include", h) for h in ("brush_b200.hpp", "brush_b200.h")]
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in [src] + hdrs):
        lib = os.path.join(ROOT, "brush_b200")
        cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I",
               os.path.join(CUDA, "include"), src, "-o", EXE, "-L", lib, "-lbrush_b200", "-L", os.path.join(CUDA, "lib64"),
               "-lcudart", f"-Wl,-rpath,{lib}", f"-Wl,-rpath,{os.path.join(CUDA, 'lib64')}"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    return EXE


@pytest.mark.gpu
def test_cpp_sparse_mesh_ply_bytes_match_python(exe, tmp_path):
    from brush_b200 import _lib
    import brush_b200.render as R
    from test_gpu_sparse_mesh import sparse_from_maps
    dims = (37, 64, 50)
    ref, origin, h, trunc, maps = fused_sphere_grid(dims, views=8, poison=True)
    inp = tmp_path / "views.bin"
    H, W = maps[0][2].shape
    with open(inp, "wb") as fh:
        fh.write(struct.pack("<3I", *dims) + np.array([*origin, h, trunc], "<f4").tobytes() + struct.pack("<3I", len(maps), W, H))
        for u, img, depth in maps:
            fh.write(bytes(_lib.camera_struct(u)) + np.ascontiguousarray(img, "<f4").tobytes()
                     + np.ascontiguousarray(depth, "<f4").tobytes())
    outp = tmp_path / "out.ply"
    r = subprocess.run([exe, str(inp), str(outp)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout, r.stderr)
    ctx = R.RenderContext(16, W, H)
    py = sparse_from_maps(ctx, dims, origin, h, trunc, maps).extract().to_ply()
    ctx.close()
    got = open(outp, "rb").read()
    assert got == py
    from brush_b200.ply import mesh_to_ply
    assert got == mesh_to_ply(*mr.extract(ref, origin, h))
