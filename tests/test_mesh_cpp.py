"""Mesh export through the C++ host layer (include/brush_b200.hpp: mesh_ply_bytes, TsdfGrid, extract_mesh), compiled with
g++ against the C ABI: the same file bytes as the Python writer."""
import os
import struct
import subprocess

import numpy as np
import pytest

import mesh_ref as mr
from test_mesh_cpu import analytic_grid

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "_build", "mesh_check")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


@pytest.fixture(scope="module")
def exe():
    from brush_b200 import build
    build.build()
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpp", "mesh_check.cpp")
    hdrs = [os.path.join(ROOT, "include", h) for h in ("brush_b200.hpp", "brush_b200.h")]
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in [src] + hdrs):
        lib = os.path.join(ROOT, "brush_b200")
        cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I",
               os.path.join(CUDA, "include"), src, "-o", EXE, "-L", lib, "-lbrush_b200", "-L", os.path.join(CUDA, "lib64"),
               "-lcudart", f"-Wl,-rpath,{lib}", f"-Wl,-rpath,{os.path.join(CUDA, 'lib64')}"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    return EXE


def test_cpp_mesh_ply_bytes_match_python(exe, tmp_path):
    from brush_b200.ply import mesh_to_ply
    for dims in [(23, 19, 21), (9, 2, 9)]:
        g, origin, h, _ = analytic_grid("torus", dims)
        v, c, f = mr.extract(g, origin, h)
        inp = tmp_path / "in.bin"
        with open(inp, "wb") as fh:
            fh.write(struct.pack("<2I", len(v), len(f)) + v.astype("<f4").tobytes() + c.tobytes() + f.astype("<u4").tobytes())
        outp = tmp_path / "out.ply"
        r = subprocess.run([exe, "ply", str(inp), str(outp)], capture_output=True, text=True, timeout=120)
        assert r.returncode == 0, (r.stdout, r.stderr)
        assert open(outp, "rb").read() == mesh_to_ply(v, c, f)


@pytest.mark.gpu
def test_cpp_extract_mesh_matches_the_restatement(exe, tmp_path):
    from brush_b200.ply import mesh_to_ply
    dims = (37, 45, 50)
    g, origin, h, trunc = analytic_grid("sphere", dims)
    inp = tmp_path / "grid.bin"
    with open(inp, "wb") as fh:
        fh.write(struct.pack("<3I", *dims) + np.array([*origin, h, trunc], "<f4").tobytes() + g["tsdf"].tobytes()
                 + g["weight"].tobytes() + g["rgb"].tobytes())
    outp = tmp_path / "out.ply"
    r = subprocess.run([exe, "grid", str(inp), str(outp)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout, r.stderr)
    assert open(outp, "rb").read() == mesh_to_ply(*mr.extract(g, origin, h))
