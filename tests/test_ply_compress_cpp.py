"""Compressed PLY export through the C++ host layer (include/brush_b200.hpp: compress_splats, compressed_ply_bytes),
compiled with g++ against the C ABI: the same file bytes as the Python writer for one seeded model."""
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "_build", "compress_check")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


@pytest.fixture(scope="module")
def exe():
    from brush_b200 import build
    build.build()
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpp", "compress_check.cpp")
    hdrs = [os.path.join(ROOT, "include", h) for h in ("brush_b200.hpp", "brush_b200.h")]
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in [src] + hdrs):
        lib = os.path.join(ROOT, "brush_b200")
        cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I",
               os.path.join(CUDA, "include"), src, "-o", EXE, "-L", lib, "-lbrush_b200", "-L", os.path.join(CUDA, "lib64"),
               "-lcudart", f"-Wl,-rpath,{lib}", f"-Wl,-rpath,{os.path.join(CUDA, 'lib64')}"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    return EXE


def test_compress_check_compiles(exe):
    assert os.access(exe, os.X_OK)


@pytest.mark.gpu
@pytest.mark.parametrize("k,mip", [(1, False), (16, True)])
def test_cpp_writer_matches_python(exe, tmp_path, k, mip):
    import torch
    import brush_b200.render as R
    import compress_ref as cr
    from brush_b200.compress import splat_to_compressed_ply
    from test_ply_compress_cpu import _model, _poison
    n = 3000
    t, sh, op = _model(n, k, seed=0xB2000410 + k, dup=100)
    _poison(t, sh, op)
    inp = tmp_path / "in.bin"
    with open(inp, "wb") as f:
        f.write(struct.pack("<3I", n, k, int(mip)) + t.tobytes() + sh.tobytes() + op.tobytes())
    outp = tmp_path / "out.ply"
    r = subprocess.run([exe, str(inp), str(outp)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.stdout, r.stderr)
    got = open(outp, "rb").read()
    ctx = R.RenderContext(n, 16, 16)
    py = splat_to_compressed_ply(ctx, *(torch.from_numpy(x).to(ctx.device) for x in (t, sh, op)), render_mip=mip)
    assert got == py
    assert got == cr.encode_file(t, sh, op, render_mip=mip)
    ctx.close()
