"""Differentiable depth through the C++ host layer (include/brush_b200.hpp: render_depth, rasterize_bwd_depth,
project_bwd_depth), compiled with g++ against the C ABI: the same image, depth and gradients as the Python mirror."""
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "_build", "depth_check")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


@pytest.fixture(scope="module")
def exe():
    from brush_b200 import build
    build.build()
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpp", "depth_check.cpp")
    hdrs = [os.path.join(ROOT, "include", h) for h in ("brush_b200.hpp", "brush_b200.h")]
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in [src] + hdrs):
        lib = os.path.join(ROOT, "brush_b200")
        cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I",
               os.path.join(CUDA, "include"), src, "-o", EXE, "-L", lib, "-lbrush_b200", "-L", os.path.join(CUDA, "lib64"),
               "-lcudart", f"-Wl,-rpath,{lib}", f"-Wl,-rpath,{os.path.join(CUDA, 'lib64')}"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    return EXE


def test_depth_check_compiles(exe):
    assert os.access(exe, os.X_OK)


@pytest.mark.gpu
@pytest.mark.parametrize("smooth", [False, True])
def test_cpp_depth_matches_python_mirror(exe, tmp_path, smooth):
    import torch
    import brush_b200.render as R
    from scenes import random_v_output, splitmix64, synthetic_scene
    from test_cpp_host import _cam_line
    from test_gpu_parity import _grad_close
    n, w, h, k = 6_000, 160, 120, 4
    cam, tr, sh, op = synthetic_scene(n, w, h, k=k, seed=0xDE0600)
    bg = np.array([0.1, 0.2, 0.3], np.float32)
    v_out = random_v_output(h, w)
    v_d = splitmix64(0xDE0601, h * w).reshape(h, w).astype(np.float32)
    line = _cam_line(cam, w, h).encode()
    inp, outp = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as f:
        f.write(struct.pack("<4I", n, k, int(smooth), len(line)))
        f.write(line)
        for a in (tr, sh, op, bg, v_out, v_d):
            f.write(np.ascontiguousarray(a, np.float32).tobytes())
    r = subprocess.run([exe, str(inp), str(outp)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    raw = np.fromfile(outp, np.float32)
    sizes = [h * w * 4, h * w, n, n * 10, n * k * 3, n]
    parts = np.split(raw, np.cumsum(sizes)[:-1])
    assert sum(sizes) == raw.size
    ctx = R.RenderContext(n, w, h)
    try:
        d = ctx.device
        ttr, tsh, top = (torch.from_numpy(x).to(d) for x in (tr, sh, op))
        out = R.render_splats(ctx, cam, (w, h), ttr, tsh, top, background=tuple(bg), rpass=2 if smooth else 1, render_depth=True)
        vc, vz = R.rasterize_bwd_depth(out, torch.from_numpy(v_out).to(d), torch.from_numpy(v_d).to(d))
        vt, vsh, vo, _ = R.project_bwd(out, ttr, tsh, top, vc, v_z=vz)
        np.testing.assert_array_equal(parts[0], out.out_img.cpu().numpy().ravel())
        np.testing.assert_array_equal(parts[1], out.depth.cpu().numpy().ravel())
        for got, want, nm in ((parts[2], vz, "v_z"), (parts[3], vt, "v_transforms"), (parts[4], vsh, "v_sh"), (parts[5], vo, "v_raw_opac")):
            _grad_close(got, want.cpu().numpy().ravel(), name=nm)   # f32 atomics: summation order may differ
    finally:
        ctx.close()
