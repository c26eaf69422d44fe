"""Depth-supervised training through the C++ host layer (include/brush_b200.hpp: SplatTrainer::step with a depth target),
compiled with g++ against the C ABI: the same losses as the Python SplatTrainer.step_fused, which drives the same
bg_train_step_depth."""
import math
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "_build", "depth_sup_check")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


@pytest.fixture(scope="module")
def exe():
    from brush_b200 import build
    build.build()
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpp", "depth_sup_check.cpp")
    hdrs = [os.path.join(ROOT, "include", h) for h in ("brush_b200.hpp", "brush_b200.h")]
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in [src] + hdrs):
        lib = os.path.join(ROOT, "brush_b200")
        cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I",
               os.path.join(CUDA, "include"), src, "-o", EXE, "-L", lib, "-lbrush_b200", "-L", os.path.join(CUDA, "lib64"),
               "-lcudart", f"-Wl,-rpath,{lib}", f"-Wl,-rpath,{os.path.join(CUDA, 'lib64')}"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    return EXE


def test_depth_sup_check_compiles(exe):
    assert os.access(exe, os.X_OK)


@pytest.mark.gpu
def test_cpp_depth_step_matches_python_fused_step(exe, tmp_path):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import brush_b200.render as R
    import brush_b200.train as T
    from scenes import splitmix64, synthetic_scene
    from test_cpp_host import _cam_line
    n, w, h, k, steps, weight = 15_000, 192, 128, 4, 3, 0.4
    cam, tr, sh, op = synthetic_scene(n, w, h, k=k, seed=57)
    ctx = R.RenderContext(n, w, h)
    d = ctx.device
    try:
        out = R.render_splats(ctx, cam, (w, h), *(torch.from_numpy(x).to(d) for x in (tr, sh, op)), render_depth=True)
        gt = R.render_splats(ctx, cam, (w, h), *(torch.from_numpy(x).to(d) for x in (tr, sh, op)), rpass=0).out_img
        gt = (gt | (255 << 24)).clone()
        a = out.out_img[..., 3].cpu().numpy()
        ed = np.where(a > 0.05, out.depth.cpu().numpy() / np.maximum(a, 1e-30), 0.0)
        target = (ed * (0.9 + 0.2 * splitmix64(0xDE5400, h * w).reshape(h, w))).astype(np.float32)
        count = int(np.count_nonzero(target))
        sh0 = (sh + np.float32(0.1)).astype(np.float32)
        bounds = T.bounds_from_pos(0.8, tr[:, :3])
        line = _cam_line(cam, w, h).encode()
        scene = tmp_path / "depth_train.bin"
        with open(scene, "wb") as f:
            f.write(struct.pack("<6I2f", n, k, w, h, steps, count, weight, bounds.median_size()))
            f.write(struct.pack("<I", len(line)) + line)
            f.write(tr.tobytes() + sh0.tobytes() + op.tobytes())
            f.write(gt.cpu().numpy().astype(np.int32).tobytes())
            f.write(target.tobytes())
        r = subprocess.run([exe, str(scene)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        cpp = [(float(ln.split()[1]), float(ln.split()[2])) for ln in r.stdout.strip().splitlines() if ln.startswith("loss")]
        cfg = T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, seed=7, depth_loss_weight=weight)
        splats = T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr, sh0, op)))
        trainer = T.SplatTrainer(cfg, ctx, bounds)
        batch = T.SceneBatch(img_packed=gt, camera=cam, depth=torch.from_numpy(target), depth_count=count)
        py = []
        for _ in range(steps):
            st = trainer.step_fused(batch, splats)
            py.append((float(st.loss.item()), float(st.depth_loss.item())))
        assert len(cpp) == steps and all(math.isfinite(x) for p in cpp for x in p) and all(p[1] > 0 for p in cpp)
        np.testing.assert_allclose(np.array(cpp), np.array(py), rtol=1e-3)
    finally:
        ctx.close()
