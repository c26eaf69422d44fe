"""The multi-view step with depth supervision through the C++ host layer (include/brush_b200.hpp: SplatTrainer::step_views
with per-camera depth targets), compiled with g++ against the C ABI: the same losses and parameters as the Python
SplatTrainer.step_views_depth, which drives the same bg_train_step_views_depth."""
import math
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "_build", "views_depth_check")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


@pytest.fixture(scope="module")
def exe():
    from brush_b200 import build
    build.build()
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpp", "views_depth_check.cpp")
    hdrs = [os.path.join(ROOT, "include", h) for h in ("brush_b200.hpp", "brush_b200.h")]
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in [src] + hdrs):
        lib = os.path.join(ROOT, "brush_b200")
        cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I",
               os.path.join(CUDA, "include"), src, "-o", EXE, "-L", lib, "-lbrush_b200", "-L", os.path.join(CUDA, "lib64"),
               "-lcudart", f"-Wl,-rpath,{lib}", f"-Wl,-rpath,{os.path.join(CUDA, 'lib64')}"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    return EXE


def test_views_depth_check_compiles(exe):
    assert os.access(exe, os.X_OK)


@pytest.mark.gpu
def test_cpp_views_depth_step_matches_python(exe, tmp_path):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import brush_b200.render as R
    import brush_b200.train as T
    from brush_b200.camera import Camera
    from scenes import splitmix64, synthetic_scene
    from test_cpp_host import _cam_line
    n, w, h, k, steps, weight = 15_000, 192, 128, 4, 2, 0.4
    cam0, tr, sh, op = synthetic_scene(n, w, h, k=k, seed=57)
    cams = [cam0]
    for ang, pos in ((3.0, (0.08, -0.03, 0.0)), (-2.0, (-0.06, 0.05, 0.0))):
        a = math.radians(ang) / 2.0
        cams.append(Camera(position=pos, rotation=(0.0, math.sin(a), 0.0, math.cos(a)), fov_x=cam0.fov_x, fov_y=cam0.fov_y,
                           center_uv=cam0.center_uv))
    ctx = R.RenderContext(n, w, h)
    d = ctx.device
    try:
        p = [torch.from_numpy(x).to(d) for x in (tr, sh, op)]
        gts, targets = [], []
        for i, cam in enumerate(cams):
            gts.append((R.render_splats(ctx, cam, (w, h), *p, rpass=0).out_img | (255 << 24)).clone())
            if i == 2:                                            # the third view carries no depth
                targets.append(None)
                continue
            out = R.render_splats(ctx, cam, (w, h), *p, render_depth=True)
            a = out.out_img[..., 3].cpu().numpy()
            ed = np.where(a > 0.05, out.depth.cpu().numpy() / np.maximum(a, 1e-30), 0.0)
            targets.append((ed * (0.9 + 0.2 * splitmix64(0xDE6400 + i, h * w).reshape(h, w))).astype(np.float32))
        counts = [0 if t is None else int(np.count_nonzero(t)) for t in targets]
        sh0 = (sh + np.float32(0.1)).astype(np.float32)
        bounds = T.bounds_from_pos(0.8, tr[:, :3])
        scene, params_out = tmp_path / "views_depth.bin", tmp_path / "params.bin"
        with open(scene, "wb") as f:
            f.write(struct.pack("<6I2f", n, k, w, h, steps, len(cams), weight, bounds.median_size()))
            f.write(tr.tobytes() + sh0.tobytes() + op.tobytes())
            for cam, gt, t, c in zip(cams, gts, targets, counts):
                line = _cam_line(cam, w, h).encode()
                f.write(struct.pack("<I", len(line)) + line)
                f.write(struct.pack("<I", c))
                f.write(gt.cpu().numpy().astype(np.int32).tobytes())
                if c > 0:
                    f.write(t.tobytes())
        r = subprocess.run([exe, str(scene), str(params_out)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        cpp = [[float(x) for x in ln.split()[1:]] for ln in r.stdout.strip().splitlines() if ln.startswith("loss")]
        cfg = T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, seed=7, depth_loss_weight=weight)
        splats = T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr, sh0, op)))
        trainer = T.SplatTrainer(cfg, ctx, bounds)
        batches = [T.SceneBatch(img_packed=g, camera=c) if t is None else
                   T.SceneBatch(img_packed=g, camera=c, depth=torch.from_numpy(t), depth_count=cnt)
                   for c, g, t, cnt in zip(cams, gts, targets, counts)]
        py = []
        for _ in range(steps):
            st = trainer.step_views_depth(batches, splats, distributed=False)
            py.append([float(st.loss.item())] + [float(x) for x in st.view_depth_losses.cpu().numpy()])
        torch.cuda.synchronize()
        assert len(cpp) == steps and all(math.isfinite(x) for row in cpp for x in row)
        assert all(row[1] > 0 and row[2] > 0 and row[3] == 0.0 for row in cpp)
        # the first step starts from the same model and runs a deterministic forward: the same f32 losses
        assert np.array_equal(np.array(cpp[0], np.float32), np.array(py[0], np.float32)), (cpp[0], py[0])
        np.testing.assert_allclose(np.array(cpp), np.array(py), rtol=1e-4)
        raw = np.fromfile(params_out, dtype=np.float32)
        got = {"transforms": raw[:n * 10], "sh_coeffs": raw[n * 10:n * 10 + n * k * 3], "raw_opacities": raw[n * 10 + n * k * 3:]}
        for name, c in got.items():
            a = getattr(splats, name).reshape(-1).double().cpu().numpy()
            close = np.abs(a - c.astype(np.float64)) <= 1e-6 + 1e-4 * np.abs(a)
            assert close.mean() > 0.995, (name, float(close.mean()))
    finally:
        ctx.close()
