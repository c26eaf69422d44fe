"""The bilateral-grid training step through the C++ host layer (include/brush_b200.hpp: BilateralGrids and
SplatTrainer::step with the grids), compiled with g++ against the C ABI: the same losses as the Python
SplatTrainer.step_fused, which drives the same bg_train_step_bilagrid."""
import math
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "_build", "bilagrid_check")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


@pytest.fixture(scope="module")
def exe():
    from brush_b200 import build
    build.build()
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpp", "bilagrid_check.cpp")
    hdrs = [os.path.join(ROOT, "include", h) for h in ("brush_b200.hpp", "brush_b200.h")]
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in [src] + hdrs):
        lib = os.path.join(ROOT, "brush_b200")
        cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I",
               os.path.join(CUDA, "include"), src, "-o", EXE, "-L", lib, "-lbrush_b200", "-L", os.path.join(CUDA, "lib64"),
               "-lcudart", f"-Wl,-rpath,{lib}", f"-Wl,-rpath,{os.path.join(CUDA, 'lib64')}"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    return EXE


def test_bilagrid_check_compiles(exe):
    assert os.access(exe, os.X_OK)


@pytest.mark.gpu
def test_cpp_grid_step_matches_python_fused_step(exe, tmp_path):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import brush_b200.render as R
    import brush_b200.train as T
    from brush_b200.bilagrid import BilateralGrids
    from scenes import synthetic_scene
    from test_cpp_host import _cam_line
    n, w, h, k, steps, views, view = 15_000, 192, 128, 4, 3, 3, 2
    cam, tr, sh, op = synthetic_scene(n, w, h, k=k, seed=61)
    ctx = R.RenderContext(n, w, h)
    d = ctx.device
    try:
        out = R.render_splats(ctx, cam, (w, h), *(torch.from_numpy(x).to(d) for x in (tr, sh, op)))
        rgb = (out.out_img[..., :3] * torch.tensor([1.15, 0.95, 0.85], device=d) + 0.02).clamp(0, 1)
        packed = torch.cat([(rgb * 255).round().to(torch.uint8), torch.full((h, w, 1), 255, dtype=torch.uint8, device=d)], -1)
        gt = packed.view(torch.int32).reshape(h, w).contiguous()
        sh0 = (sh + np.float32(0.1)).astype(np.float32)
        bounds = T.bounds_from_pos(0.8, tr[:, :3])
        line = _cam_line(cam, w, h).encode()
        scene = tmp_path / "bilagrid_train.bin"
        with open(scene, "wb") as f:
            f.write(struct.pack("<7If", n, k, w, h, steps, views, view, bounds.median_size()))
            f.write(struct.pack("<I", len(line)) + line)
            f.write(tr.tobytes() + sh0.tobytes() + op.tobytes())
            f.write(gt.cpu().numpy().astype(np.int32).tobytes())
        r = subprocess.run([exe, str(scene)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        lines = r.stdout.strip().splitlines()
        cpp = [(float(ln.split()[1]), float(ln.split()[2])) for ln in lines if ln.startswith("loss")]
        counts = [int(x) for ln in lines if ln.startswith("steps") for x in ln.split()[1:]]
        cfg = T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, seed=7, bilateral_grid=True)
        splats = T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr, sh0, op)))
        grids = BilateralGrids(views, d)
        trainer = T.SplatTrainer(cfg, ctx, bounds, bilateral_grids=grids)
        batch = T.SceneBatch(img_packed=gt, camera=cam, view_index=view)
        py = []
        for _ in range(steps):
            st = trainer.step_fused(batch, splats)
            py.append((float(st.loss.item()), float(st.tv_loss.item())))
        assert len(cpp) == steps and all(math.isfinite(x) for p in cpp for x in p)
        assert counts == grids.steps == [0, 0, steps]
        assert cpp[0][1] == 0.0 and cpp[-1][1] > 0.0          # identity start: no TV term; the grid moved
        np.testing.assert_allclose(np.array(cpp), np.array(py), rtol=1e-3, atol=1e-12)
    finally:
        ctx.close()
