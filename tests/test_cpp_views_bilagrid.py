"""The multi-view step with bilateral grids through the C++ host layer (include/brush_b200.hpp:
SplatTrainer::step_views_bilagrid), compiled with g++ against the C ABI: the same losses, parameters, grids and grid step
counts as the Python SplatTrainer.step_views_bilagrid, which drives the same bg_train_step_views_bilagrid."""
import math
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "_build", "views_bilagrid_check")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


@pytest.fixture(scope="module")
def exe():
    from brush_b200 import build
    build.build()
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    src = os.path.join(ROOT, "tests", "cpp", "views_bilagrid_check.cpp")
    hdrs = [os.path.join(ROOT, "include", h) for h in ("brush_b200.hpp", "brush_b200.h")]
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in [src] + hdrs):
        lib = os.path.join(ROOT, "brush_b200")
        cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-ffp-contract=off", "-I", os.path.join(ROOT, "include"), "-I",
               os.path.join(CUDA, "include"), src, "-o", EXE, "-L", lib, "-lbrush_b200", "-L", os.path.join(CUDA, "lib64"),
               "-lcudart", f"-Wl,-rpath,{lib}", f"-Wl,-rpath,{os.path.join(CUDA, 'lib64')}"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    return EXE


def test_views_bilagrid_check_compiles(exe):
    assert os.access(exe, os.X_OK)


@pytest.mark.gpu
def test_cpp_views_bilagrid_step_matches_python(exe, tmp_path):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import brush_b200.bilagrid as B
    import brush_b200.render as R
    import brush_b200.train as T
    from brush_b200.camera import Camera
    from scenes import synthetic_scene
    from test_cpp_host import _cam_line
    n, w, h, k, steps, num_grids = 15_000, 192, 128, 4, 3, 4
    cam0, tr, sh, op = synthetic_scene(n, w, h, k=k, seed=57)
    cams = [cam0]
    for ang, pos in ((3.0, (0.08, -0.03, 0.0)), (-2.0, (-0.06, 0.05, 0.0))):
        a = math.radians(ang) / 2.0
        cams.append(Camera(position=pos, rotation=(0.0, math.sin(a), 0.0, math.cos(a)), fov_x=cam0.fov_x, fov_y=cam0.fov_y,
                           center_uv=cam0.center_uv))
    view_index = [2, 0, 2]                                        # training view 2 twice in every step, view 1 and 3 never
    ctx = R.RenderContext(n, w, h)
    d = ctx.device
    try:
        p = [torch.from_numpy(x).to(d) for x in (tr, sh, op)]
        gts = []
        for i, cam in enumerate(cams):
            out = R.render_splats(ctx, cam, (w, h), *p)
            rgb = (out.out_img[..., :3] * torch.tensor([1.15, 0.9, 0.85], device=d) + 0.02 * i).clamp(0, 1)
            q = torch.cat([(rgb * 255).round().to(torch.uint8), torch.full((h, w, 1), 255, dtype=torch.uint8, device=d)], -1)
            gts.append(q.view(torch.int32).reshape(h, w).contiguous())
        sh0 = (sh + np.float32(0.1)).astype(np.float32)
        bounds = T.bounds_from_pos(0.8, tr[:, :3])
        scene, params_out = tmp_path / "views_bilagrid.bin", tmp_path / "params.bin"
        with open(scene, "wb") as f:
            f.write(struct.pack("<7If", n, k, w, h, steps, len(cams), num_grids, bounds.median_size()))
            f.write(tr.tobytes() + sh0.tobytes() + op.tobytes())
            for cam, gt, v in zip(cams, gts, view_index):
                line = _cam_line(cam, w, h).encode()
                f.write(struct.pack("<I", len(line)) + line)
                f.write(struct.pack("<I", v))
                f.write(gt.cpu().numpy().astype(np.int32).tobytes())
        r = subprocess.run([exe, str(scene), str(params_out)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        lines = r.stdout.strip().splitlines()
        cpp = [[float(x) for x in ln.split()[1:]] for ln in lines if ln.startswith("loss")]
        cpp_steps = [int(x) for x in lines[-1].split()[1:]]
        cfg = T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, seed=7, bilateral_grid=True)
        splats = T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr, sh0, op)))
        grids = B.BilateralGrids(num_grids, d)
        trainer = T.SplatTrainer(cfg, ctx, bounds, bilateral_grids=grids)
        batches = [T.SceneBatch(img_packed=g, camera=c, view_index=v) for c, g, v in zip(cams, gts, view_index)]
        py = []
        for _ in range(steps):
            st = trainer.step_views_bilagrid(batches, splats, distributed=False)
            py.append([float(st.loss.item())] + [float(x) for x in st.tv_loss.cpu().numpy()])
        torch.cuda.synchronize()
        assert len(cpp) == steps and all(math.isfinite(x) for row in cpp for x in row)
        assert cpp_steps == grids.steps == [steps, 0, steps, 0]
        # the first step starts from the same model and identity grids and runs a deterministic forward: the same losses
        assert np.array_equal(np.array(cpp[0], np.float32), np.array(py[0], np.float32)), (cpp[0], py[0])
        assert cpp[-1][1] > 0.0 and cpp[-1][1] == cpp[-1][3]        # view 2's two slots report its one TV value
        np.testing.assert_allclose(np.array(cpp), np.array(py), rtol=1e-4, atol=1e-9)
        raw = np.fromfile(params_out, dtype=np.float32)
        o = n * 10 + n * k * 3 + n
        got = {"transforms": raw[:n * 10], "sh_coeffs": raw[n * 10:n * 10 + n * k * 3], "raw_opacities": raw[n * 10 + n * k * 3:o]}
        for name, c in got.items():
            a = getattr(splats, name).reshape(-1).double().cpu().numpy()
            close = np.abs(a - c.astype(np.float64)) <= 1e-6 + 1e-4 * np.abs(a)
            assert close.mean() > 0.995, (name, float(close.mean()))
        a = grids.grids.reshape(-1).double().cpu().numpy()
        close = np.abs(a - raw[o:].astype(np.float64)) <= 1e-7 + 1e-4 * np.abs(a)
        assert close.mean() > 0.995, float(close.mean())
    finally:
        ctx.close()
