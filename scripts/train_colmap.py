#!/usr/bin/env python
"""BASELINE config [2]: a full training run on a synthetic COLMAP-format set.

  1. a hidden scene (tests/scenes.py generator, K=16) is rendered from `views` cameras scattered around the generator's
     viewpoint with THIS repo's forward kernels (the same images the oracle renders -- tests/test_gpu_train_loop.py
     checks that on a small set); images go to <root>/images/*.png, the model to <root>/sparse/0/{cameras,images}.txt +
     points3D.bin in COLMAP's layout (brush-dataset/src/formats/colmap.rs:102-390, colmap-reader/src/lib.rs);
  2. the set is loaded back through brush_b200.dataset.load_colmap (every 8th view held out for evaluation), the
     initial Gaussians come from the COLMAP points (KNN scales, splat_init.rs), and loop.train_loop runs
     loader -> step -> refine -> eval exactly as brush-process/src/train_stream.rs:220-497 schedules them;
  3. reported: iterations / s (whole run, wall clock, refine and data loading included), PSNR / SSIM on the held-out
     views, the splat count after every refine.

With --depth-loss-weight W > 0 the set also gets depths/view_XXXX.png: 16-bit millimetres of the hidden scene's expected
depth D / alpha on covered pixels (alpha >= 0.5), 0 elsewhere; the run trains with the depth term (DESIGN.md section
4.7) and the evaluation adds depth_abs_rel / depth_rmse / depth_coverage.  W = 0 (the default) writes and runs exactly
what it did before.  --write-depths writes the depth maps at W = 0 too (the plain step; evaluation reports the depth
figures).

  python scripts/train_colmap.py --iters 3000 --views 200 --init-points 500000 --max-splats 2000000
"""
from __future__ import annotations

import argparse
import json
import math
import os
import shutil
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

SH_C0 = 0.2820947917738781


def view_camera(base, i: int, rng: np.random.Generator):
    """View i: the generator's camera moved inside a small box and turned by a few degrees (all views keep the
    generated frustum in sight, like a forward-facing capture)."""
    from brush_b200.camera import Camera
    if i == 0:
        return base
    pos = (rng.uniform(-0.35, 0.35), rng.uniform(-0.25, 0.25), rng.uniform(-0.3, 0.15))
    yaw, pitch = math.radians(rng.uniform(-7.0, 7.0)), math.radians(rng.uniform(-4.0, 4.0))
    qy = (0.0, math.sin(yaw / 2), 0.0, math.cos(yaw / 2))            # glam order (x, y, z, w)
    qx = (math.sin(pitch / 2), 0.0, 0.0, math.cos(pitch / 2))
    ax, ay, az, aw = qy
    bx, by, bz, bw = qx
    q = (aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw,
         aw * bw - ax * bx - ay * by - az * bz)
    return Camera(position=pos, rotation=q, fov_x=base.fov_x, fov_y=base.fov_y, center_uv=base.center_uv)


def colmap_pose(cam):
    """Camera (position, local->world quaternion xyzw) -> COLMAP (qw qx qy qz, tx ty tz) of the world->camera pose."""
    from brush_b200.dataset import _quat_to_mat
    x, y, z, w = (float(v) for v in cam.rotation)
    q = (w, -x, -y, -z)
    t = -_quat_to_mat(*q) @ np.array(cam.position, np.float64)
    return q, tuple(float(v) for v in t)


def make_dataset(root: str, ctx, views: int, w: int, h: int, hidden_n: int, init_points: int, seed: int = 0xB2000002,
                 depth: bool = False):
    """Writes the COLMAP-format set under `root` (with depth: also depths/*.png); returns (hidden scene arrays, cameras)."""
    import torch
    from PIL import Image
    import brush_b200.render as R
    from scenes import synthetic_scene
    base, tr, sh, op = synthetic_scene(hidden_n, w, h, k=16, seed=seed)
    dev = ctx.device
    ttr, tsh, top = (torch.from_numpy(x).to(dev) for x in (tr, sh, op))
    rng = np.random.default_rng(seed & 0xFFFF)
    cams = [view_camera(base, i, rng) for i in range(views)]
    os.makedirs(os.path.join(root, "images"), exist_ok=True)
    sparse = os.path.join(root, "sparse", "0")
    os.makedirs(sparse, exist_ok=True)
    focal = float(base.focal(w, h)[0])
    with open(os.path.join(sparse, "cameras.txt"), "w") as f:
        f.write("# Camera list with one line of data per camera:\n#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n")
        f.write(f"1 PINHOLE {w} {h} {focal!r} {float(base.focal(w, h)[1])!r} {w / 2.0} {h / 2.0}\n")
    lines = ["# Image list with two lines of data per image:\n#   IMAGE_ID, QW, QX, QY, QZ, TX, TY, TZ, CAMERA_ID, NAME\n"
             "#   POINTS2D[] as (X, Y, POINT3D_ID)\n"]
    pool = ThreadPoolExecutor(max_workers=8)
    jobs = []
    for i, cam in enumerate(cams):
        name = f"view_{i:04d}.png"
        out = R.render_splats(ctx, cam, (w, h), ttr, tsh, top, rpass=R.PASS_FORWARD)       # packed rgba8, black background
        rgba = out.out_img.cpu().numpy().view(np.uint8).reshape(h, w, 4)
        rgb = np.ascontiguousarray(rgba[..., :3])
        jobs.append(pool.submit(lambda a, p: Image.fromarray(a).save(p, compress_level=1), rgb, os.path.join(root, "images", name)))
        if depth:
            dout = R.render_splats(ctx, cam, (w, h), ttr, tsh, top, rpass=R.PASS_BACKWARD, render_depth=True)
            a = dout.out_img[..., 3]
            ed = torch.where(a >= 0.5, dout.depth / a.clamp_min(1e-30), torch.zeros_like(a))
            mm = (ed * 1000.0).round().clamp(0, 65535).to(torch.int32).cpu().numpy().astype(np.uint16)
            os.makedirs(os.path.join(root, "depths"), exist_ok=True)
            jobs.append(pool.submit(lambda a, p: Image.fromarray(a).save(p, compress_level=1), mm, os.path.join(root, "depths", name)))
        q, t = colmap_pose(cam)
        lines.append(f"{i + 1} {q[0]!r} {q[1]!r} {q[2]!r} {q[3]!r} {t[0]!r} {t[1]!r} {t[2]!r} 1 {name}\n\n")
    with open(os.path.join(sparse, "images.txt"), "w") as f:
        f.writelines(lines)
    # sparse points: a subset of the hidden means, slightly displaced, coloured by the DC term (what SfM would give)
    pick = rng.permutation(hidden_n)[:init_points]
    xyz = tr[pick, :3].astype(np.float64) + rng.normal(0.0, 0.002, (pick.size, 3))
    rgb = np.clip((0.5 + SH_C0 * sh[pick, 0, :]) * 255.0, 0, 255).astype(np.uint8)
    rec = np.zeros(pick.size, dtype=np.dtype([("id", "<i8"), ("xyz", "<f8", 3), ("rgb", "u1", 3), ("err", "<f8"), ("track", "<u8")]))
    rec["id"], rec["xyz"], rec["rgb"], rec["err"] = np.arange(1, pick.size + 1), xyz, rgb, 0.5
    with open(os.path.join(sparse, "points3D.bin"), "wb") as f:
        f.write(np.uint64(pick.size).tobytes())
        f.write(rec.tobytes())
    for j in jobs:
        j.result()
    pool.shutdown()
    return (base, tr, sh, op), cams


def run(device: int = 0, iters: int = 3000, views: int = 200, width: int = 1920, height: int = 1080, hidden_n: int = 1_000_000,
        init_points: int = 500_000, max_splats: int = 2_000_000, refine_every: int = None, root: str = None, quiet: bool = False,
        keep: bool = False, depth_loss_weight: float = 0.0, write_depths: bool = False) -> dict:
    import torch
    import brush_b200.render as R
    import brush_b200.train as T
    from brush_b200 import dataset as ds
    from brush_b200 import splat_init
    from brush_b200.loop import ProcessConfig, train_loop
    say = (lambda *a: None) if quiet else (lambda *a: print(*a, file=sys.stderr, flush=True))
    torch.cuda.set_device(device)
    own_root = root is None
    root = root or tempfile.mkdtemp(prefix="bg_colmap_")
    ctx = R.RenderContext(max_splats, width, height, 0, device=device)
    t0 = time.time()
    make_dataset(root, ctx, views, width, height, hidden_n, init_points, depth=depth_loss_weight > 0 or write_depths)
    t_data = time.time() - t0
    say(f"dataset: {views} views {width}x{height} in {t_data:.1f} s -> {root}")
    t0 = time.time()
    loaded = ds.load_colmap(root, eval_split_every=8)
    tr0, sh0, op0 = splat_init.to_init_splats(loaded.init_splat)
    sh0 = splat_init.with_sh_degree(sh0, 3)
    dev = ctx.device
    splats = T.Splats(*(torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (tr0, sh0, op0)))
    t_init = time.time() - t0
    say(f"loaded {len(loaded.train)} train / {len(loaded.eval)} eval views, {splats.num_splats()} initial splats in {t_init:.1f} s")
    if refine_every is None:
        refine_every = 200 if iters >= 2000 else max(50, iters // 6)
    cfg = T.TrainConfig(total_train_iters=iters, max_splats=max_splats, refine_every=refine_every,
                        growth_stop_iter=max(int(iters * 0.8), 1), seed=1, depth_loss_weight=depth_loss_weight)
    counts, step_ms = [], []
    marks = {"t": None, "done": 0}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def on_step(done, stats, refine):
        if refine is not None:
            counts.append((done, refine.total_splats))
            say(f"  iter {done}: refine -> {refine.total_splats} splats (+{refine.num_added}, -{refine.num_pruned})")
        # device time of the steps between two refines (no refine, no eval inside the window)
        if marks["t"] is None and refine is None and done % refine_every == 2:
            ev0.record(); marks["t"] = done
        elif marks["t"] is not None and done % refine_every == refine_every - 1:
            ev1.record(); ev1.synchronize()
            step_ms.append((done - marks["t"], ev0.elapsed_time(ev1), splats.num_splats()))
            marks["t"] = None

    torch.cuda.synchronize(dev)
    t0 = time.time()
    evals = train_loop(ctx, splats, loaded.train, loaded.eval, cfg, ProcessConfig(eval_every=max(iters, 1), export_every=10 ** 9, seed=7),
                       on_step=on_step, alpha_mode=ds.ALPHA_MASKED)
    wall = time.time() - t0
    res = {"workload": f"configs[2]: {views}-view synthetic COLMAP set {width}x{height}, {init_points} -> <= {max_splats} Gaussians, "
                       f"L1 + D-SSIM, Adam, refine every {refine_every}",
           "iters": iters, "iters_per_s_wall": iters / wall, "wall_s": wall, "dataset_s": t_data, "load_init_s": t_init,
           "final_splats": splats.num_splats(), "splats_after_refine": counts,
           "step_windows": [{"steps": s, "ms_per_step": ms / s, "splats": n} for s, ms, n in step_ms],
           "eval": evals[-1] if evals else None}
    if depth_loss_weight > 0:
        res["depth_loss_weight"] = depth_loss_weight
    if step_ms:
        res["iters_per_s_steps_only"] = sum(s for s, _, _ in step_ms) / (sum(ms for _, ms, _ in step_ms) * 1e-3)
    say(json.dumps(res))
    ctx.close()
    if own_root and not keep:
        shutil.rmtree(root, ignore_errors=True)
    return res


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3000)
    ap.add_argument("--views", type=int, default=200)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--hidden", type=int, default=1_000_000)
    ap.add_argument("--init-points", type=int, default=500_000)
    ap.add_argument("--max-splats", type=int, default=2_000_000)
    ap.add_argument("--refine-every", type=int, default=None)
    ap.add_argument("--root", default=None)
    ap.add_argument("--keep", action="store_true")
    ap.add_argument("--depth-loss-weight", type=float, default=0.0)
    ap.add_argument("--write-depths", action="store_true")
    a = ap.parse_args()
    r = run(iters=a.iters, views=a.views, width=a.width, height=a.height, hidden_n=a.hidden, init_points=a.init_points,
            max_splats=a.max_splats, refine_every=a.refine_every, root=a.root, keep=a.keep, depth_loss_weight=a.depth_loss_weight,
            write_depths=a.write_depths)
    print(json.dumps(r))
