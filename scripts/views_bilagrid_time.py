"""Cost of bilateral grids in the multi-view step at BASELINE config [4] (development aid, not the bench): 2M Gaussians,
K = 16, 8 views of 1920x1080 per step on one device.  SplatTrainer.step_views (bg_train_step_views) against
step_views_bilagrid (bg_train_step_views_bilagrid, a grid per view), alternated rep by rep, CUDA-event medians; then the
batched grid update (bg_bilagrid_update_views over the step's 8 slots) against one bg_bilagrid_update, each timed on its
own over many launches.  Prints one JSON line with the card and its power limit.
Usage: views_bilagrid_time.py [n] [views] [w] [h] [reps]"""
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np
import torch

import brush_b200.bilagrid as B
import brush_b200.render as R
import brush_b200.train as T
from brush_b200.camera import Camera
from scenes import synthetic_scene

n = int(sys.argv[1]) if len(sys.argv) > 1 else 2_000_000
views = int(sys.argv[2]) if len(sys.argv) > 2 else 8
w = int(sys.argv[3]) if len(sys.argv) > 3 else 1920
h = int(sys.argv[4]) if len(sys.argv) > 4 else 1080
reps = int(sys.argv[5]) if len(sys.argv) > 5 else 20
cam0, tr, sh, op = synthetic_scene(n, w, h)
ctx = R.RenderContext(n, w, h)
d = ctx.device
ttr, tsh, top = (torch.from_numpy(x).to(d) for x in (tr, sh, op))


def cam(v):
    a = math.radians(1.5 * v) / 2.0
    return Camera(position=(cam0.position[0] + 0.02 * v, cam0.position[1] - 0.01 * v, cam0.position[2]),
                  rotation=(0.0, math.sin(a), 0.0, math.cos(a)), fov_x=cam0.fov_x, fov_y=cam0.fov_y, center_uv=cam0.center_uv)


batches = []
for v in range(views):
    c = cam(v)
    gt = (R.render_splats(ctx, c, (w, h), ttr, tsh, top, rpass=R.PASS_FORWARD).out_img | (255 << 24)).clone()
    batches.append(T.SceneBatch(img_packed=gt, camera=c, view_index=v))
bounds = T.bounds_from_pos(0.8, tr[:, :3])
runs = {}
for key in ("plain", "grids"):
    cfg = T.TrainConfig(total_train_iters=10_000, background_noise_strength=0.0, seed=1, bilateral_grid=key == "grids")
    s = T.Splats(ttr.clone(), (tsh + 0.05).contiguous(), top.clone())
    runs[key] = (T.SplatTrainer(cfg, ctx, bounds, bilateral_grids=B.BilateralGrids(views, d) if key == "grids" else None), s)


def step(key):
    t, s = runs[key]
    return (t.step_views if key == "plain" else t.step_views_bilagrid)(batches, s, distributed=False)


for _ in range(3):                              # warm-up of both paths
    step("plain")
    step("grids")
torch.cuda.synchronize()
ms = {"plain": [], "grids": []}
for _ in range(reps):
    for key in ("plain", "grids"):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step(key)
        e1.record()
        torch.cuda.synchronize()
        ms[key].append(e0.elapsed_time(e1))

# the grid update on its own: the batched update of the step's slots, and one single-view update, per launch
g = B.BilateralGrids(views, d)
slots = torch.randn((views, B.L, B.H, B.W, 12), device=d) * 1e-4
one = torch.randn((B.L, B.H, B.W, 12), device=d) * 1e-4


def per_launch_us(fn, launches=200):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) * 1e3 / launches)
    return float(np.median(out)), float(min(out)), float(max(out))


batched = per_launch_us(lambda: B.update_views(ctx, g, list(range(views)), slots, 1e-5, 10.0))
single = per_launch_us(lambda: B.update(ctx, g, 0, one, 1e-5, 10.0))
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
p, q = float(np.median(ms["plain"])), float(np.median(ms["grids"]))
rec = {"n": n, "views": views, "w": w, "h": h, "k": int(sh.shape[1]), "reps": reps,
       "step_views_ms": {"plain": p, "grids": q, "ratio": q / p,
                         "plain_min_max": [float(min(ms["plain"])), float(max(ms["plain"]))],
                         "grids_min_max": [float(min(ms["grids"])), float(max(ms["grids"]))]},
       "update_us": {"batched_views": batched[0], "batched_min_max": list(batched[1:]),
                     "single_view": single[0], "single_min_max": list(single[1:])},
       "card": smi}
print(json.dumps(rec))
ctx.close()
