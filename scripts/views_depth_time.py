"""Cost of depth supervision in the multi-view step at BASELINE config [4] (development aid, not the bench): 2M Gaussians,
K = 16, 8 views of 1920x1080 per step on one device, a depth target on every pixel.  SplatTrainer.step_views
(bg_train_step_views) against step_views_depth (bg_train_step_views_depth, every view with the term), alternated rep by
rep, CUDA-event medians.  Prints one JSON line with the card and its power limit.
Usage: views_depth_time.py [n] [views] [w] [h] [reps]"""
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np
import torch

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


plain, depth = [], []
for v in range(views):
    c = cam(v)
    gt = (R.render_splats(ctx, c, (w, h), ttr, tsh, top, rpass=R.PASS_FORWARD).out_img | (255 << 24)).clone()
    ref = R.render_splats(ctx, c, (w, h), ttr, tsh, top, render_depth=True)
    a = ref.out_img[..., 3]
    # a target on every pixel: the expected depth where covered, a far plane elsewhere
    t = torch.where(a > 0.05, ref.depth / a.clamp_min(1e-30), torch.full_like(a, 50.0)).contiguous()
    plain.append(T.SceneBatch(img_packed=gt, camera=c))
    depth.append(T.SceneBatch(img_packed=gt, camera=c, depth=t, depth_count=w * h))
cfg = T.TrainConfig(total_train_iters=10_000, background_noise_strength=0.0, seed=1, depth_loss_weight=0.5)
bounds = T.bounds_from_pos(0.8, tr[:, :3])
runs = {}
for key in ("plain", "depth"):
    s = T.Splats(ttr.clone(), (tsh + 0.05).contiguous(), top.clone())
    runs[key] = (T.SplatTrainer(cfg, ctx, bounds), s)


def step(key):
    t, s = runs[key]
    if key == "plain":
        return t.step_views(plain, s, distributed=False)
    return t.step_views_depth(depth, s, distributed=False)


for _ in range(3):                              # warm-up of both paths
    step("plain")
    step("depth")
torch.cuda.synchronize()
ms = {"plain": [], "depth": []}
for _ in range(reps):
    for key in ("plain", "depth"):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step(key)
        e1.record()
        torch.cuda.synchronize()
        ms[key].append(e0.elapsed_time(e1))
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
p, q = float(np.median(ms["plain"])), float(np.median(ms["depth"]))
rec = {"n": n, "views": views, "w": w, "h": h, "k": int(sh.shape[1]), "reps": reps,
       "step_views_ms": {"plain": p, "depth": q, "ratio": q / p,
                         "plain_min_max": [float(min(ms["plain"])), float(max(ms["plain"]))],
                         "depth_min_max": [float(min(ms["depth"])), float(max(ms["depth"]))]},
       "mpix_per_s": {"plain": views * w * h / (p * 1e3), "depth": views * w * h / (q * 1e3)},
       "card": smi}
print(json.dumps(rec))
ctx.close()
