"""Cost of depth supervision at 1M Gaussians / K = 16 / 1080p (development aid, not the bench): the fused training step
(SplatTrainer.step_fused -> bg_train_step) against the same step with a depth target (bg_train_step_depth), alternated
rep by rep (CUDA events, medians), and bg_depth_loss_fused alone: per call with the host wrapper (events over 200 calls)
and the kernel's device time (torch.profiler).  Prints one JSON line with the card and its power limit.
Usage: depth_sup_time.py [n] [w] [h] [reps]"""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np
import torch

import brush_b200.loss as L
import brush_b200.render as R
import brush_b200.train as T
from scenes import splitmix64, synthetic_scene

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
w = int(sys.argv[2]) if len(sys.argv) > 2 else 1920
h = int(sys.argv[3]) if len(sys.argv) > 3 else 1080
reps = int(sys.argv[4]) if len(sys.argv) > 4 else 30
cam, tr, sh, op = synthetic_scene(n, w, h)
ctx = R.RenderContext(n, w, h)
d = ctx.device
ttr, tsh, top = (torch.from_numpy(x).to(d) for x in (tr, sh, op))
# ground truth: the scene itself; depth target: its expected depth on covered pixels, jittered by +-10 %
gt = (R.render_splats(ctx, cam, (w, h), ttr, tsh, top, rpass=R.PASS_FORWARD).out_img | (255 << 24)).clone()
ref = R.render_splats(ctx, cam, (w, h), ttr, tsh, top, render_depth=True)
a = ref.out_img[..., 3]
jit = torch.from_numpy((splitmix64(0xDE7200, h * w).reshape(h, w) * 0.2 + 0.9).astype(np.float32)).to(d)
target = torch.where(a >= 0.5, ref.depth / a.clamp_min(1e-30) * jit, torch.zeros_like(a)).contiguous()
count = int((target > 0).sum())
cfg = T.TrainConfig(total_train_iters=10_000, background_noise_strength=0.0, seed=1, depth_loss_weight=0.5)
bounds = T.bounds_from_pos(0.8, tr[:, :3])
plain_batch = T.SceneBatch(img_packed=gt, camera=cam)
depth_batch = T.SceneBatch(img_packed=gt, camera=cam, depth=target, depth_count=count)
runs = {}
for key in ("plain", "depth"):
    s = T.Splats(ttr.clone(), (tsh + 0.05).contiguous(), top.clone())
    runs[key] = (T.SplatTrainer(cfg, ctx, bounds), s, plain_batch if key == "plain" else depth_batch)


def step(key):
    t, s, b = runs[key]
    return t.step_fused(b, s)


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

# the kernel alone: 200 launches between two events, over an image and depth of the scene
vo = torch.zeros((h, w, 4), dtype=torch.float32, device=d)
vd = torch.empty((h, w), dtype=torch.float32, device=d)
chain = float(np.float32(0.5) / np.float32(count))
for _ in range(5):
    L.depth_loss_fused(ctx, ref.out_img, ref.depth, target, chain, vo, vd)
kern = []
for _ in range(5):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(200):
        L.depth_loss_fused(ctx, ref.out_img, ref.depth, target, chain, vo, vd)
    e1.record()
    torch.cuda.synchronize()
    kern.append(e0.elapsed_time(e1) / 200)
# device time of the kernel itself (separate run: tracing slows the host)
from torch.profiler import ProfilerActivity, profile  # noqa: E402

with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(20):
        L.depth_loss_fused(ctx, ref.out_img, ref.depth, target, chain, vo, vd)
    torch.cuda.synchronize()
kernel_dev_ms = next((e.device_time_total / e.count / 1000.0 for e in prof.key_averages() if "depth_loss_fused_kernel" in e.key), None)
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
step_plain, step_depth = float(np.median(ms["plain"])), float(np.median(ms["depth"]))
call_ms = float(np.median(kern))
kernel_ms = kernel_dev_ms if kernel_dev_ms is not None else float("nan")
bytes_px = 16 + 4 + 4 + 4     # out_img (128-bit load), D, t read, v_depth written (v_output[...,3] on active pixels on top)
rec = {"n": n, "w": w, "h": h, "k": int(sh.shape[1]), "reps": reps, "valid_pixels": count,
       "step_fused_ms": {"plain": step_plain, "depth": step_depth, "ratio": step_depth / step_plain},
       "depth_loss_call_ms": call_ms, "depth_loss_kernel_ms": kernel_ms,
       "depth_loss_gb_per_s_at_28_b_per_px": bytes_px * w * h / (kernel_ms * 1e-3) / 1e9,
       "card": smi}
print(json.dumps(rec))
ctx.close()
