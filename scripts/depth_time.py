"""Cost of rendering depth at 1M Gaussians / K = 16 / 1080p (development aid, not the bench): forward, blend backward and
forward + backward (render -> rasterize backward -> projection backward), plain against depth, alternated rep by rep;
CUDA events, medians.  A second, profiled pass gives the blend kernels' own device time.  Prints one JSON line with the
card and its power limit.  Usage: depth_time.py [n] [w] [h] [reps]"""
import json
import os
import re
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np
import torch

import brush_b200.render as R
from scenes import random_v_output, splitmix64, synthetic_scene

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
w = int(sys.argv[2]) if len(sys.argv) > 2 else 1920
h = int(sys.argv[3]) if len(sys.argv) > 3 else 1080
reps = int(sys.argv[4]) if len(sys.argv) > 4 else 30
cam, tr, sh, op = synthetic_scene(n, w, h)
ctx = R.RenderContext(n, w, h)
d = ctx.device
ttr, tsh, top = (torch.from_numpy(x).to(d) for x in (tr, sh, op))
v_out = torch.from_numpy(random_v_output(h, w)).to(d)
v_depth = torch.from_numpy(splitmix64(0xDE7100, h * w).reshape(h, w).astype(np.float32)).to(d)


def run(depth, ev=None):
    """one forward + backward; ev: 4 events around forward / blend backward / projection backward"""
    mark = (lambda i: ev[i].record()) if ev else (lambda i: None)
    mark(0)
    out = R.render_splats(ctx, cam, (w, h), ttr, tsh, top, render_depth=depth)
    mark(1)
    if depth:
        vc, vz = R.rasterize_bwd_depth(out, v_out, v_depth)
    else:
        vc, vz = R.rasterize_bwd(out, v_out), None
    mark(2)
    R.project_bwd(out, ttr, tsh, top, vc, v_z=vz)
    mark(3)


for depth in (False, True, False, True):      # warm-up of both paths
    run(depth)
torch.cuda.synchronize()
ms = {False: [], True: []}
for _ in range(reps):
    for depth in (False, True):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        run(depth, ev)
        torch.cuda.synchronize()
        ms[depth].append((ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2]), ev[0].elapsed_time(ev[3])))

# device time of the blend kernels themselves (separate run: tracing slows the host)
from torch.profiler import ProfilerActivity, profile  # noqa: E402

with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(10):
        run(False)
        run(True)
    torch.cuda.synchronize()
kern = {}
for e in prof.key_averages():
    m = re.search(r"blend_(fwd|bwd)_kernel<([^>]*)>", e.key)
    if m:
        flags = [f.strip() for f in m.group(2).split(",")]
        name = f"blend_{m.group(1)}" + ("_depth" if flags[-1] == "true" else "")
        kern[name] = kern.get(name, 0.0) + e.device_time_total / e.count / 1000.0
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()


def med(depth, i):
    return float(np.median([m[i] for m in ms[depth]]))


rec = {"n": n, "w": w, "h": h, "k": int(sh.shape[1]), "reps": reps}
for i, nm in enumerate(("forward_ms", "blend_backward_ms", "fwd_bwd_ms")):
    rec[nm] = {"plain": med(False, i), "depth": med(True, i), "ratio": med(True, i) / med(False, i)}
rec["kernel_ms"] = kern
if "blend_fwd" in kern and "blend_fwd_depth" in kern:
    rec["blend_fwd_kernel_ratio"] = kern["blend_fwd_depth"] / kern["blend_fwd"]
if "blend_bwd" in kern and "blend_bwd_depth" in kern:
    rec["blend_bwd_kernel_ratio"] = kern["blend_bwd_depth"] / kern["blend_bwd"]
rec["card"] = smi
print(json.dumps(rec))
ctx.close()
