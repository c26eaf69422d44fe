"""Device time per kernel of one forward + rasterize backward + project backward step (development aid, not the bench).

Runs the headline scene (1M synthetic Gaussians, 1920x1080, the generator and seed of bench.py's config [1]) at K = 16
and the same scene at K = 1.  For each: the step time from CUDA events with the profiler off, then one torch.profiler
run (CUDA activities only) over --steps steps after the warm-up, and one table of kernel name, calls per step, mean
device time per call and share of the summed device time of the step.  The card's name and power limit are read in the
same run and printed with the tables.

    python scripts/forward_stages_time.py [--steps 30] [--warmup 10]
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import brush_b200.render as R  # noqa: E402
from scenes import random_v_output, synthetic_scene  # noqa: E402

N, W, H, SEED = 1_000_000, 1920, 1080, 0xB2000001   # bench.py CONFIGS[1]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def short_name(name: str) -> str:
    name = re.sub(r"^void ", "", name)
    name = re.sub(r"\(.*$", "", name)        # drop the parameter list, keep the template arguments
    return name.replace("bg::", "")


def run(k: int, steps: int, warmup: int):
    cam, tr, sh, op = synthetic_scene(N, W, H, k=k, seed=SEED)
    ctx = R.RenderContext(N, W, H, 0)
    d = ctx.device
    ttr, tsh, top = (torch.from_numpy(x).to(d) for x in (tr, sh, op))
    vout = torch.from_numpy(random_v_output(H, W)).to(d)
    grads = (torch.empty((N, 10), device=d), torch.empty((N, k, 3), device=d), torch.empty(N, device=d),
             torch.empty(N, device=d))

    def step():
        out = R.render_splats(ctx, cam, (W, H), ttr, tsh, top)
        vc = R.rasterize_bwd(out, vout)
        R.project_bwd(out, ttr, tsh, top, vc, outputs=grads)
        return out

    for _ in range(warmup):
        out = step()
    torch.cuda.synchronize()
    V, I = out.num_visible, out.num_intersections
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms_step = e0.elapsed_time(e1) / steps

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        trace = json.load(open(path))
    calls, total = collections.Counter(), collections.Counter()
    for ev in trace.get("traceEvents", []):
        if ev.get("ph") != "X" or ev.get("cat") not in ("kernel", "gpu_memset", "gpu_memcpy"):
            continue
        name = short_name(ev["name"]) if ev["cat"] == "kernel" else ev["name"]
        calls[name] += 1
        total[name] += float(ev["dur"])
    ctx.close()
    return ms_step, V, I, calls, total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "forward_stages_time.py measures on a GPU"
    print(f"card: {card()}  (name, power limit, max SM clock)")
    for k in (16, 1):
        ms_step, V, I, calls, total = run(k, args.steps, args.warmup)
        busy = sum(total.values()) / args.steps
        print(f"\n1M@1920x1080 K={k}: V={V} I={I}  step {ms_step:.3f} ms (events, profiler off)  "
              f"device busy {busy / 1e3:.3f} ms/step (profiled, {args.steps} steps)")
        print(f"{'kernel':<64} {'calls':>6} {'mean us':>9} {'us/step':>9} {'share':>7}")
        for name, t in sorted(total.items(), key=lambda kv: -kv[1]):
            per_step = t / args.steps
            print(f"{name[:64]:<64} {calls[name] / args.steps:>6.2f} {t / calls[name]:>9.1f} {per_step:>9.1f} "
                  f"{100.0 * per_step / busy:>6.1f}%")


if __name__ == "__main__":
    main()
