"""Blend kernels' staging counts and device times on the headline scene (development aid, not the bench).

Runs bench.py's config [1] scene (1M synthetic Gaussians, 1920x1080) at K = 16 and K = 1 and prints, per view:
  * tile-list entries and the backward's staged rows (the counting variant's warp-splat iterations: one staged row
    per set bit of the walked hand-off words);
  * blend_fwd_kernel and blend_bwd_kernel device time, median over --calls calls, from a torch.profiler run with CUDA
    activities only;
  * the card's name, power limit and max SM clock, read in the same run.

    python scripts/blend_staging_time.py [--calls 60]
"""
import argparse
import json
import os
import statistics
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


def run(k: int, calls: int):
    cam, tr, sh, op = synthetic_scene(N, W, H, k=k, seed=SEED)
    ctx = R.RenderContext(N, W, H, 0)
    d = ctx.device
    ttr, tsh, top = (torch.from_numpy(x).to(d) for x in (tr, sh, op))
    vout = torch.from_numpy(random_v_output(H, W)).to(d)

    def step():
        out = R.render_splats(ctx, cam, (W, H), ttr, tsh, top)
        R.rasterize_bwd(out, vout)
        return out

    for _ in range(5):
        out = step()
    torch.cuda.synchronize()
    st = R.blend_stats(out, vout)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            step()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        trace = json.load(open(path))
    durs = {"blend_fwd_kernel": [], "blend_bwd_kernel": []}
    for ev in trace.get("traceEvents", []):
        if ev.get("ph") == "X" and ev.get("cat") == "kernel":
            for name in durs:
                if name in ev["name"]:
                    durs[name].append(float(ev["dur"]))
    ctx.close()
    return st, {name: statistics.median(v) for name, v in durs.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=60)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "blend_staging_time.py measures on a GPU"
    print(f"card: {card()}  (name, power limit, max SM clock)")
    for k in (16, 1):
        st, med = run(k, args.calls)
        print(f"1M@1920x1080 K={k}: tile-list entries {st['tile_list_entries']}  backward rows staged "
              f"{st['warp_splat_iterations']}  blend_fwd_kernel {med['blend_fwd_kernel']:.1f} us  "
              f"blend_bwd_kernel {med['blend_bwd_kernel']:.1f} us  (median of {args.calls} calls)")


if __name__ == "__main__":
    main()
