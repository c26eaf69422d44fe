"""blend_bwd_kernel's device time, loop counts and residency on the headline scene, for one or more builds of the
library side by side (development aid, not the bench).

Runs bench.py's config [1] scene (1M synthetic Gaussians, 1920x1080) at K = 16 and K = 1 and prints, per build and view:
  * blend_bwd_kernel device time, median over --calls calls, from a torch.profiler run with CUDA activities only;
  * the counting variant's warp-splat iterations, live pairs and stopping pairs (bg_debug_blend_stats);
  * the default instantiation's registers per thread, shared memory per CTA and the CTAs per SM they allow;
  * the relative L2 distance of each build's v_combined from the first build's;
  * the card's name, power limit and max SM clock, read in the same run.
With --depth the same runs time the DEPTH variant as well (render_depth=True, rasterize_bwd_depth with a random v_depth).

Each build is a libbrush_b200.so path (default: the one in the tree).  Builds run in child processes, one per
(round, build), alternated over --rounds rounds so that drift of the card's clock or load spreads over all of them.

    python scripts/blend_bwd_time.py [--calls 60] [--rounds 2] [--depth] [--lib A.so --lib B.so ...]
"""
import argparse
import json
import os
import re
import shutil
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, W, H, SEED = 1_000_000, 1920, 1080, 0xB2000001   # bench.py CONFIGS[1]
KERNEL = "blend_bwd_kernelILb0ELb0ELb0E"          # the default instantiation (no STATS, SMOOTH or DEPTH)
REGS_PER_SM, SMEM_PER_SM, MAX_WARPS_PER_SM, THREADS = 65536, 233472, 64, 128   # H100 (sm_90)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.stdout.strip() else "unknown"


def residency(lib: str):
    """(registers, shared memory per CTA, CTAs per SM) of the default blend_bwd_kernel, from cuobjdump -res-usage."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([tool, "-res-usage", lib], capture_output=True, text=True).stdout
    lines = out.splitlines()
    for i, line in enumerate(lines):
        if KERNEL in line and i + 1 < len(lines):
            regs = int(re.search(r"REG:(\d+)", lines[i + 1]).group(1))
            smem = int(re.search(r"SHARED:(\d+)", lines[i + 1]).group(1))
            by_regs = REGS_PER_SM // (((regs + 7) // 8) * 8 * THREADS)
            # (SHARED is ptxas's static figure plus the 1 KB reserved per CTA on sm_90: 20 480 B for ptxas's 19 456 B)
            by_smem = SMEM_PER_SM // smem
            return regs, smem, min(by_regs, by_smem, MAX_WARPS_PER_SM // (THREADS // 32))
    return None, None, None


def child(lib: str, calls: int, out_dir: str, depth: bool):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    import brush_b200._lib as L
    L.LIB_PATH = lib
    import brush_b200.render as R
    from scenes import random_v_output, synthetic_scene

    assert torch.cuda.is_available(), "blend_bwd_time.py measures on a GPU"
    res = {}
    for k, dep in [(16, False), (1, False)] + ([(16, True)] if depth else []):
        cam, tr, sh, op = synthetic_scene(N, W, H, k=k, seed=SEED)
        ctx = R.RenderContext(N, W, H, 0)
        d = ctx.device
        ttr, tsh, top = (torch.from_numpy(x).to(d) for x in (tr, sh, op))
        vout = torch.from_numpy(random_v_output(H, W)).to(d)
        vdep = torch.rand((H, W), device=d, generator=torch.Generator(d).manual_seed(1))

        def step():
            out = R.render_splats(ctx, cam, (W, H), ttr, tsh, top, render_depth=dep)
            return out, (R.rasterize_bwd_depth(out, vout, vdep)[0] if dep else R.rasterize_bwd(out, vout))

        for _ in range(5):
            out, vc = step()
        torch.cuda.synchronize()
        key = f"{k}{'d' if dep else ''}"
        np.save(os.path.join(out_dir, f"vc_k{key}.npy"), vc.cpu().numpy())
        st = R.blend_stats(out, vout) if not dep else dict(warp_splat_iterations=None, pairs_live=None, pairs_stopping=None)   # (no counting variant with DEPTH)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                step()
            torch.cuda.synchronize()
        path = os.path.join(out_dir, "trace.json")
        prof.export_chrome_trace(path)
        durs = [float(ev["dur"]) for ev in json.load(open(path)).get("traceEvents", [])
                if ev.get("ph") == "X" and ev.get("cat") == "kernel" and "blend_bwd_kernel" in ev["name"]]
        os.remove(path)
        ctx.close()
        res[key] = dict(us=statistics.median(durs), n=len(durs), iters=st["warp_splat_iterations"],
                      live=st["pairs_live"], stop=st["pairs_stopping"])
    json.dump(res, open(os.path.join(out_dir, "res.json"), "w"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--lib", action="append", help="libbrush_b200.so to time (repeat; default: the tree's)")
    ap.add_argument("--depth", action="store_true", help="also time the DEPTH variant at K = 16")
    ap.add_argument("--child", help=argparse.SUPPRESS)
    ap.add_argument("--out", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child(args.child, args.calls, args.out, args.depth)
        return
    import numpy as np
    libs = [os.path.abspath(p) for p in (args.lib or [os.path.join(ROOT, "brush_b200", "libbrush_b200.so")])]
    print(f"card: {card()}  (name, power limit, max SM clock)")
    for lib in libs:
        regs, smem, ctas = residency(lib)
        print(f"{lib}: blend_bwd_kernel<false,false,false> {regs} registers, {smem} B shared, {ctas} CTAs per SM")
    times = {}
    first = {}
    with tempfile.TemporaryDirectory() as td:
        for r in range(args.rounds):
            for li, lib in enumerate(libs):
                od = os.path.join(td, f"{r}_{li}")
                os.makedirs(od)
                subprocess.run([sys.executable, os.path.abspath(__file__), "--child", lib, "--out", od,
                                "--calls", str(args.calls)] + (["--depth"] if args.depth else []), check=True)
                res = json.load(open(os.path.join(od, "res.json")))
                for k, v in res.items():
                    times.setdefault((lib, k), []).append(v["us"])
                    vc = np.load(os.path.join(od, f"vc_k{k}.npy")).astype(np.float64)
                    if k not in first:
                        first[k] = vc
                    rel = float(np.linalg.norm(vc - first[k]) / max(np.linalg.norm(first[k]), 1e-30))
                    print(f"round {r} {os.path.basename(os.path.dirname(lib)) or lib} 1M@1920x1080 K={k.rstrip('d')}"
                          f"{' (DEPTH)' if k.endswith('d') else ''}: "
                          f"blend_bwd_kernel {v['us']:.1f} us (median of {v['n']})  "
                          + ("" if k.endswith("d") else f"iterations {v['iters']}  live pairs {v['live']}  "
                             f"stopping pairs {v['stop']}  ") + f"v_combined rel L2 vs first {rel:.2e}",
                          flush=True)
    for (lib, k), ts in times.items():
        print(f"{lib} K={k}: blend_bwd_kernel median over rounds {statistics.median(ts):.1f} us  {ts}")


if __name__ == "__main__":
    main()
