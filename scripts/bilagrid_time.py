"""Device time of the bilateral grid (DESIGN.md section 4.11; development aid, not the bench).

The headline scene (1M synthetic Gaussians, 1920x1080, K = 16, bench.py's config [1] generator and seed): the
single-view step through step_fused, without and with a bilateral grid, alternated call by call in blocks of --block
steps between CUDA events (median block), and each new kernel alone (bg_bilagrid_slice, bg_bilagrid_slice_backward,
bg_bilagrid_update) with CUDA events around each call (median).  The slice's algorithmic bytes are 32 per pixel, the
backward's 48; the rates are against the H100 SXM data-sheet HBM3 rate of 3.35 TB/s.  The card's name and power limit
are read in the same run.  Prints one JSON line.

    python scripts/bilagrid_time.py [--iters 50] [--block 10]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import brush_b200.bilagrid as B  # noqa: E402
import brush_b200.render as R  # noqa: E402
import brush_b200.train as T  # noqa: E402
from scenes import random_v_output, synthetic_scene  # noqa: E402

N, W, H, K, SEED = 1_000_000, 1920, 1080, 16, 0xB2000001
HBM_TBS = 3.35


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def median_ms(fn, iters):
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for _ in range(3):
        fn()
    for e0, e1 in evs:
        e0.record()
        fn()
        e1.record()
    torch.cuda.synchronize()
    return float(np.median([e0.elapsed_time(e1) for e0, e1 in evs]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--block", type=int, default=10)
    a = ap.parse_args()
    cam, tr, sh, op = synthetic_scene(N, W, H, k=K, seed=SEED)
    ctx = R.RenderContext(N, W, H, 0)
    d = ctx.device
    target = R.render_splats(ctx, cam, (W, H), *(torch.from_numpy(x).to(d) for x in (tr, sh, op)), rpass=0)
    gt = (target.out_img | (255 << 24)).clone()
    batch = T.SceneBatch(img_packed=gt, camera=cam, view_index=0)
    runs = {}
    for use in (False, True):
        cfg = T.TrainConfig(total_train_iters=30000, background_noise_strength=0.0, seed=1, bilateral_grid=use)
        s = T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr, sh + np.float32(0.05), op)))
        grids = B.BilateralGrids(1, d) if use else None
        runs[use] = (T.SplatTrainer(cfg, ctx, T.bounds_from_pos(0.8, tr[:, :3]), bilateral_grids=grids), s)
    for use in (False, True):                         # warm-up: every shape, module load and workspace
        for _ in range(3):
            runs[use][0].step_fused(batch, runs[use][1])
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for _ in range(a.iters // 2 or 1):
        for use in (False, True):
            t, s = runs[use]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.block):
                t.step_fused(batch, s)
            e1.record()
            e1.synchronize()
            times[use].append(e0.elapsed_time(e1) / a.block)
    step_off, step_on = float(np.median(times[False])), float(np.median(times[True]))
    # the kernels alone, on a raw render of the scene and a trained-looking grid
    out = R.render_splats(ctx, cam, (W, H), *(torch.from_numpy(x).to(d) for x in (tr, sh, op)), rpass=1)
    img = out.out_img
    rng = np.random.default_rng(1)
    grid = torch.from_numpy((B.identity_grids(1, "cpu")[0].numpy() + rng.normal(0, 0.05, (8, 16, 16, 12))).astype(np.float32)).to(d)
    sliced = torch.empty_like(img)
    v_out = torch.from_numpy(random_v_output(H, W)).to(d)
    v_img = torch.empty_like(v_out)
    v_grid = torch.empty((8, 16, 16, 12), device=d)
    grids = B.BilateralGrids(1, d)
    ms_slice = median_ms(lambda: B.slice(ctx, grid, img, out=sliced), a.iters)
    ms_bwd = median_ms(lambda: B.slice_backward(ctx, grid, img, v_out, v_img=v_img, v_grid=v_grid), a.iters)
    ms_upd = median_ms(lambda: B.update(ctx, grids, 0, v_grid, 1e-3, 10.0), a.iters)
    px = W * H
    res = {
        "card": card(),
        "scene": f"1M synthetic Gaussians, {W}x{H}, K={K}, step_fused",
        "step_ms_without_grid": step_off, "step_ms_with_grid": step_on,
        "added_pct": 100.0 * (step_on - step_off) / step_off,
        "slice_us": ms_slice * 1e3, "slice_tbs": 32 * px / (ms_slice * 1e-3) / 1e12,
        "slice_bwd_us": ms_bwd * 1e3, "slice_bwd_tbs": 48 * px / (ms_bwd * 1e-3) / 1e12,
        "update_us": ms_upd * 1e3,
        "hbm_datasheet_tbs": HBM_TBS,
    }
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
