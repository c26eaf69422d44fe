"""Device time and effective bandwidth of the projection backward (bg_project_backward), and hashes of its outputs
(development aid, not the bench).

Timing: the headline scene (1M synthetic Gaussians, 1920x1080, the generator and seed of bench.py's config [1]) at
K = 16 and K = 1, once in the scene's own view and once with the camera turned 40 degrees about its y axis, so that
about a third of the splats survive the cull.  Per case: one render and rasterize backward, then --iters calls of
project_bwd, each between its own pair of CUDA events; the median call is reported with the bandwidth it reaches on
the pass's algorithmic bytes, (88 + 12K) V + (48 + 12K) N (V visible splats of N), against the H100 SXM data-sheet
rate of 3.35 TB/s.  The factored variant (12-byte v_color rows in place of the dense v_sh) is timed the same way.
The card's name and power limit are read in the same run and printed with the table.

--dump DIR writes DIR/project_bwd_hashes.json: the SHA-256 of every output array of bg_project_backward (v_transforms,
v_sh, v_raw_opac, v_refine), of the factored variant (its v_color) and of bg_project_backward_depth (v_transforms) for
K in {1, 4, 9, 16, 25}, Mip off and on, a pinhole and a Kannala-Brandt camera, at n = 1 000 003 (a ragged last block),
each on a fixed synthetic v_combined over the forward's visible set (see synthetic_v_combined).  Two builds that
compute the same thing write the same file.

    python scripts/project_bwd_time.py [--iters 50] [--dump DIR]
"""
import argparse
import hashlib
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import brush_b200.render as R  # noqa: E402
from brush_b200.camera import KANNALA_BRANDT_4, Camera  # noqa: E402
from scenes import random_v_output, splitmix64, synthetic_scene  # noqa: E402

N, W, H, SEED = 1_000_000, 1920, 1080, 0xB2000001   # bench.py CONFIGS[1]
HBM_TBS = 3.35                                      # H100 SXM data-sheet HBM3 rate
TURN_DEG = 40.0                                     # low-visibility view: yaw that leaves about a third in view


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def turned(cam: Camera, deg: float) -> Camera:
    h = math.radians(deg) / 2.0
    return Camera(position=cam.position, rotation=(0.0, math.sin(h), 0.0, math.cos(h)), fov_x=cam.fov_x,
                  fov_y=cam.fov_y, center_uv=cam.center_uv, camera_model=cam.camera_model,
                  model_params=cam.model_params)


def median_ms(fn, iters: int) -> float:
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for _ in range(3):
        fn()
    for e0, e1 in evs:
        e0.record()
        fn()
        e1.record()
    torch.cuda.synchronize()
    return float(np.median([e0.elapsed_time(e1) for e0, e1 in evs]))


def time_case(k: int, turn: float, iters: int):
    cam, tr, sh, op = synthetic_scene(N, W, H, k=k, seed=SEED)
    if turn:
        cam = turned(cam, turn)
    ctx = R.RenderContext(N, W, H, 0)
    d = ctx.device
    ttr, tsh, top = (torch.from_numpy(x).to(d) for x in (tr, sh, op))
    out = R.render_splats(ctx, cam, (W, H), ttr, tsh, top)
    vc = R.rasterize_bwd(out, torch.from_numpy(random_v_output(H, W)).to(d))
    dense = (torch.empty((N, 10), device=d), torch.empty((N, k, 3), device=d), torch.empty(N, device=d),
             torch.empty(N, device=d))
    fact = (torch.empty((N, 10), device=d), torch.empty((N, 3), device=d), torch.empty(N, device=d),
            torch.empty(N, device=d))
    ms = median_ms(lambda: R.project_bwd(out, ttr, tsh, top, vc, outputs=dense), iters)
    ms_f = median_ms(lambda: R.project_bwd_factored(out, ttr, tsh, top, vc, outputs=fact), iters)
    V = out.num_visible
    ctx.close()
    return V, ms, ms_f


def run_timing(iters: int):
    print(f"card: {card()}  (name, power limit, max SM clock)")
    print(f"1M@{W}x{H}, project_bwd median of {iters} calls (CUDA events); bytes = (88+12K)V + (48+12K)N, "
          f"rate vs {HBM_TBS} TB/s")
    print(f"{'K':>3} {'view':>10} {'V':>9} {'us':>8} {'MB':>8} {'TB/s':>6} {'of peak':>8} {'factored us':>12}")
    rows = []
    for k in (16, 1):
        for turn in (0.0, TURN_DEG):
            V, ms, ms_f = time_case(k, turn, iters)
            nbytes = (88 + 12 * k) * V + (48 + 12 * k) * N
            tbs = nbytes / (ms * 1e-3) / 1e12
            view = "scene" if not turn else f"turn {turn:.0f}"
            print(f"{k:>3} {view:>10} {V:>9} {ms * 1e3:>8.1f} {nbytes / 1e6:>8.1f} {tbs:>6.2f} {100 * tbs / HBM_TBS:>7.1f}% "
                  f"{ms_f * 1e3:>12.1f}")
            rows.append({"k": k, "turn_deg": turn, "visible": V, "us": ms * 1e3, "bytes": nbytes, "tb_s": tbs,
                         "factored_us": ms_f * 1e3})
    return rows


def sha(t: torch.Tensor) -> str:
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()


def synthetic_v_combined(n: int, visible: int, d):
    """A fixed upstream gradient for the projection backward: v_combined [n, 10] and v_z [n] by compact id.  The blend
    backward accumulates v_combined with float atomics, so its low bits vary from run to run; hashes of the projection
    backward's outputs compare builds only on an input that does not.  Every fifth visible row is all zero (a splat
    whose row is never read) and every seventh has only its refine weight set."""
    r = splitmix64(0xB2000303, n * 11).reshape(n, 11).astype(np.float32)
    vc = (r[:, :10] - np.float32(0.5)) * np.float32(1e-2)
    vz = (r[:, 10] - np.float32(0.5)) * np.float32(1e-2)
    cid = np.arange(n)
    vc[cid >= visible] = 0.0
    vz[cid >= visible] = 0.0
    vc[cid % 5 == 3] = 0.0
    vc[cid % 7 == 4, :9] = 0.0
    return torch.from_numpy(vc).to(d), torch.from_numpy(vz).to(d)


def run_dump(dump_dir: str):
    n, w, h = 1_000_003, 1280, 720
    d = torch.device("cuda", torch.cuda.current_device())
    hashes = {}
    for k in (1, 4, 9, 16, 25):
        cam0, tr, sh, op = synthetic_scene(n, w, h, k=k, seed=SEED)
        ttr, tsh, top = (torch.from_numpy(x).to(d) for x in (tr, sh, op))
        for model in ("pinhole", "kb4"):
            cam = cam0 if model == "pinhole" else Camera(
                position=cam0.position, rotation=cam0.rotation, fov_x=cam0.fov_x, fov_y=cam0.fov_y,
                camera_model=KANNALA_BRANDT_4, model_params=(0.05, -0.01, 0.002, -0.0005))
            for mip in (False, True):
                ctx = R.RenderContext(n, w, h, 0)
                out = R.render_splats(ctx, cam, (w, h), ttr, tsh, top, mip=mip)
                vc, vz = synthetic_v_combined(n, out.num_visible, d)
                vt, vsh, vo, vr = R.project_bwd(out, ttr, tsh, top, vc)
                _, vcol, _, _ = R.project_bwd_factored(out, ttr, tsh, top, vc)
                vtd, _, _, _ = R.project_bwd(out, ttr, tsh, top, vc, v_z=vz)
                key = f"k{k}_{model}_mip{int(mip)}"
                hashes[key] = {"visible": out.num_visible, "v_transforms": sha(vt), "v_sh": sha(vsh),
                               "v_raw_opac": sha(vo), "v_refine": sha(vr), "factored_v_color": sha(vcol),
                               "depth_v_transforms": sha(vtd)}
                print(f"{key}: V={out.num_visible} v_sh {hashes[key]['v_sh'][:16]}", flush=True)
                ctx.close()
    os.makedirs(dump_dir, exist_ok=True)
    with open(os.path.join(dump_dir, "project_bwd_hashes.json"), "w") as f:
        json.dump(hashes, f, indent=1, sort_keys=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--dump", metavar="DIR", default=None, help="write output hashes (no timing)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "project_bwd_time.py measures on a GPU"
    if args.dump:
        run_dump(args.dump)
    else:
        run_timing(args.iters)


if __name__ == "__main__":
    main()
