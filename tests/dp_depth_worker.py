"""Worker of tests/test_gpu_nccl_depth.py (one process per GPU, launched by torch.distributed.run).

Checks the view-sharded step with depth supervision under NCCL (bg_train_step_views_depth, DESIGN.md section 4.7), two
local views per rank: rank 0's both carry depth, rank 1's first does and its second does not.  After three steps
  1. every parameter, moment and statistic is BIT-IDENTICAL across ranks (the depth gradient travels in the exchanged rows);
  2. they equal the one-device step_views_depth over all the views, within the tolerances of tests/dp_worker.py;
  3. each rank's per-view depth losses equal the one-device values bit for bit (the forward and the depth reduction are
     deterministic, and the first step starts from the same parameters).
"""
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np
import torch
import torch.distributed as dist


def main():
    rank, world, local_rank = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    dist.init_process_group("nccl", device_id=dev)
    import brush_b200.render as R
    import brush_b200.train as T
    from brush_b200.camera import Camera
    from scenes import splitmix64, synthetic_scene

    n, w, h, k = 20_000, 192, 128, 9
    local = 2
    views = local * world
    cam0, tr, sh, op = synthetic_scene(n, w, h, k=k, seed=21)
    ctx = R.RenderContext(n, w, h, 0, device=local_rank)

    def cam(v):
        a = math.radians(3.0 * v) / 2.0
        return Camera(position=(0.05 * v, -0.02 * v, 0.0), rotation=(0.0, math.sin(a), 0.0, math.cos(a)), fov_x=cam0.fov_x,
                      fov_y=cam0.fov_y, center_uv=cam0.center_uv)

    params = lambda: [torch.from_numpy(x.copy()).to(dev) for x in (tr, sh, op)]
    batches_all = []
    for v in range(views):
        tgt = R.render_splats(ctx, cam(v), (w, h), *params(), rpass=0)
        gt = (tgt.out_img | (255 << 24)).clone()
        if v % local == 1 and v // local == 1:        # rank 1's second view: no depth
            batches_all.append(T.SceneBatch(img_packed=gt, camera=cam(v)))
            continue
        out = R.render_splats(ctx, cam(v), (w, h), *params(), render_depth=True)
        a = out.out_img[..., 3]
        jit = torch.from_numpy((splitmix64(0xDE6300 + v, h * w).reshape(h, w) * 0.2 + 0.9).astype(np.float32)).to(dev)
        t = torch.where(a > 0.05, out.depth / a.clamp_min(1e-30) * jit, torch.zeros_like(a)).contiguous()
        batches_all.append(T.SceneBatch(img_packed=gt, camera=cam(v), depth=t, depth_count=int((t > 0).sum())))
    mine = batches_all[rank * local:(rank + 1) * local]
    cfg = T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, mean_noise_weight=50.0, seed=5, depth_loss_weight=0.4)
    bounds = T.bounds_from_pos(0.8, tr[:, :3])

    def run(batches, group_on, steps=3):
        p = params()
        s = T.Splats(p[0], p[1] + 0.1, p[2])
        t = T.SplatTrainer(cfg, ctx, bounds)
        losses, dls = [], []
        for _ in range(steps):
            st = t.step_views_depth(batches, s, distributed=group_on)
            losses.append(float(st.loss.item()))
            dls.append(st.view_depth_losses.cpu().numpy().copy())
        torch.cuda.synchronize()
        return s, t, losses, dls

    s_dp, t_dp, l_dp, d_dp = run(mine, True)
    # 1. bit-identical across ranks
    def flat(s, t):
        return torch.cat([s.transforms.reshape(-1), s.sh_coeffs.reshape(-1), s.raw_opacities.reshape(-1)] +
                         [t._state[x].reshape(-1) for x in ("m_t", "v_t", "m_sh", "v_sh", "m_o", "v_o", "refine_norm", "vis_weight", "max_screen")])
    mineflat = flat(s_dp, t_dp)
    gathered = [torch.empty_like(mineflat) for _ in range(world)]
    dist.all_gather(gathered, mineflat)
    for r in range(world):
        assert torch.equal(gathered[r].view(torch.int32), gathered[0].view(torch.int32)), f"rank {r} differs from rank 0"
    # 2. equals the one-device step over all views
    s_one, t_one, l_one, d_one = run(batches_all, False)
    for name in ("transforms", "sh_coeffs", "raw_opacities"):
        a, b = getattr(s_one, name).double(), getattr(s_dp, name).double()
        close = (a - b).abs() <= 1e-6 + 1e-3 * a.abs()
        assert close.double().mean() > 0.99, (name, float(close.double().mean()))
    for key in ("m_t", "m_sh", "m_o"):
        a, b = t_one._state[key].double(), t_dp._state[key].double()
        assert (a - b).norm() / a.norm() < 1e-3, (key, float((a - b).norm() / a.norm()))
    for key in ("vis_weight", "max_screen"):
        a, b = t_one._state[key].double(), t_dp._state[key].double()
        assert ((a - b).abs() <= 1e-6 + 1e-3 * a.abs()).double().mean() > 0.999, key
    # 3. the first step's per-view depth losses are the one-device ones bit for bit; rank 1's view without depth has 0
    want = d_one[0][rank * local:(rank + 1) * local]
    assert np.array_equal(d_dp[0].view(np.uint32), want.view(np.uint32)), (d_dp[0], want)
    if rank == 1:
        assert all(d[1] == 0.0 for d in d_dp)
    assert all((d[0] > 0.0) for d in d_dp)
    lt = torch.tensor(l_dp, device=dev, dtype=torch.float64)
    dist.all_reduce(lt)
    np.testing.assert_allclose((lt / world).cpu().numpy(), np.array(l_one), rtol=1e-4)
    ctx.close()
    dist.barrier()
    if rank == 0:
        print(f"DP_DEPTH_WORKER_OK world={world} losses={l_dp}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
