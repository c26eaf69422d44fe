"""Worker of tests/test_gpu_nccl_bilagrid.py (one process per GPU, launched by torch.distributed.run).

Checks the view-sharded step with bilateral grids under NCCL (bg_train_step_views_bilagrid, DESIGN.md section 4.11), two
local views per rank over four training views; training view 2 is rendered by both ranks in every step (rank 0's second
view and rank 1's first), so its grid takes one update from the sum of two gradients that live on different ranks.  After
three steps
  1. every splat parameter, moment and statistic, and every grid, grid moment and grid step count is BIT-IDENTICAL across
     ranks (each rank updates the grids from the same gathered slots in the same order);
  2. they equal the one-device step_views_bilagrid over all the views, within the tolerances of tests/dp_depth_worker.py;
  3. the grid step counts are the true counts: view 2 once per step, view 3 never.
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
    import brush_b200.bilagrid as B
    import brush_b200.render as R
    import brush_b200.train as T
    from brush_b200.camera import Camera
    from scenes import synthetic_scene

    n, w, h, k = 20_000, 192, 128, 9
    local = 2
    cam0, tr, sh, op = synthetic_scene(n, w, h, k=k, seed=21)
    ctx = R.RenderContext(n, w, h, 0, device=local_rank)

    def cam(v):
        a = math.radians(3.0 * v) / 2.0
        return Camera(position=(0.05 * v, -0.02 * v, 0.0), rotation=(0.0, math.sin(a), 0.0, math.cos(a)), fov_x=cam0.fov_x,
                      fov_y=cam0.fov_y, center_uv=cam0.center_uv)

    params = lambda: [torch.from_numpy(x.copy()).to(dev) for x in (tr, sh, op)]
    gains = ((1.2, 0.9, 0.8), (0.85, 1.1, 1.0), (1.0, 0.8, 1.25), (1.1, 1.1, 0.9))
    train_views = []
    for v in range(4):
        tgt = R.render_splats(ctx, cam(v), (w, h), *params())
        rgb = (tgt.out_img[..., :3] * torch.tensor(gains[v], device=dev) + 0.02).clamp(0, 1)
        q = torch.cat([(rgb * 255).round().to(torch.uint8), torch.full((h, w, 1), 255, dtype=torch.uint8, device=dev)], -1)
        train_views.append(T.SceneBatch(img_packed=q.view(torch.int32).reshape(h, w).contiguous(), camera=cam(v), view_index=v))
    order = [0, 2, 2, 1]                                  # global slot order rank * local + i; view 2 on both ranks
    batches_all = [train_views[v] for v in order]
    mine = batches_all[rank * local:(rank + 1) * local]
    cfg = T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, mean_noise_weight=50.0, seed=5, bilateral_grid=True)
    bounds = T.bounds_from_pos(0.8, tr[:, :3])
    rng = np.random.default_rng(17)
    grid0 = torch.from_numpy((B.identity_grids(4, "cpu").numpy() + rng.normal(0.0, 0.05, (4, 8, 16, 16, 12))).astype(np.float32))

    def run(batches, group_on, steps=3):
        p = params()
        s = T.Splats(p[0], p[1] + 0.1, p[2])
        g = B.BilateralGrids(4, dev)
        g.grids.copy_(grid0)
        t = T.SplatTrainer(cfg, ctx, bounds, bilateral_grids=g)
        losses = []
        for _ in range(steps):
            st = t.step_views_bilagrid(batches, s, distributed=group_on)
            losses.append(float(st.loss.item()))
        torch.cuda.synchronize()
        return s, t, g, losses

    s_dp, t_dp, g_dp, l_dp = run(mine, True)

    def flat(s, t, g):
        return torch.cat([s.transforms.reshape(-1), s.sh_coeffs.reshape(-1), s.raw_opacities.reshape(-1)] +
                         [t._state[x].reshape(-1) for x in ("m_t", "v_t", "m_sh", "v_sh", "m_o", "v_o", "refine_norm", "vis_weight",
                                                             "max_screen")] +
                         [g.grids.reshape(-1), g.m.reshape(-1), g.v.reshape(-1), g.device_steps.view(torch.float32)])
    mineflat = flat(s_dp, t_dp, g_dp)
    gathered = [torch.empty_like(mineflat) for _ in range(world)]
    dist.all_gather(gathered, mineflat)
    for r in range(world):
        assert torch.equal(gathered[r].view(torch.int32), gathered[0].view(torch.int32)), f"rank {r} differs from rank 0"
    assert g_dp.steps == [3, 3, 3, 0], g_dp.steps
    assert torch.equal(g_dp.grids[3], grid0[3].to(dev))
    s_one, t_one, g_one, l_one = run(batches_all, False)
    assert g_one.steps == g_dp.steps
    for name in ("transforms", "sh_coeffs", "raw_opacities"):
        a, b = getattr(s_one, name).double(), getattr(s_dp, name).double()
        close = (a - b).abs() <= 1e-6 + 1e-3 * a.abs()
        assert close.double().mean() > 0.99, (name, float(close.double().mean()))
    for key in ("m_t", "m_sh", "m_o"):
        a, b = t_one._state[key].double(), t_dp._state[key].double()
        assert (a - b).norm() / a.norm() < 1e-3, (key, float((a - b).norm() / a.norm()))
    for name in ("grids", "m", "v"):
        a, b = getattr(g_one, name).double(), getattr(g_dp, name).double()
        assert ((a - b).abs() <= 1e-7 + 1e-3 * a.abs()).double().mean() > 0.99, name
    lt = torch.tensor(l_dp, device=dev, dtype=torch.float64)
    dist.all_reduce(lt)
    np.testing.assert_allclose((lt / world).cpu().numpy(), np.array(l_one), rtol=1e-4)
    ctx.close()
    dist.barrier()
    if rank == 0:
        print(f"DP_BILAGRID_WORKER_OK world={world} losses={l_dp}")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
