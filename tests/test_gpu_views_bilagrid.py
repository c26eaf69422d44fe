"""Bilateral grids in the multi-view step on the GPU (bg_train_step_views_bilagrid, DESIGN.md section 4.11): the batched grid
update against sequential bg_bilagrid_update calls bit for bit, the step against a host-orchestrated restatement and
against the single-view step, the depth term, the step counts across both paths, CUDA-graph replay, argument errors, a
scene whose training images carry per-view colour distortions trained four views per step, and the kernels' ptxas
report."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from test_gpu_bilagrid import _close_state, _surface_scene, _train_case  # noqa: E402
from test_gpu_views_depth import _parity_scene  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STATE = ("m_t", "v_t", "m_sh", "v_sh", "m_o", "v_o", "refine_norm", "vis_weight", "max_screen")
FLOATS = 8 * 16 * 16 * 12


@pytest.fixture(scope="module")
def rt():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import brush_b200.bilagrid as B
    import brush_b200.render as R
    import brush_b200.train as T
    from brush_b200 import _lib

    class RT:
        pass

    r = RT()
    r.B, r.R, r.T, r.lib = B, R, T, _lib
    r.ctx = R.RenderContext(max_splats=1 << 16, max_w=1920, max_h=1080, max_intersections=1 << 22)
    yield r
    r.ctx.close()


def _bits(x):
    return x.contiguous().view(torch.int32)


def _perturbed_grids(rt, views, seed, sigma=0.05):
    g = rt.B.BilateralGrids(views, rt.ctx.device)
    rng = np.random.default_rng(seed)
    g.grids.add_(torch.from_numpy(rng.normal(0.0, sigma, tuple(g.grids.shape)).astype(np.float32)).to(g.grids.device))
    return g


def test_update_views_matches_sequential_updates_bit_for_bit(rt):
    """5 slots over 3 of 4 views (views 2 and 0 twice each): each view's update equals one bg_bilagrid_update given the
    float32 sum of its slots in slot order; view 3 is untouched."""
    d = rt.ctx.device
    rng = np.random.default_rng(41)
    a, b = _perturbed_grids(rt, 4, 3), _perturbed_grids(rt, 4, 3)
    m = torch.from_numpy(rng.normal(0.0, 1e-3, (4, 8, 16, 16, 12)).astype(np.float32)).to(d)
    v = torch.from_numpy(rng.uniform(0.0, 1e-6, (4, 8, 16, 16, 12)).astype(np.float32)).to(d)
    for g in (a, b):
        g.m.copy_(m)
        g.v.copy_(v)
    counts = [3, 0, 7, 2]                                   # view 1 takes its first step (the Adam start)
    a.steps[:] = counts
    b.advance_on_device().copy_(torch.tensor(counts, dtype=torch.int32))
    slot_view = [2, 0, 1, 2, 0]
    slots = torch.from_numpy(rng.normal(0.0, 1e-3, (5, 8, 16, 16, 12)).astype(np.float32)).to(d)
    lr, tvw = 2.5e-3, 10.0
    given = slots.clone()                                   # update_views adds into the owner slots in place
    tv_b = rt.B.update_views(rt.ctx, b, slot_view, slots, lr, tvw)
    want_tv, want_g = {}, {}
    for view in (2, 0, 1):
        idx = [j for j, x in enumerate(slot_view) if x == view]
        g = _slot_sum(given, idx)
        want_tv[view] = rt.B.update(rt.ctx, a, view, g, lr, tvw).clone()
        want_g[view] = (idx[0], g)
    torch.cuda.synchronize()
    for name in ("grids", "m", "v"):
        assert torch.equal(_bits(getattr(a, name)), _bits(getattr(b, name))), name
    assert b.steps == a.steps == [4, 1, 8, 2]
    assert b.device_steps.tolist() == [4, 1, 8, 2]
    for j, view in enumerate(slot_view):
        assert torch.equal(_bits(tv_b[j]), _bits(want_tv[view])), (j, view)
    for view, (j, g) in want_g.items():                    # the owner slot holds the sum + the TV gradient
        assert torch.equal(_bits(slots[j]), _bits(g)), view
    assert float(want_tv[2]) > 0.0
    assert torch.equal(_bits(b.grids[3]), _bits(_perturbed_grids(rt, 4, 3).grids[3]))


def _slot_sum(slots, idx):
    s = slots[idx[0]].clone()
    for j in idx[1:]:
        s = s + slots[j]
    return s


def test_step_equals_host_orchestrated_restatement(rt):
    """Three views in one step against the operators: per view render, slice, loss, slice backward, rasterize and project
    backward (SplatTrainer.step with its update captured); the splat gradients averaged into bg_train_update; each view's
    grid updated with its own gradient through bg_bilagrid_update."""
    tr, sh, op, batches = _parity_scene(rt)
    batches = [rt.T.SceneBatch(img_packed=b.img_packed, camera=b.camera, view_index=i) for i, b in enumerate(batches)]
    d = rt.ctx.device
    cfg = rt.T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, mean_noise_weight=50.0, seed=11,
                           bilateral_grid=True)
    captured = {}

    class Capture(rt.T.SplatTrainer):
        def _apply_updates(self, splats, v_t, v_sh, v_o, v_r, visible, max_radius, median_scale):
            captured.update(v_t=v_t.clone(), v_sh=v_sh.clone(), v_o=v_o.clone(), v_r=v_r.clone(), vis=visible.clone(),
                            rad=max_radius.clone())
            return 0.0

    bounds = rt.T.bounds_from_pos(0.8, tr[:, :3])
    p = [torch.from_numpy(x.copy()).to(d) for x in (tr, sh, op)]
    fresh = lambda: rt.T.Splats(p[0].clone(), p[1] + 0.1, p[2].clone())
    multi, g_multi = fresh(), _perturbed_grids(rt, 3, 8)
    st = rt.T.SplatTrainer(cfg, rt.ctx, bounds, bilateral_grids=g_multi).step_views_bilagrid(batches, multi, distributed=False)
    loss, tv = float(st.loss.item()), st.tv_loss.clone()
    per_view, singles = [], []
    for b in batches:
        g = _perturbed_grids(rt, 3, 8)
        s1 = Capture(cfg, rt.ctx, bounds, bilateral_grids=g).step(b, fresh())
        per_view.append(dict(captured))
        singles.append((float(s1.loss.item()), s1.tv_loss.clone(), g))
    torch.cuda.synchronize()
    assert abs(loss - np.mean([x[0] for x in singles])) <= 1e-5 * abs(loss)
    for i, (_, tv1, g) in enumerate(singles):
        assert torch.equal(_bits(tv[i]), _bits(tv1)), i           # TV of the same grid: one kernel, the same bits
        assert float(tv1) > 0.0
        for name in ("grids", "m", "v"):
            a, b = getattr(g, name)[i].double(), getattr(g_multi, name)[i].double()
            assert ((a - b).abs() <= 1e-7 + 1e-4 * a.abs()).double().mean() > 0.995, (i, name)
    assert g_multi.steps == [1, 1, 1]
    V = len(batches)
    avg = {k: (sum(pv[k].double() for pv in per_view) / V).float() for k in ("v_t", "v_sh", "v_o")}
    vr = torch.stack([pv["v_r"] for pv in per_view]).amax(0)
    vis = per_view[0]["vis"] + per_view[1]["vis"] + per_view[2]["vis"]
    rad = torch.stack([pv["rad"] for pv in per_view]).amax(0)
    ref = fresh()
    t_ref = rt.T.SplatTrainer(rt.T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, mean_noise_weight=50.0,
                                               seed=11), rt.ctx, bounds)
    t_ref._ensure_state(ref)
    t_ref.step_count = 1
    t_ref._apply_updates(ref, avg["v_t"], avg["v_sh"], avg["v_o"], vr, vis, rad, bounds.median_size())
    torch.cuda.synchronize()
    for name in ("transforms", "sh_coeffs", "raw_opacities"):
        a, b = getattr(ref, name).double(), getattr(multi, name).double()
        assert torch.isfinite(b).all()
        close = (a - b).abs() <= 1e-6 + 1e-4 * a.abs()
        assert close.double().mean() > 0.995, (name, float(close.double().mean()))


def test_one_view_per_step_matches_the_single_view_step(rt):
    cam, tr, sh, op, batch = _train_case(rt)
    d = rt.ctx.device
    cfg = rt.T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, seed=7, bilateral_grid=True)
    runs = []
    for views_path in (False, True):
        s = rt.T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr, sh + np.float32(0.1), op)))
        g = rt.B.BilateralGrids(3, d)
        t = rt.T.SplatTrainer(cfg, rt.ctx, rt.T.bounds_from_pos(0.8, tr[:, :3]), bilateral_grids=g)
        losses = []
        for _ in range(3):
            st = t.step_views_bilagrid([batch], s, distributed=False) if views_path else t.step_fused(batch, s)
            losses.append((float(st.loss.item()), float(st.tv_loss.reshape(-1)[0].item())))
        runs.append((s, t, g, losses))
    (s_a, t_a, g_a, l_a), (s_b, t_b, g_b, l_b) = runs
    for (la, tva), (lb, tvb) in zip(l_a, l_b):
        assert abs(la - lb) <= 2e-4 * abs(la)
        assert abs(tva - tvb) <= 1e-4 * abs(tva) + 1e-12
    assert l_b[-1][1] > 0.0
    _close_state(s_a, t_a, g_a, s_b, t_b, g_b)
    assert g_b.device_steps.tolist() == [0, 3, 0]
    assert torch.equal(g_b.grids[0], g_b.grids[2])


def test_depth_views_report_step_views_depth_losses(rt):
    """Views with and without depth: each view's depth term is the one step_views_depth computes (on the raw render, bit
    for bit), and every view's grid trains."""
    tr, sh, op, batches = _parity_scene(rt)
    d = rt.ctx.device
    base = dict(total_train_iters=1000, background_noise_strength=0.0, seed=11, depth_loss_weight=0.4)
    bounds = rt.T.bounds_from_pos(0.8, tr[:, :3])
    fresh = lambda: rt.T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr, sh + np.float32(0.1), op)))
    want = rt.T.SplatTrainer(rt.T.TrainConfig(**base), rt.ctx, bounds).step_views_depth(batches, fresh(), distributed=False)
    want = want.view_depth_losses.clone()
    g = rt.B.BilateralGrids(3, d)
    vb = [rt.T.SceneBatch(img_packed=b.img_packed, camera=b.camera, depth=b.depth, depth_count=b.depth_count, view_index=i)
          for i, b in enumerate(batches)]
    t = rt.T.SplatTrainer(rt.T.TrainConfig(**base, bilateral_grid=True), rt.ctx, bounds, bilateral_grids=g)
    st = t.step_views_bilagrid(vb, fresh(), distributed=False)
    torch.cuda.synchronize()
    assert torch.equal(_bits(st.view_depth_losses), _bits(want))
    dl = st.view_depth_losses.cpu().numpy()
    assert dl[0] > 0 and dl[1] > 0 and dl[2] == 0.0
    assert abs(float(st.depth_loss) - float(np.mean(dl.astype(np.float64)))) <= 1e-6 * float(st.depth_loss)
    assert (st.tv_loss == 0).all()                               # identity grids: no TV yet
    st2 = t.step_views_bilagrid(vb, fresh(), distributed=False)
    assert (st2.tv_loss > 0).all()                                # ... but every grid moved
    assert g.steps == [2, 2, 2]


def test_step_counts_across_both_paths(rt):
    cam, tr, sh, op, batch = _train_case(rt, n=10_000, seed=99)
    d = rt.ctx.device
    views = [rt.T.SceneBatch(img_packed=batch.img_packed, camera=cam, view_index=v) for v in range(4)]
    cfg = rt.T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, seed=7, bilateral_grid=True)
    s = rt.T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr, sh + np.float32(0.1), op)))
    g = rt.B.BilateralGrids(4, d)
    t = rt.T.SplatTrainer(cfg, rt.ctx, rt.T.bounds_from_pos(0.8, tr[:, :3]), bilateral_grids=g)
    want = [0, 0, 0, 0]
    plan = [("fused", [1]), ("views", [0, 1, 1]), ("views", [3]), ("fused", [3]), ("fused", [1]), ("views", [2, 0])]
    for kind, vs in plan:
        if kind == "fused":
            t.step_fused(views[vs[0]], s)
        else:
            t.step_views_bilagrid([views[v] for v in vs], s, distributed=False)
        for v in set(vs):
            want[v] += 1
        assert g.steps == want, (kind, vs)
        assert g.device_steps.tolist() == want, (kind, vs)


def test_step_replays_under_cuda_graph(rt):
    cam, tr, sh, op, batch = _train_case(rt, n=10_000, seed=321)
    d = rt.ctx.device
    views = [rt.T.SceneBatch(img_packed=batch.img_packed.to(d), camera=cam, view_index=v) for v in range(2)]
    cfg = rt.T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, seed=7, bilateral_grid=True)

    def trainer():
        s = rt.T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr, sh + np.float32(0.1), op)))
        g = rt.B.BilateralGrids(3, d)
        return s, g, rt.T.SplatTrainer(cfg, rt.ctx, rt.T.bounds_from_pos(0.8, tr[:, :3]), bilateral_grids=g)

    s_e, g_e, t_e = trainer()
    for _ in range(2):
        st_e = t_e.step_views_bilagrid(views[:2], s_e, distributed=False)
    l_e = float(st_e.loss.item())
    s_g, g_g, t_g = trainer()
    t_g.step_views_bilagrid(views[:2], s_g, distributed=False)       # the workspace and the device counts exist
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        st_g = t_g.step_views_bilagrid(views[:2], s_g, distributed=False)
    graph.replay()
    torch.cuda.synchronize()
    assert abs(float(st_g.loss.item()) - l_e) <= 2e-4 * abs(l_e)
    for name in ("transforms", "sh_coeffs", "raw_opacities"):
        a, b = getattr(s_e, name).double(), getattr(s_g, name).double()
        assert ((a - b).abs() <= 1e-6 + 1e-4 * a.abs()).double().mean() > 0.995, name
    a, b = g_e.grids.double(), g_g.grids.double()
    assert ((a - b).abs() <= 1e-7 + 1e-4 * a.abs()).double().mean() > 0.995
    assert g_g.steps == g_e.steps == [2, 2, 0]


def test_argument_errors_are_checked_before_any_launch(rt):
    cam, tr, sh, op, batch = _train_case(rt, n=10_000, seed=5)
    d = rt.ctx.device
    lib, L = rt.lib.load(), rt.lib
    views = [rt.T.SceneBatch(img_packed=batch.img_packed, camera=cam, view_index=v) for v in (0, 2)]
    cfg = rt.T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, seed=7, bilateral_grid=True)
    s = rt.T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr, sh + np.float32(0.1), op)))
    g = rt.B.BilateralGrids(3, d)
    t = rt.T.SplatTrainer(cfg, rt.ctx, rt.T.bounds_from_pos(0.8, tr[:, :3]), bilateral_grids=g)
    t._ensure_state(s)
    t.step_count = 1
    n, k = s.num_splats(), s.sh_coeffs.shape[1]
    w, h = batch.img_size()[1], batch.img_size()[0]
    need = int(lib.bg_train_step_views_bilagrid_workspace_bytes(n, k, w, h, 2, 1))
    assert need > int(lib.bg_train_step_views_depth_workspace_bytes(n, k, w, h, 2, 1))
    ws = torch.empty(need, dtype=torch.uint8, device=d)
    loss = torch.zeros(1, device=d)
    a, _, keep = t._views_args(views, s, ws, need, 0)
    a.loss_out = loss.data_ptr()
    tv = torch.full((16,), 9.0, device=d)
    snap = lambda: [x.clone() for x in (s.transforms, s.sh_coeffs, s.raw_opacities, g.grids, g.m, g.v, g.device_steps,
                                        *(t._state[k_] for k_ in STATE))]
    before = snap()

    def call(mutate=None, grids=True):
        gv, idx = g.views_args([0, 2], 1e-3, 10.0, tv)
        if mutate:
            mutate(gv)
        st = lib.bg_train_step_views_bilagrid(rt.ctx.handle, None, None, C.byref(a), None, C.byref(gv) if grids else None)
        torch.cuda.synchronize()
        return st

    def setf(field, value):
        return lambda gv: setattr(gv, field, value)

    assert call(grids=False) == L.BG_ERR_NULL
    for field in ("grids", "m", "v", "steps", "tv_loss_out", "view_index"):
        assert call(setf(field, None)) == L.BG_ERR_NULL, field
    assert call(setf("grids", g.grids.data_ptr() + 4)) == L.BG_ERR_INVALID          # misaligned
    assert call(setf("steps", g.device_steps.data_ptr() + 2)) == L.BG_ERR_INVALID
    assert call(setf("num_views", 2)) == L.BG_ERR_INVALID                            # view 2 out of range
    assert call(setf("num_views", 0)) == L.BG_ERR_INVALID
    for bad in (-1e-3, float("nan"), float("inf")):
        assert call(setf("lr", bad)) == L.BG_ERR_INVALID
        assert call(setf("tv_weight", bad)) == L.BG_ERR_INVALID
    a.workspace_bytes = need - 256
    assert call() == L.BG_ERR_CAPACITY
    a.workspace_bytes = need
    a.local_views = 17                                                              # more than 16 views
    assert call() == L.BG_ERR_INVALID
    a.local_views = 2
    a.step = 0                                                                      # a check of bg_train_step_views
    assert call() == L.BG_ERR_INVALID
    a.step = 1
    for x, y in zip(before, snap()):
        assert torch.equal(_bits(x), _bits(y))                                      # nothing ran
    assert (tv == 9.0).all()
    # the operator: 1..16 slots, aligned gradients
    sv = torch.zeros(17, dtype=torch.int32, device=d)
    vg = torch.zeros((17, FLOATS), device=d)
    gv, _ = g.views_args(None, 1e-3, 10.0, tv)
    for slots, ptr in ((0, vg.data_ptr()), (17, vg.data_ptr()), (1, vg.data_ptr() + 4)):
        assert lib.bg_bilagrid_update_views(rt.ctx.handle, None, C.byref(gv), slots, sv.data_ptr(), ptr) == L.BG_ERR_INVALID
    assert lib.bg_bilagrid_update_views(rt.ctx.handle, None, C.byref(gv), 1, None, vg.data_ptr()) == L.BG_ERR_NULL
    torch.cuda.synchronize()
    for x, y in zip(before, snap()):
        assert torch.equal(_bits(x), _bits(y))
    # and the call that passes runs
    assert call() == L.BG_OK
    assert g.steps == [1, 0, 1]
    del keep


def test_grids_absorb_per_view_colour_distortion_four_views_per_step(rt):
    """The distorted-capture scene of test_gpu_bilagrid.test_grids_absorb_per_view_colour_distortion trained four views
    per step: 600 steps of step_views_bilagrid against 600 steps of step_views without grids (2400 view passes each).
    The grids' learning rate follows the trainer's step (a 1000-step warm-up), so the single-view test's 600 steps are
    kept rather than its 600 view passes: at 150 steps of four views the grids reached a fraction of their rate and the
    margin measured on an H100 was +0.08 dB (28.27 dB without grids, 28.35 dB with them).  At 600 steps the same H100 (80 GB
    HBM3, 700 W power limit) measured 22.88 dB without grids and 24.76 dB with them (+1.89 dB).  Held-out PSNR with grids
    must be at least 0.3 dB above the run without."""
    from brush_b200.camera import Camera
    from brush_b200.eval import eval_stats
    d = rt.ctx.device
    w, h = 160, 120
    tr, sh, op = _surface_scene(6_000, 21)
    hidden = [torch.from_numpy(x).to(d) for x in (tr, sh, op)]
    rng = np.random.default_rng(9)

    def cam_at(px, py):
        return Camera(position=(float(px), float(py), 0.0), rotation=(0.0, 0.0, 0.0, 1.0), fov_x=1.0, fov_y=0.78)

    train_cams = [cam_at(px, py) for px in (-0.3, 0.0, 0.3) for py in (-0.2, 0.2)]
    eval_cams = [cam_at(0.15, 0.0), cam_at(-0.15, 0.1)]

    def render_rgb(cam):
        return rt.R.render_splats(rt.ctx, cam, (w, h), *hidden).out_img[..., :3].clamp(0, 1)

    def pack(rgb):
        q = torch.cat([(rgb * 255).round().to(torch.uint8), torch.full((h, w, 1), 255, dtype=torch.uint8, device=d)], -1)
        return q.view(torch.int32).reshape(h, w).contiguous()

    batches = []
    for i, cam in enumerate(train_cams):
        gain = torch.tensor(rng.uniform(0.6, 1.4, 3), dtype=torch.float32, device=d)
        offset = torch.tensor(rng.uniform(-0.05, 0.05, 3), dtype=torch.float32, device=d)
        gamma = float(rng.uniform(0.7, 1.4))
        batches.append(rt.T.SceneBatch(img_packed=pack((render_rgb(cam).pow(gamma) * gain + offset).clamp(0, 1)), camera=cam,
                                       view_index=i))
    eval_gt = [(render_rgb(c) * 255).round().to(torch.uint8).cpu().numpy() for c in eval_cams]
    r = np.random.default_rng(5)
    tr0 = tr.copy()
    tr0[:, :3] += r.normal(0.0, 0.02, (tr.shape[0], 3)).astype(np.float32)
    sh0 = r.uniform(-0.5, 0.5, sh.shape).astype(np.float32)
    per_step, steps = 4, 600
    res = {}
    for use in (False, True):
        cfg = rt.T.TrainConfig(total_train_iters=steps, mean_noise_weight=0.0, background_noise_strength=0.0, seed=3,
                               bilateral_grid=use)
        s = rt.T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr0, sh0, op)))
        grids = rt.B.BilateralGrids(len(batches), d) if use else None
        t = rt.T.SplatTrainer(cfg, rt.ctx, rt.T.bounds_from_pos(0.8, tr0[:, :3]), bilateral_grids=grids)
        for i in range(steps):
            step = [batches[(per_step * i + j) % len(batches)] for j in range(per_step)]
            (t.step_views_bilagrid if use else t.step_views)(step, s, distributed=False)
        res[use] = float(np.mean([float(eval_stats(rt.ctx, s, c, g).psnr) for c, g in zip(eval_cams, eval_gt)]))
    print(f"four views per step: held-out PSNR without grids {res[False]:.2f} dB, with grids {res[True]:.2f} dB "
          f"({res[True] - res[False]:+.2f} dB)")
    assert res[True] > res[False] + 0.3, res


def test_changed_kernels_are_sm90a_only_and_do_not_spill():
    for obj_name, kernels in (("bilagrid.o", ("bilagrid_tv_kernel",)), ("dp.o", ("write_grid_index_kernel",))):
        obj = os.path.join(ROOT, "brush_b200", "csrc", "_obj", obj_name)
        txt = open(obj + ".ptxas.txt").read()
        for kname in kernels:
            props = [m for m in re.finditer(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                                            r"(\d+) bytes spill loads", txt) if kname in m.group(1)]
            assert len(props) == 1, kname
            assert props[0].group(2, 3, 4) == ("0", "0", "0"), props[0].group(0)
        assert set(re.findall(r"for '(sm_\w+)'", txt)) == {"sm_90a"}
        sass = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
        assert all(kname in sass for kname in kernels)
        assert set(re.findall(r"arch = (sm_\w+)", sass)) == {"sm_90a"}
