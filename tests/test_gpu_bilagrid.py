"""The bilateral grid of DESIGN.md section 4.11 on the GPU: slice and slice backward against the float64 restatement,
bg_bilagrid_update against TV + Adam restated, the fused step against the host-orchestrated one (with and without the
depth term, and under CUDA-graph replay), a scene whose training images carry a per-view colour distortion, the
training loop's colour-corrected metrics, and the new kernels' SASS."""
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import bilagrid_ref as ref  # noqa: E402
from scenes import synthetic_scene  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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


def _inputs(h, w, seed):
    rng = np.random.default_rng(seed)
    grid = ref.identity()[0] + rng.normal(0.0, 0.1, (8, 16, 16, 12))
    img = rng.uniform(-0.1, 1.1, (h, w, 4))
    img[..., 3] = rng.uniform(0.0, 1.0, (h, w))
    img[::5, ::3, 0:3] += 0.4                       # some gray above 1
    img[1::7, ::4, 0:3] -= 0.4                      # some below 0
    v_out = rng.normal(size=(h, w, 4))
    return grid.astype(np.float32), img.astype(np.float32), v_out.astype(np.float32)


SIZES = [(1, 1), (37, 61), (256, 256), (1080, 1920)]


@pytest.mark.parametrize("h,w", SIZES)
def test_slice_matches_the_reference(rt, h, w):
    grid, img, _ = _inputs(h, w, h * 7 + w)
    d = rt.ctx.device
    out = rt.B.slice(rt.ctx, torch.from_numpy(grid).to(d), torch.from_numpy(img).to(d)).cpu().numpy()
    want = ref.np_slice(grid.astype(np.float64), img.astype(np.float64))
    gray = img[..., 0:3].astype(np.float64) @ ref.LUMA
    assert ((gray < 0) | (gray > 1)).any() or h * w == 1
    assert np.abs(out - want).max() <= 1e-5 * max(1.0, np.abs(want).max() / 2.0)
    assert np.array_equal(out[..., 3], img[..., 3])


@pytest.mark.parametrize("h,w", SIZES)
def test_slice_backward_matches_the_reference(rt, h, w):
    grid, img, v_out = _inputs(h, w, h * 11 + w)
    d = rt.ctx.device
    tg, ti, tv = (torch.from_numpy(x).to(d) for x in (grid, img, v_out))
    v_img, v_grid = rt.B.slice_backward(rt.ctx, tg, ti, tv)
    want_vi, want_vg = ref.np_slice_backward(grid.astype(np.float64), img.astype(np.float64), v_out.astype(np.float64))
    keep = ~ref.kink_mask(img, 1e-6)                 # flagged pixels: gray at a clamp or a level kink
    vi = v_img.cpu().numpy()
    rel = np.linalg.norm((vi - want_vi)[keep]) / max(np.linalg.norm(want_vi[keep]), 1e-30)
    assert rel <= 1e-5, rel
    vg = v_grid.cpu().numpy()
    for k in range(12):
        n = np.linalg.norm(want_vg[..., k])
        if n > 0:
            assert np.linalg.norm(vg[..., k] - want_vg[..., k]) / n <= 1e-4, k
    # in place over v_out gives the same bits; v_grid is overwritten, not accumulated
    v_grid.fill_(7.0)
    vi2, vg2 = rt.B.slice_backward(rt.ctx, tg, ti, tv, v_img=tv, v_grid=v_grid)
    assert vi2.data_ptr() == tv.data_ptr()
    assert np.array_equal(tv.cpu().numpy()[keep], vi[keep])
    np.testing.assert_allclose(vg2.cpu().numpy(), vg, rtol=1e-5, atol=1e-5 * max(np.abs(vg).max(), 1e-30))


def test_update_matches_tv_plus_adam_with_per_view_steps(rt):
    d = rt.ctx.device
    grids = rt.B.BilateralGrids(2, d)
    rng = np.random.default_rng(5)
    init = ref.identity(2) + rng.normal(0.0, 0.05, (2, 8, 16, 16, 12))
    grids.grids.copy_(torch.from_numpy(init.astype(np.float32)))
    p = init.astype(np.float32).astype(np.float64)
    m, v = np.zeros_like(p), np.zeros_like(p)
    t = [0, 0]
    lr, tvw = 3e-3, 10.0
    for view in (0, 1, 0):
        g = rng.normal(0.0, 1e-3, (8, 16, 16, 12)).astype(np.float32)
        vg = torch.from_numpy(g).to(d)
        tv = float(rt.B.update(rt.ctx, grids, view, vg, lr, tvw).item())
        val, dtv = ref.np_tv(p[view])
        assert abs(tv - tvw * val) <= 1e-4 * max(tvw * val, 1e-12)
        t[view] += 1
        p[view], m[view], v[view] = ref.adam_ref(p[view], g.astype(np.float64) + tvw * dtv, m[view], v[view], t[view], lr)
        assert grids.steps == t
    got = grids.grids.cpu().numpy().astype(np.float64)
    assert np.abs(got - p).max() <= 1e-5, np.abs(got - p).max()
    np.testing.assert_allclose(grids.m.cpu().numpy(), m, rtol=1e-3, atol=1e-9)


def _train_case(rt, n=20_000, w=192, h=128, seed=123, depth=False):
    cam, tr, sh, op = synthetic_scene(n, w, h, k=4, seed=seed)
    d = rt.ctx.device
    out = rt.R.render_splats(rt.ctx, cam, (w, h), *(torch.from_numpy(x).to(d) for x in (tr, sh, op)), render_depth=True)
    # a colour-shifted target: the grid has something to learn
    rgb = (out.out_img[..., :3] * torch.tensor([1.2, 0.9, 0.8], device=d) + 0.03).clamp(0, 1)
    packed = torch.cat([(rgb * 255).round().to(torch.uint8), torch.full((h, w, 1), 255, dtype=torch.uint8, device=d)], -1)
    gt = packed.view(torch.int32).reshape(h, w).contiguous()
    kw = {}
    if depth:
        a = out.out_img[..., 3]
        t = torch.where(a > 0.05, out.depth / a.clamp_min(1e-30) * 1.05, torch.zeros_like(a)).contiguous()
        kw = dict(depth=t, depth_count=int((t > 0).sum()))
    return cam, tr, sh, op, rt.T.SceneBatch(img_packed=gt, camera=cam, view_index=1, **kw)


def _run(rt, cfg, batch, tr, sh, op, fused, steps=3):
    d = rt.ctx.device
    s = rt.T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr, sh + np.float32(0.1), op)))
    grids = rt.B.BilateralGrids(3, d)
    t = rt.T.SplatTrainer(cfg, rt.ctx, rt.T.bounds_from_pos(0.8, tr[:, :3]), bilateral_grids=grids)
    losses = []
    for _ in range(steps):
        st = (t.step_fused if fused else t.step)(batch, s)
        losses.append((float(st.loss.item()), float(st.tv_loss.item()),
                       None if st.depth_loss is None else float(st.depth_loss.item())))
    return s, t, grids, losses


def _close_state(s_a, t_a, g_a, s_b, t_b, g_b):
    for name in ("transforms", "sh_coeffs", "raw_opacities"):
        a, b = getattr(s_a, name).double(), getattr(s_b, name).double()
        assert torch.isfinite(b).all()
        close = (a - b).abs() <= 1e-6 + 1e-4 * a.abs()
        assert close.double().mean() > 0.995, (name, float(close.double().mean()))
    for key in ("m_t", "m_sh", "m_o"):
        a, b = t_a._state[key].double(), t_b._state[key].double()
        assert ((a - b).abs() <= 1e-9 + 1e-3 * a.abs()).double().mean() > 0.99, key
    for name in ("grids", "m", "v"):
        a, b = getattr(g_a, name).double(), getattr(g_b, name).double()
        assert ((a - b).abs() <= 1e-7 + 1e-4 * a.abs()).double().mean() > 0.995, name
    assert g_a.steps == g_b.steps == [0, 3, 0]


@pytest.mark.parametrize("depth", [False, True])
def test_fused_step_matches_host_orchestrated_step(rt, depth):
    cam, tr, sh, op, batch = _train_case(rt, depth=depth)
    cfg = rt.T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, seed=7, bilateral_grid=True,
                           depth_loss_weight=0.3 if depth else 0.0)
    s_a, t_a, g_a, l_a = _run(rt, cfg, batch, tr, sh, op, fused=False)
    s_b, t_b, g_b, l_b = _run(rt, cfg, batch, tr, sh, op, fused=True)
    for (la, tva, da), (lb, tvb, db) in zip(l_a, l_b):
        assert abs(la - lb) <= 2e-4 * abs(la)
        assert abs(tva - tvb) <= 1e-4 * abs(tva) + 1e-12
        if depth:
            assert da > 0 and abs(da - db) <= 2e-4 * abs(da)
    assert l_a[0][1] == 0.0 and l_a[-1][1] > 0.0            # identity start: no TV; the grid moved
    _close_state(s_a, t_a, g_a, s_b, t_b, g_b)
    assert not torch.equal(g_b.grids[1], g_b.grids[0])      # only the rendered view's grid changed
    assert torch.equal(g_b.grids[0], g_b.grids[2])


def test_fused_step_replays_under_cuda_graph(rt):
    cam, tr, sh, op, batch = _train_case(rt, n=10_000, seed=321)
    d = rt.ctx.device
    batch = rt.T.SceneBatch(img_packed=batch.img_packed.to(d), camera=cam, view_index=1)
    cfg = rt.T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, seed=7, bilateral_grid=True)
    s_e, _, g_e, l_e = _run(rt, cfg, batch, tr, sh, op, fused=True, steps=1)
    s_g = rt.T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr, sh + np.float32(0.1), op)))
    g_g = rt.B.BilateralGrids(3, d)
    t_g = rt.T.SplatTrainer(cfg, rt.ctx, rt.T.bounds_from_pos(0.8, tr[:, :3]), bilateral_grids=g_g)
    t_g._ensure_state(s_g)
    need = int(rt.lib.load().bg_train_step_bilagrid_workspace_bytes(s_g.num_splats(), 4, *reversed(batch.img_size())))
    t_g._fused_ws = torch.empty(need, dtype=torch.uint8, device=d)
    t_g._fused_loss = torch.zeros(1, dtype=torch.float32, device=d)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        st_g = t_g.step_fused(batch, s_g)
    graph.replay()
    torch.cuda.synchronize()
    assert abs(float(st_g.loss.item()) - l_e[0][0]) <= 2e-4 * abs(l_e[0][0])
    for name in ("transforms", "sh_coeffs", "raw_opacities"):
        a, b = getattr(s_e, name).double(), getattr(s_g, name).double()
        assert ((a - b).abs() <= 1e-6 + 1e-4 * a.abs()).double().mean() > 0.995, name
    a, b = g_e.grids.double(), g_g.grids.double()
    assert ((a - b).abs() <= 1e-7 + 1e-4 * a.abs()).double().mean() > 0.995


def test_argument_errors(rt):
    """Tensors of the wrong dtype, shape or device, and overlapping outputs, are refused before any launch."""
    d = rt.ctx.device
    h, w = 24, 40
    grid, img, v_out = (torch.from_numpy(x).to(d) for x in _inputs(h, w, 77))
    bad_grids = [grid.double(), grid[:4], grid.cpu(), grid.reshape(-1)[:-12].reshape(-1)]
    for g in bad_grids:
        with pytest.raises(ValueError):
            rt.B.slice(rt.ctx, g, img)
        with pytest.raises(ValueError):
            rt.B.slice_backward(rt.ctx, g, img, v_out)
    with pytest.raises(ValueError):
        rt.B.slice(rt.ctx, grid, img, out=torch.empty((h, w - 1, 4), device=d))
    with pytest.raises(ValueError):
        rt.B.slice(rt.ctx, grid, img, out=img)                                        # in place over the input
    with pytest.raises(ValueError):
        rt.B.slice_backward(rt.ctx, grid, img, v_out, v_grid=torch.empty(100, device=d))   # short gradient buffer
    with pytest.raises(ValueError):
        rt.B.slice_backward(rt.ctx, grid, img, v_out, v_img=img)
    with pytest.raises(ValueError):
        rt.B.slice_backward(rt.ctx, grid, img, v_out[:, 1:].contiguous())
    grids = rt.B.BilateralGrids(2, d)
    with pytest.raises(ValueError):
        rt.B.update(rt.ctx, grids, 0, torch.empty(100, device=d), 1e-3, 10.0)
    assert grids.steps == [0, 0]
    # the C boundary refuses overlap too, with the images' own extent
    lib, L = rt.lib.load(), rt.lib
    buf = torch.empty((2 * h, w, 4), device=d)
    s = 0
    assert lib.bg_bilagrid_slice(rt.ctx.handle, s, grid.data_ptr(), buf.data_ptr(), h, w, buf[h // 2].data_ptr()) == L.BG_ERR_INVALID
    assert lib.bg_bilagrid_slice(rt.ctx.handle, s, grid.data_ptr(), buf.data_ptr(), h, w, buf[h].data_ptr()) == L.BG_OK
    vg = torch.empty((8, 16, 16, 12), device=d)
    assert lib.bg_bilagrid_slice_backward(rt.ctx.handle, s, grid.data_ptr(), buf.data_ptr(), v_out.data_ptr(), h, w,
                                          buf[1].data_ptr(), vg.data_ptr()) == L.BG_ERR_INVALID
    v2 = torch.empty((2 * h, w, 4), device=d)
    assert lib.bg_bilagrid_slice_backward(rt.ctx.handle, s, grid.data_ptr(), img.data_ptr(), v2.data_ptr(), h, w,
                                          v2[1].data_ptr(), vg.data_ptr()) == L.BG_ERR_INVALID
    assert lib.bg_bilagrid_slice_backward(rt.ctx.handle, s, grid.data_ptr(), img.data_ptr(), v2.data_ptr(), h, w,
                                          v2.data_ptr(), vg.data_ptr()) == L.BG_OK
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------- it helps
def _surface_scene(n, seed):
    r = np.random.default_rng(seed)
    x, y = r.uniform(-1.6, 1.6, n), r.uniform(-1.2, 1.2, n)
    z = 4.0 + 0.3 * np.sin(1.3 * x) * np.cos(1.1 * y)
    means = np.stack([x, y, z], 1)
    quats = np.tile([1.0, 0.0, 0.0, 0.0], (n, 1))
    log_scales = np.full((n, 3), math.log(0.04))
    sh = r.uniform(-1.2, 1.2, (n, 1, 3))
    op = np.full(n, 3.0)
    return (np.concatenate([means, quats, log_scales], 1).astype(np.float32), sh.astype(np.float32), op.astype(np.float32))


def test_grids_absorb_per_view_colour_distortion(rt):
    """Training views carry a per-view, luminance-dependent colour distortion (channel gains in [0.6, 1.4], an offset,
    a tone curve); held-out views are clean.  With grids the model explains the distortion with the grids and renders
    the held-out views better; the sliced training renders match their distorted images better than the raw renders.
    Measured on an H100 80 GB HBM3 at a 700 W power limit: held-out PSNR 23.38 dB without grids, 23.96 dB with them
    (+0.57 dB, below the 1 dB first assumed); the test asks for +0.3 dB.  On the training views the sliced renders'
    MSE against the distorted images was 13 % below the raw renders' (0.0767 against 0.0882, summed over the views)."""
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
        out = rt.R.render_splats(rt.ctx, cam, (w, h), *hidden)
        return out.out_img[..., :3].clamp(0, 1)

    def pack(rgb):
        q = torch.cat([(rgb * 255).round().to(torch.uint8), torch.full((h, w, 1), 255, dtype=torch.uint8, device=d)], -1)
        return q.view(torch.int32).reshape(h, w).contiguous()

    batches, distorted = [], []
    for i, cam in enumerate(train_cams):
        gain = torch.tensor(rng.uniform(0.6, 1.4, 3), dtype=torch.float32, device=d)
        offset = torch.tensor(rng.uniform(-0.05, 0.05, 3), dtype=torch.float32, device=d)
        gamma = float(rng.uniform(0.7, 1.4))
        rgb = (render_rgb(cam).pow(gamma) * gain + offset).clamp(0, 1)
        distorted.append(rgb)
        batches.append(rt.T.SceneBatch(img_packed=pack(rgb), camera=cam, view_index=i))
    eval_gt = [(render_rgb(c) * 255).round().to(torch.uint8).cpu().numpy() for c in eval_cams]
    r = np.random.default_rng(5)
    tr0 = tr.copy()
    tr0[:, :3] += r.normal(0.0, 0.02, (tr.shape[0], 3)).astype(np.float32)
    sh0 = r.uniform(-0.5, 0.5, sh.shape).astype(np.float32)
    steps = 600
    res, models = {}, {}
    for use in (False, True):
        cfg = rt.T.TrainConfig(total_train_iters=steps, mean_noise_weight=0.0, background_noise_strength=0.0, seed=3,
                               bilateral_grid=use)
        s = rt.T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr0, sh0, op)))
        grids = rt.B.BilateralGrids(len(batches), d) if use else None
        t = rt.T.SplatTrainer(cfg, rt.ctx, rt.T.bounds_from_pos(0.8, tr0[:, :3]), bilateral_grids=grids)
        for i in range(steps):
            t.step_fused(batches[i % len(batches)], s)
        res[use] = float(np.mean([float(eval_stats(rt.ctx, s, c, g).psnr) for c, g in zip(eval_cams, eval_gt)]))
        models[use] = (s, grids)
    print(f"held-out PSNR without grids {res[False]:.2f} dB, with grids {res[True]:.2f} dB")
    assert res[True] > res[False] + 0.3, res
    s, grids = models[True]
    raw_err, sliced_err = 0.0, 0.0
    for i, cam in enumerate(train_cams):
        out = rt.R.render_splats(rt.ctx, cam, (w, h), s.transforms, s.sh_coeffs, s.raw_opacities)
        sliced = rt.B.apply_bilateral_grid(rt.ctx, out.out_img, grids, i)
        raw_err += float((out.out_img[..., :3] - distorted[i]).pow(2).mean())
        sliced_err += float((sliced[..., :3] - distorted[i]).pow(2).mean())
    print(f"training views: raw MSE {raw_err / len(train_cams):.3e}, sliced MSE {sliced_err / len(train_cams):.3e}")
    assert sliced_err < raw_err


def test_train_loop_reports_colour_corrected_metrics(tmp_path):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import train_colmap
    kw = dict(iters=40, views=10, width=128, height=96, hidden_n=3_000, init_points=1_500, max_splats=10_000, quiet=True)
    on = train_colmap.run(root=str(tmp_path / "on"), bilateral_grid=True, **kw)["eval"]
    assert {"cc_psnr", "cc_ssim"} <= set(on) and math.isfinite(on["cc_psnr"]) and 0 < on["cc_ssim"] <= 1
    assert on["cc_psnr"] >= on["psnr"] - 0.05     # the affine fit can only help, up to the 8-bit rounding
    off = train_colmap.run(root=str(tmp_path / "off"), **kw)["eval"]
    assert "cc_psnr" not in off and "cc_ssim" not in off


def test_new_kernels_are_sm90a_only_and_do_not_spill():
    obj = os.path.join(ROOT, "brush_b200", "csrc", "_obj", "bilagrid.o")
    txt = open(obj + ".ptxas.txt").read()
    found = 0
    for m in re.finditer(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", txt):
        assert (m.group(2), m.group(3), m.group(4)) == ("0", "0", "0"), m.group(0)
        found += 1
    assert found == 3
    assert set(re.findall(r"for '(sm_\w+)'", txt)) == {"sm_90a"}
    sass = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    for k in ("bilagrid_slice_kernel", "bilagrid_slice_bwd_kernel", "bilagrid_tv_kernel"):
        assert k in sass, k
    assert set(re.findall(r"arch = (sm_\w+)", sass)) == {"sm_90a"}
