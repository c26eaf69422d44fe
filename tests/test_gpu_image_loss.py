"""The image-loss kernels (bg_image_loss_fused, bg_image_loss_forward / _backward) and the train step's loss scalar
against the float64 restatement of tests/image_loss_ref.py, at the shapes, layouts and values where their index
arithmetic can go wrong: images smaller than the 11-tap window or one tile, the switch between interior and border
tiles of the fused kernel (a 32-wide tile is interior when x0 >= 10 and x0 + 42 <= W: W = 73/74 and 105/106/107 sit on
the edge), 1080p and 4K, every pred layout the strided addressing accepts, predictions outside [0, 1], exact ties,
constant blocks (variance rounding below 0), masked-out regions and the 4-channel alpha term.

Yardstick, per channel (as in test_gpu_blend_opaque.py): the C oracle's own error against the reference on the same
inputs.  ||gpu - ref|| <= k ||orc - ref|| + 4e-6 ||ref||, and element-wise |gpu - ref| <= tol * scale on all but 1e-4 of
the elements, where scale is |l1_w| + |ssim_w| for the map and max(max |ref|, max(dl) (|l1_w| + |ssim_w|)) for the
gradient.  k = 2 and tol = 1e-5, except on the constant-block regime: k = 4 and tol = 2e-3.  Pixels whose L1 sign is a
rounding decision (|pred - gt_eff| within 4 ulps, not 0) leave the L2 sums and may differ by one sign flip, 2 l1_w dl.
The tie regime (pred equal to the decoded GT, gradient ~0 there) is held to the element-wise absolute bound only.

Measured on an H100 80GB HBM3 (SXM, 700 W power limit), over the 123 fused cases and 31 unfused ones:
- gpu relative L2 error <= 2.9e-6 outside the constant blocks; element-wise <= 2.2e-6 of scale.  Wherever the
  relative error exceeds 1e-6, the ratio gpu / oracle is <= 1.0 on the unfused map and <= 2 on the fused gradient
  but for one case: 6.2 at 2.0e-6 relative (1 x 107, SSIM only, composited and masked).  Ratios up to 14 occur at
  relative errors of 1e-7..3e-7.  At that level both errors are a few f32 roundings.  The fused kernel rounds in a
  different order from the oracle (sums by input position in paired FMAs, and correctly rounded reciprocals for the
  four SSIM quotients), so their ratio is noise.  Hence the floor is 4e-6 ||ref|| (~70 ulps), not 1e-6.
- constant 16 x 16 blocks: relative L2 error up to 3.8e-4, element-wise 1.6e-4 of scale; ratio up to 3.4 (unfused
  map) and 2.8 (fused gradient).  Inside a constant block sigma^2 = E[x^2] - mu^2 cancels to f32 noise of about 1e-4
  of C2 (test_image_loss_ref_cpu.py).  Which pixels get how much of it depends on the rounding of each window sum:
  FMA contraction on the device, the fused kernel's order.  So the GPU's and the oracle's errors are two samples of
  the same noise, not one error and its double.  Hence k = 4 there.
- the train step's loss scalar: 6.3e-7 (rgb) and 5.2e-7 (alpha, composited) of sum |terms|; eval_stats at
  1079 x 1917: PSNR within 1.3e-7 dB, SSIM within 5.4e-7.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from image_loss_ref import gt_effective, loss_and_grad, loss_map, pack_rgba, weighted_sum  # noqa: E402
from test_image_loss_ref_cpu import REGIMES, grad_scale, make_case, near_ties  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAYOUTS = ("hwc4", "hwc3", "chw", "slice", "transposed")
OPTIONS = ((None, False), ((0.2, 0.4, 0.6), False), (None, True), ((0.7, 0.1, 0.3), True))   # composite bg, mask
WEIGHTS = ((0.8, -0.2), (1.0, 0.0), (0.0, 1.0))
SHAPES = [(1, 1), (1, 2), (2, 1), (1, 107), (107, 1), (2, 5), (5, 11), (11, 5), (11, 16), (16, 17), (17, 31), (31, 32),
          (32, 33), (33, 42), (42, 43), (43, 52), (52, 53), (53, 73), (73, 74), (74, 73), (74, 105), (105, 106),
          (106, 107), (107, 106)]


def _small_cases():
    """Every (shape, regime) pair once; the 120 (layout, channels, options, weights) combinations spread over them by a
    bijection, so each appears exactly once (hwc3 with 4 channels runs as hwc4)."""
    out = []
    for r, regime in enumerate(REGIMES):
        for s, (h, w) in enumerate(SHAPES):
            j = ((r * len(SHAPES) + s) * 7) % 120
            layout, channels = LAYOUTS[j % 5], (3, 4)[(j // 5) % 2]
            if layout == "hwc3" and channels == 4:
                layout = "hwc4"
            out.append((h, w, regime, layout, channels, (j // 10) % 4, (j // 40) % 3))
    return out


SMALL = _small_cases()
LARGE = [(1080, 1920, "uniform", "hwc4", 3, 0, 0), (1079, 1917, "alpha0", "slice", 4, 3, 0),
         (2160, 3840, "uniform", "hwc4", 3, 0, 0)]
MEASURED = []   # (case and quantity, gpu/orc L2 ratio, gpu rel L2, max elem err / scale), printed at the end


@pytest.fixture(scope="module")
def rt():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import brush_b200.loss as L
    import brush_b200.render as R
    import brush_b200.train as T
    from brush_b200 import _lib
    from oracle import oracle as orc

    class RT:
        pass

    r = RT()
    r.L, r.R, r.T, r.orc, r.lib = L, R, T, orc, _lib
    r.ctx = R.RenderContext(max_splats=1 << 18, max_w=1920, max_h=1080, max_intersections=1 << 24)
    yield r
    r.ctx.close()
    if MEASURED:
        print("\nimage-loss yardstick (ratio, gpu rel L2, max elem / scale):")
        for m in MEASURED:
            print("  " + " ".join(str(x) for x in m))


def _layout(pred4: np.ndarray, layout: str, dev) -> torch.Tensor:
    """pred4 [4,h,w] f32 -> an [h,w,C'] view with the named memory layout."""
    h, w = pred4.shape[1:]
    hwc = torch.from_numpy(np.ascontiguousarray(pred4.transpose(1, 2, 0))).to(dev)
    if layout == "hwc4":
        return hwc
    if layout == "hwc3":
        return hwc[..., :3].contiguous()
    if layout == "chw":
        return torch.from_numpy(np.ascontiguousarray(pred4)).to(dev).permute(1, 2, 0)
    if layout == "slice":
        base = torch.full((h, w + 13, 4), 7.0, dtype=torch.float32, device=dev)
        base[:, 5:5 + w] = hwc
        return base[:, 5:5 + w]
    if layout == "transposed":
        return hwc.transpose(0, 1).contiguous().transpose(0, 1)
    raise ValueError(layout)


def _chain(channels, h, w):
    """The train step's dL/dmap per channel (api.cu view_loss), in f32."""
    npx = np.float32(w) * np.float32(h)
    c = [np.float32(1.0) / (np.float32(3.0) * npx)] * 3 + ([np.float32(0.1) / npx] if channels == 4 else [])
    return [float(x) for x in c]


def _yardstick(name, gpu, ref, orc, ok, scale, tol, flip, ratio_check=True, k=2.0):
    """Failure messages for one channel; records the measured ratio."""
    gpu, orc = gpu.astype(np.float64), orc.astype(np.float64)
    d = np.abs(gpu - ref)
    e, eo, nrm = (float(np.linalg.norm(x[ok])) for x in (gpu - ref, orc - ref, ref))
    MEASURED.append((name, f"{e / eo if eo > 0 else float('nan'):.2f}", f"{e / max(nrm, 1e-30):.1e}",
                     f"{d[ok].max() / scale if ok.any() else 0.0:.1e}"))
    fails = []
    if ratio_check and e > k * eo + 4e-6 * nrm:
        fails.append(f"{name}: ||gpu-ref|| {e:.3e} > {k} ||orc-ref|| {eo:.3e} + 4e-6 ||ref|| {nrm:.3e}")
    bad = (d > tol * scale) & ok
    if bad.sum() > 1e-4 * d.size:
        fails.append(f"{name}: {bad.sum()} of {d.size} beyond {tol} x {scale:.3e} (max {d[ok].max():.3e})")
    if (d[~ok] > flip + tol * scale).any():
        fails.append(f"{name}: a near-tie pixel differs by more than one L1 sign flip")
    return fails


def _ref_device(h, w):
    return "cuda" if h * w > 200_000 else "cpu"


def _run_fused(rt, h, w, regime, layout, channels, opt, wts, seed):
    bg, mask = OPTIONS[opt]
    if regime == "alpha0":
        mask = True
    l1_w, ssim_w = WEIGHTS[wts]
    pred4, packed = make_case(h, w, channels, regime, seed, bg, mask)
    d = rt.ctx.device
    tp = _layout(pred4, layout, d)
    tg = torch.from_numpy(packed.view(np.int32)).to(d)
    cfg = rt.L.ImageLossConfig(l1_w, ssim_w, bg, mask)
    chain = _chain(channels, h, w)
    g, loss = rt.L.image_loss_fused(rt.ctx, tp, tg, channels, cfg, chain)
    g = g.permute(2, 0, 1).cpu().numpy()
    pred_c = np.ascontiguousarray(pred4[:channels])
    ref_map, ref_g = loss_and_grad(pred_c, packed, np.array(chain, np.float32), l1_w, ssim_w, bg, mask, _ref_device(h, w))
    dl = np.broadcast_to(np.array(chain, np.float32)[:, None, None], (channels, h, w)).copy()
    og = rt.orc.image_loss_backward(pred_c, packed, dl, l1_w, ssim_w, bg=bg, mask=mask)
    return dict(pred_c=pred_c, packed=packed, bg=bg, mask=mask, l1_w=l1_w, ssim_w=ssim_w, chain=chain, g=g,
                loss=float(loss.item()), ref_map=ref_map, ref_g=ref_g, og=og, dl=dl, tp=tp, tg=tg, cfg=cfg)


def _check_grad(tag, r, regime, gpu_g, ref_g, og, dl):
    channels = ref_g.shape[0]
    ok = np.ones_like(ref_g, bool)
    ok[:3] &= ~near_ties(r["pred_c"], r["packed"], r["bg"])
    scale = grad_scale(ref_g, dl, r["l1_w"], r["ssim_w"])
    tol = 2e-3 if regime == "const" else 1e-5
    fails = []
    for c in range(channels):
        flip = 2.0 * abs(r["l1_w"]) * float(dl[c].max())
        fails += _yardstick(f"{tag} grad[{c}]", gpu_g[c], ref_g[c], og[c], ok[c], scale, tol, flip, regime != "ties",
                            4.0 if regime == "const" else 2.0)
    return fails


def _check_fused(tag, r, regime, channels):
    fails = _check_grad(tag, r, regime, r["g"][:channels], r["ref_g"], r["og"], r["dl"])
    if r["g"].shape[0] > channels:
        assert (r["g"][channels:] == 0).all(), f"{tag}: output channels beyond {channels} were written"
    exp = weighted_sum(r["ref_map"], r["chain"])
    mag = sum(r["chain"][c] * float(np.abs(r["ref_map"][c]).sum()) for c in range(channels))
    tol = 1e-5 * mag + 1e-12
    if regime == "const":   # plus the map's own f32 noise on constant blocks, at its element-wise bound
        tol += 2e-3 * (abs(r["l1_w"]) + abs(r["ssim_w"])) * sum(r["chain"]) * r["ref_map"][0].size
    if abs(r["loss"] - exp) > tol:
        fails.append(f"{tag}: loss {r['loss']!r} vs {exp!r} (sum |terms| {mag:.3e})")
    if r["mask"]:   # masked-out pixels: map exactly zero; gradient exactly zero where the whole +-10 window is masked out
        ga = (r["packed"] >> 24) == 0
        if ga.any():
            assert (r["ref_map"][:, ga] == 0).all()
            h, w = ga.shape
            pad = np.pad(ga, 10, constant_values=False)
            dead = np.ones_like(ga)
            for dy in range(21):
                for dx in range(21):
                    dead &= pad[dy:dy + h, dx:dx + w]
            if dead.any():
                assert (r["g"][:channels][:, dead] == 0).all(), f"{tag}: gradient inside a masked-out region"
    return fails


def _id(case):
    h, w, regime, layout, channels, opt, wts = case
    return f"{h}x{w}-{regime}-{layout}-c{channels}-o{opt}-w{wts}"


@pytest.mark.parametrize("case", SMALL + LARGE, ids=_id)
def test_fused_vs_reference(rt, case):
    h, w, regime, layout, channels, opt, wts = case
    r = _run_fused(rt, h, w, regime, layout, channels, opt, wts, seed=h * 1009 + w)
    fails = _check_fused(_id(case), r, regime, channels)
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("case", SMALL[::4] + LARGE[1:2], ids=_id)
def test_unfused_forward_backward_and_fused_agreement(rt, case):
    """The 16x16-tile forward and backward with a non-uniform dL/dmap against the reference; then the fused kernel
    against them: its gradient equals the backward with the constant chain, its loss the chain-weighted sum of the
    forward map, to f32 rounding."""
    h, w, regime, layout, channels, opt, wts = case
    r = _run_fused(rt, h, w, regime, layout, channels, opt, wts, seed=h * 1013 + w)
    d = rt.ctx.device
    m = rt.L.image_loss_forward(rt.ctx, r["tp"], r["tg"], channels, r["cfg"]).cpu().numpy()
    om = rt.orc.image_loss_forward(r["pred_c"], r["packed"], r["l1_w"], r["ssim_w"], bg=r["bg"], mask=r["mask"])
    dl = np.random.default_rng(h + w).uniform(0.1, 1.0, (channels, h, w)).astype(np.float32)
    ref_map, ref_g = loss_and_grad(r["pred_c"], r["packed"], dl, r["l1_w"], r["ssim_w"], r["bg"], r["mask"], _ref_device(h, w))
    og = rt.orc.image_loss_backward(r["pred_c"], r["packed"], dl, r["l1_w"], r["ssim_w"], bg=r["bg"], mask=r["mask"])
    g = rt.L.image_loss_backward(rt.ctx, r["tp"], r["tg"], torch.from_numpy(dl).to(d), channels, r["cfg"])
    g = g.permute(2, 0, 1).cpu().numpy()
    tag = _id(case)
    mscale = abs(r["l1_w"]) + abs(r["ssim_w"])
    mtol = 2e-3 if regime == "const" else 1e-5
    fails = []
    allok = np.ones((h, w), bool)
    for c in range(channels):
        fails += _yardstick(f"{tag} map[{c}]", m[c], ref_map[c], om[c], allok, mscale, mtol, 0.0, regime != "ties",
                            4.0 if regime == "const" else 2.0)
    fails += _check_grad(tag + " unfused", r, regime, g[:channels], ref_g, og, dl)
    if g.shape[0] > channels:
        assert (g[channels:] == 0).all()
    if r["mask"]:
        ga = (r["packed"] >> 24) == 0
        assert (m[:, ga] == 0).all(), "masked-out map values must be zero"
    assert not fails, "\n".join(fails)
    # fused == forward -> sum(chain * map) -> backward with the constant chain
    fwd_loss = sum(r["chain"][c] * float(m[c].astype(np.float64).sum()) for c in range(channels))
    mag = sum(r["chain"][c] * float(np.abs(m[c]).astype(np.float64).sum()) for c in range(channels))
    tol = 1e-5 * mag + 1e-12
    if regime == "const":   # the two kernels' maps differ by the constant blocks' f32 noise (element-wise bound above)
        tol += 2e-3 * mscale * sum(r["chain"]) * h * w
    assert abs(r["loss"] - fwd_loss) <= tol, (r["loss"], fwd_loss, mag)
    gc = rt.L.image_loss_backward(rt.ctx, r["tp"], r["tg"], torch.from_numpy(r["dl"]).to(d), channels, r["cfg"])
    gc = gc.permute(2, 0, 1).cpu().numpy()[:channels]
    scale = grad_scale(r["ref_g"], r["dl"], r["l1_w"], r["ssim_w"])
    diff = np.abs(gc.astype(np.float64) - r["g"][:channels])
    ok = np.ones_like(diff, bool)
    ok[:3] &= ~near_ties(r["pred_c"], r["packed"], r["bg"])
    assert (diff[ok] <= (2e-3 if regime == "const" else 1e-5) * scale).all(), diff[ok].max() / scale


def _fused_raw(rt, tp, tg, channels, cfg, chain):
    """bg_image_loss_fused straight through the ABI: (dL/dpred, per-block partials)."""
    import ctypes as C
    lib = rt.lib.load()
    h, w = tp.shape[0], tp.shape[1]
    out = torch.zeros_like(tp)
    part = torch.empty(int(lib.bg_image_loss_num_partials(channels, h, w)), dtype=torch.float32, device=tp.device)
    sy, sx, sc = tp.stride()
    rt.lib.check(lib.bg_image_loss_fused(rt.ctx.handle, rt.R._stream_ptr(rt.ctx.device), tp.data_ptr(), tg.data_ptr(), channels,
                                         h, w, sc, sy, sx, cfg.l1_weight, cfg.ssim_weight, None, int(cfg.mask),
                                         (C.c_float * channels)(*chain), out.data_ptr(), part.data_ptr()), "bg_image_loss_fused")
    return out, part


def test_fused_is_deterministic(rt):
    h, w = 1080, 1920
    pred4, packed = make_case(h, w, 4, "wide", 5, None, True)
    d = rt.ctx.device
    tp = _layout(pred4, "hwc4", d)
    tg = torch.from_numpy(packed.view(np.int32)).to(d)
    cfg = rt.L.ImageLossConfig(0.8, -0.2, None, True)
    a = _fused_raw(rt, tp, tg, 4, cfg, _chain(4, h, w))
    b = _fused_raw(rt, tp, tg, 4, cfg, _chain(4, h, w))
    torch.cuda.synchronize()
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32))
    assert torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))


_CAPTURE = r"""
import json, sys
import numpy as np
import torch
sys.path.insert(0, sys.argv[1])
import brush_b200.loss as L
import brush_b200.render as R
ctx = R.RenderContext(1024, 256, 256)
d = ctx.device
h, w = 157, 203
rng = np.random.default_rng(4)
pred = torch.from_numpy(rng.uniform(0, 1, (h, w, 4)).astype(np.float32)).to(d)
gt8 = rng.integers(0, 256, (h, w, 4), dtype=np.uint32)
gt = torch.from_numpy((gt8[..., 0] | gt8[..., 1] << 8 | gt8[..., 2] << 16 | gt8[..., 3] << 24).astype(np.uint32).view(np.int32)).to(d)
cfg = L.ImageLossConfig(0.8, -0.2, (0.2, 0.4, 0.6), True)
chain = [1.0 / (3 * h * w)] * 3 + [0.1 / (h * w)]
weights = torch.tensor(chain, dtype=torch.float32, device=d)
out = torch.zeros((h, w, 4), dtype=torch.float32, device=d)
torch.cuda.synchronize()
graph = torch.cuda.CUDAGraph()
with torch.cuda.graph(graph):   # the first fused-loss call of the process
    g_cap, loss_cap = L.image_loss_fused(ctx, pred, gt, 4, cfg, chain, out, weights=weights)
out.fill_(float("nan"))
graph.replay()
torch.cuda.synchronize()
g_eager, loss_eager = L.image_loss_fused(ctx, pred, gt, 4, cfg, chain, weights=weights)
torch.cuda.synchronize()
print(json.dumps(dict(grad=bool(torch.equal(g_cap.view(torch.int32), g_eager.view(torch.int32))),
                      loss=bool(torch.equal(loss_cap.view(torch.int32), loss_eager.view(torch.int32))),
                      finite=bool(torch.isfinite(g_cap).all()), loss_value=float(loss_cap))))
ctx.close()
"""


def test_first_fused_call_can_be_captured():
    """A process whose first fused-loss call is captured into a CUDA graph (torch's global capture mode): the capture
    succeeds and one replay equals a later eager call bit for bit."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    r = subprocess.run([sys.executable, "-c", _CAPTURE, ROOT], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["grad"] and res["loss"] and res["finite"], res


@pytest.mark.parametrize("alpha", [False, True], ids=["rgb", "alpha"])
def test_train_step_loss_scalar(rt, alpha):
    """step_fused's first-step loss (bg_train_step: the fused kernel's partials reduced by launch_loss_reduce with the
    chain of the loss setup) against the float64 loss of the same render.  The scalar is an f32 sum through a fixed
    tree: per-thread runs of <= 16 map values, a 32-lane shuffle tree and 8 warp sums per 32x32 tile, then per channel
    256 strided runs of <= 32 partials (8160 tiles at 4K) and a 256-way tree: about 70 f32 roundings deep, so at most
    ~70 * 6e-8 = 4e-6 of the sum of |terms|, on top of the map's own ~1e-6.  Bound: 1e-5 of sum_c chain[c] sum |map[c]|."""
    from brush_b200.render import PASS_BACKWARD
    from scenes import synthetic_scene
    T = rt.T
    n, w, h = 60_000, 1920, 1080
    cam, tr, sh, op = synthetic_scene(n, w, h, k=4, seed=77)
    d = rt.ctx.device
    bgc = (0.1, 0.2, 0.3) if alpha else (0.0, 0.0, 0.0)
    rng = np.random.default_rng(8)
    gt8 = rng.integers(0, 256, (h, w, 4), dtype=np.uint32)
    if not alpha:
        gt8[..., 3] = 255
    packed = pack_rgba(gt8)
    out = rt.R.render_splats(rt.ctx, cam, (w, h), *(torch.from_numpy(x.copy()).to(d) for x in (tr, sh, op)), mip=False,
                             background=bgc, rpass=PASS_BACKWARD)
    img = out.out_img.permute(2, 0, 1).double()
    cfg = T.TrainConfig(background_noise_strength=0.0, background_color=bgc, total_train_iters=100)
    trainer = T.SplatTrainer(cfg, rt.ctx, T.bounds_from_pos(0.8, tr[:, :3]))
    splats = T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr, sh, op)))
    batch = T.SceneBatch(img_packed=torch.from_numpy(packed.view(np.int32)), camera=cam, has_alpha=alpha)
    st = trainer.step_fused(batch, splats)
    got = float(st.loss.item())
    channels = 4 if alpha else 3
    with torch.no_grad():
        m = loss_map(img[:channels], packed, 0.8, -0.2, bgc if alpha else None, False).cpu().numpy()
    chain = _chain(channels, h, w)
    exp = weighted_sum(m, chain)
    mag = sum(chain[c] * float(np.abs(m[c]).sum()) for c in range(channels))
    MEASURED.append((f"step loss {'alpha' if alpha else 'rgb'}", f"rel {abs(got - exp) / mag:.1e}"))
    assert abs(got - exp) <= 1e-5 * mag, (got, exp, mag)


def test_eval_stats_vs_float64(rt):
    """eval_stats at 1079 x 1917: PSNR from the mean squared L1 map and SSIM as the mean SSIM map of the returned 8-bit
    render, against float64 on the same image."""
    from brush_b200.eval import eval_stats
    from scenes import synthetic_scene
    n, w, h = 40_000, 1917, 1079
    cam, tr, sh, op = synthetic_scene(n, w, h, k=4, seed=31)
    d = rt.ctx.device
    gt = np.random.default_rng(12).integers(0, 256, (h, w, 3), dtype=np.uint8)
    splats = rt.T.Splats(*(torch.from_numpy(x).to(d) for x in (tr, sh, op)))
    s = eval_stats(rt.ctx, splats, cam, gt)
    rgb = s.rendered.permute(2, 0, 1).double()
    packed = pack_rgba(np.concatenate([gt, np.full((h, w, 1), 255, np.uint8)], 2))
    y = torch.from_numpy(gt_effective(packed)).to(d)
    mse = float(((rgb - y) ** 2).mean())
    psnr = 10.0 * np.log10(1.0 / mse)
    with torch.no_grad():
        ssim = float(loss_map(rgb, packed, 0.0, 1.0).mean())
    MEASURED.append(("eval", f"psnr {abs(float(s.psnr) - psnr):.1e}", f"ssim {abs(float(s.ssim) - ssim):.1e}"))
    assert abs(float(s.psnr) - psnr) <= 1e-4, (float(s.psnr), psnr)
    assert abs(float(s.ssim) - ssim) <= 5e-6, (float(s.ssim), ssim)
