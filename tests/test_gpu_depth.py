"""Differentiable depth on the GPU (DESIGN.md section 4.6): the DEPTH instantiations of the blend kernels against the
CPU oracle, their identity with the plain kernels where they must agree, the autograd path, argument errors and graph
capture."""
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from scenes import finite_diff_base_scene, random_v_output, splitmix64, synthetic_scene  # noqa: E402
from test_gpu_parity import _CAM_MODELS, _grad_close, _img_close, _model_camera  # noqa: E402


@pytest.fixture(scope="module")
def rt():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import brush_b200.render as R
    from brush_b200 import _lib
    from brush_b200.camera import build_uniforms
    from oracle import oracle as orc
    from oracle import oracle_depth as orcd

    class RT:
        pass

    r = RT()
    r.R, r.orc, r.orcd, r.lib, r.build_uniforms = R, orc, orcd, _lib, build_uniforms
    r.ctx = R.RenderContext(max_splats=1 << 18, max_w=1024, max_h=1024, max_intersections=1 << 23)
    yield r
    r.ctx.close()


def _dev(rt, *arrs):
    return tuple(torch.from_numpy(x).to(rt.ctx.device) for x in arrs)


def _v_depth(h, w, seed=0xDE0001):
    return splitmix64(seed, h * w).reshape(h, w).astype(np.float32)


def _depth_close(gpu, ref, zmax):
    """_img_close with the threshold-flip magnitude scaled by the largest depth of the scene."""
    return _img_close(gpu, ref, flip_mag=1.5 / 255 * 1.5 * zmax)


FWD_CASES = [(10_000, 256, 256, 16, False), (10_000, 250, 131, 1, False), (20_000, 320, 200, 4, True),
             (5_000, 96, 64, 9, False), (3_000, 64, 48, 25, True), (100_000, 640, 360, 16, False)]


@pytest.mark.parametrize("n,w,h,k,mip", FWD_CASES)
def test_depth_forward_vs_oracle(rt, n, w, h, k, mip):
    cam, tr, sh, op = synthetic_scene(n, w, h, k=k, seed=0xB2000000 + n + k)
    bg = (0.1, 0.2, 0.3)
    ttr, tsh, top = _dev(rt, tr, sh, op)
    plain = rt.R.render_splats(rt.ctx, cam, (w, h), ttr, tsh, top, mip=mip, background=bg)
    img, vis, rad, toff = (x.clone() for x in (plain.out_img, plain.visible, plain.max_radius, plain.tile_offsets()))
    out = rt.R.render_splats(rt.ctx, cam, (w, h), ttr, tsh, top, mip=mip, background=bg, render_depth=True)
    # everything but the depth is bit-identical to the plain forward
    assert out.depth is not None and tuple(out.depth.shape) == (h, w)
    assert torch.equal(out.out_img, img) and torch.equal(out.visible, vis) and torch.equal(out.max_radius, rad)
    assert torch.equal(out.tile_offsets(), toff)
    o = rt.orc.render_forward(rt.build_uniforms(cam, w, h), w, h, tr, sh, op, mip=mip, bg=bg)
    assert out.num_visible == o.num_visible
    np.testing.assert_array_equal(out.depths().cpu().numpy().view(np.uint32), o.depths_sorted.view(np.uint32))
    _depth_close(out.depth.cpu().numpy(), rt.orcd.render_depth(o), float(o.depths_sorted.max()))


@pytest.mark.parametrize("name", list(_CAM_MODELS))
def test_depth_forward_camera_models_vs_oracle(rt, name):
    model, params = _CAM_MODELS[name]
    n, w, h = 20_000, 320, 240
    cam0, tr, sh, op = synthetic_scene(n, w, h, k=4, seed=0xCA0000 + model)
    cam = _model_camera(cam0, model, params, 1.1, 0.9)
    o = rt.orc.render_forward(rt.build_uniforms(cam, w, h), w, h, tr, sh, op, bg=(0.1, 0.2, 0.3))
    out = rt.R.render_splats(rt.ctx, cam, (w, h), *_dev(rt, tr, sh, op), background=(0.1, 0.2, 0.3), render_depth=True)
    assert out.num_visible == o.num_visible
    _img_close(out.out_img.cpu().numpy(), o.out_img)
    _depth_close(out.depth.cpu().numpy(), rt.orcd.render_depth(o), float(o.depths_sorted.max()))


@pytest.mark.parametrize("n,w,h,k,mip,smooth", [(10_000, 256, 256, 16, False, False), (4_000, 100, 75, 1, True, False),
                                                (8_000, 160, 128, 9, False, True), (50_000, 480, 270, 16, False, False),
                                                (6_000, 200, 150, 4, True, True)])
def test_depth_backward_vs_oracle(rt, n, w, h, k, mip, smooth):
    cam, tr, sh, op = synthetic_scene(n, w, h, k=k, seed=0xB2001000 + n)
    bg = (0.05, 0.1, 0.15)
    rpass = 2 if smooth else 1
    o = rt.orc.render_forward(rt.build_uniforms(cam, w, h), w, h, tr, sh, op, mip=mip, bg=bg, rpass=rpass)
    v_out, v_d = random_v_output(h, w), _v_depth(h, w)
    ovc, ovz = rt.orcd.rasterize_backward_depth(o, v_out, v_d)
    ovt, ovsh, ovo, ovr = rt.orcd.project_backward_depth(o, ovc, ovz)
    ttr, tsh, top = _dev(rt, tr, sh, op)
    out = rt.R.render_splats(rt.ctx, cam, (w, h), ttr, tsh, top, mip=mip, background=bg, rpass=rpass, render_depth=True)
    vc, vz = rt.R.rasterize_bwd_depth(out, *_dev(rt, v_out, v_d))
    vt, vsh, vo, vr = rt.R.project_bwd(out, ttr, tsh, top, vc, v_z=vz)
    V = o.num_visible
    assert out.num_visible == V
    vc_np, vz_np = vc.cpu().numpy(), vz.cpu().numpy()
    assert np.isfinite(vc_np).all() and np.isfinite(vz_np).all()
    assert (vc_np[V:] == 0).all() and (vz_np[V:] == 0).all()
    for col, nm in enumerate(["v_xy_x", "v_xy_y", "v_conic_x", "v_conic_y", "v_conic_z", "v_r", "v_g", "v_b", "v_opac", "refine"]):
        _grad_close(vc_np[:V, col], ovc[:, col], name=nm)
    _grad_close(vz_np[:V], ovz, name="v_z")
    _grad_close(vt.cpu().numpy()[:, 0:3], ovt[:, 0:3], name="v_means")
    _grad_close(vt.cpu().numpy()[:, 3:7], ovt[:, 3:7], name="v_quats")
    _grad_close(vt.cpu().numpy()[:, 7:10], ovt[:, 7:10], name="v_log_scales")
    _grad_close(vsh.cpu().numpy(), ovsh, name="v_sh")
    _grad_close(vo.cpu().numpy(), ovo, name="v_raw_opac")
    _grad_close(vr.cpu().numpy(), ovr, name="v_refine")


@pytest.mark.parametrize("smooth", [False, True])
def test_zero_depth_gradient_matches_plain_backward(rt, smooth):
    n, w, h = 30_000, 320, 240
    cam, tr, sh, op = synthetic_scene(n, w, h, k=4, seed=0xDE0100)
    rpass = 2 if smooth else 1
    ttr, tsh, top = _dev(rt, tr, sh, op)
    (v_out,) = _dev(rt, random_v_output(h, w))
    out = rt.R.render_splats(rt.ctx, cam, (w, h), ttr, tsh, top, rpass=rpass, render_depth=True)
    vc0 = rt.R.rasterize_bwd(out, v_out)
    g0 = rt.R.project_bwd(out, ttr, tsh, top, vc0)
    vc, vz = rt.R.rasterize_bwd_depth(out, v_out, torch.zeros(h, w, device=rt.ctx.device))
    assert bool((vz == 0).all())
    _grad_close(vc.cpu().numpy(), vc0.cpu().numpy(), name="v_combined, v_depth = 0")   # f32 atomics: order may differ
    # with the same v_combined, the depth projection backward is the plain one, bit for bit
    g = rt.R.project_bwd(out, ttr, tsh, top, vc0, v_z=vz)
    for a, b in zip(g, g0):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_finite_difference_expected_depth_through_autograd(rt):
    """Central differences of a loss on the expected depth and the image (smooth cutoff) against the gradients that
    RenderDepthFunction + expected_depth return: abs 1e-4 + rel 2 %."""
    cam, tr, sh, op = finite_diff_base_scene()
    w = h = 32
    d = rt.ctx.device
    wd = torch.from_numpy(_v_depth(h, w, 0xDE0200) / (h * w)).to(d)
    wi = torch.from_numpy(random_v_output(h, w, 0xDE0201) / (h * w * 4)).to(d)

    def loss(tr_, op_, grad=False):
        ttr, tsh, top = (torch.from_numpy(x).to(d) for x in (tr_, sh, op_))
        if grad:
            ttr.requires_grad_(True); top.requires_grad_(True)
        holder = torch.zeros(tr_.shape[0], device=d, requires_grad=grad)
        img, depth, _, _ = rt.R.RenderDepthFunction.apply(ttr, tsh, top, holder, rt.ctx, cam, (w, h), False, (0.0, 0.0, 0.0), 2)
        ed = rt.R.expected_depth(img, depth)
        l = (ed.double() * wd * img[..., 3].double()).sum() + (img.double() * wi).sum()
        return l, ttr, top

    l, ttr, top = loss(tr, op, grad=True)
    l.backward()
    vt, vo = ttr.grad.cpu().numpy(), top.grad.cpu().numpy()
    eps = 3e-4
    cases = [("t", 0, 0), ("t", 0, 1), ("t", 0, 2), ("t", 1, 2), ("t", 0, 3), ("t", 1, 5), ("t", 0, 7), ("t", 1, 8),
             ("op", 0, 0), ("op", 2, 0)]
    fails = []
    for kind, s, c in cases:
        def pert(dv):
            t2, o2 = tr.copy(), op.copy()
            if kind == "t":
                t2[s, c] += dv
            else:
                o2[s] += dv
            return float(loss(t2, o2)[0].item())
        num = (pert(eps) - pert(-eps)) / (2 * eps)
        an = vt[s, c] if kind == "t" else vo[s]
        if abs(num - an) > 1e-4 + 0.02 * max(abs(num), abs(an), 1e-8):
            fails.append(f"{kind}[{s},{c}] numerical {num:.6f} analytical {an:.6f}")
    assert not fails, "\n".join(fails)


def test_depth_autograd_without_depth_gradient_is_the_plain_path(rt):
    cam, tr, sh, op = synthetic_scene(5_000, 128, 96, k=4, seed=0xDE0300)
    d = rt.ctx.device
    grads = []
    for fn in (rt.R.RenderFunction, rt.R.RenderDepthFunction):
        ttr, tsh, top = (torch.from_numpy(x).to(d).requires_grad_(True) for x in (tr, sh, op))
        holder = torch.zeros(tr.shape[0], device=d, requires_grad=True)
        outs = fn.apply(ttr, tsh, top, holder, rt.ctx, cam, (128, 96), False, (0.0, 0.0, 0.0), 1)
        outs[0].mean().backward()
        grads.append([g.grad.clone() for g in (ttr, tsh, top, holder)])
    for a, b in zip(*grads):
        _grad_close(a.cpu().numpy(), b.cpu().numpy())
    # expected depth of an opaque pixel lies between the nearest and farthest splat
    img, depth, _, _ = rt.R.RenderDepthFunction.apply(*(torch.from_numpy(x).to(d) for x in (tr, sh, op)), None, rt.ctx, cam,
                                                     (128, 96), False, (0.0, 0.0, 0.0), 1)
    ed = rt.R.expected_depth(img, depth)
    covered = img[..., 3] > 0.5
    assert covered.any() and bool((ed[covered] >= 1.99).all()) and bool((ed[covered] <= 12.01).all())


def test_depth_error_codes(rt):
    lib = rt.lib.load()
    n, w, h = 2_000, 64, 48
    cam, tr, sh, op = synthetic_scene(n, w, h, k=1, seed=0xDE0400)
    d = rt.ctx.device
    ttr, tsh, top = _dev(rt, tr, sh, op)
    with pytest.raises(rt.lib.BgError) as e:
        rt.R.render_splats(rt.ctx, cam, (w, h), ttr, tsh, top, rpass=0, render_depth=True)
    assert e.value.status == rt.lib.BG_ERR_INVALID
    depth_out = rt.R.render_splats(rt.ctx, cam, (w, h), ttr, tsh, top, render_depth=True)
    out = rt.R.render_splats(rt.ctx, cam, (w, h), ttr, tsh, top)   # plain forward: the context's last forward
    v_out, v_d = _dev(rt, random_v_output(h, w), _v_depth(h, w))
    bg = (C.c_float * 3)(*out.background)

    def backward(state, smooth=0):
        vc = torch.full((n, 10), 7.0, device=d)
        vz = torch.full((n,), 7.0, device=d)
        status = lib.bg_rasterize_backward_depth(rt.ctx.handle, rt.R._stream_ptr(d), C.byref(state), out.out_img.data_ptr(),
                                                 depth_out.depth.data_ptr(), v_out.data_ptr(), v_d.data_ptr(), bg, smooth,
                                                 vc.data_ptr(), n, vz.data_ptr())
        torch.cuda.synchronize(d)
        return status, bool((vc == 7.0).all()) and bool((vz == 7.0).all())

    assert backward(out.state) == (rt.lib.BG_ERR_INVALID, True)          # the last forward rendered no depth
    again = rt.R.render_splats(rt.ctx, cam, (w, h), ttr, tsh, top, render_depth=True)
    assert backward(again.state, smooth=1) == (rt.lib.BG_ERR_INVALID, True)   # smooth flag vs hard-cutoff pass
    assert backward(again.state) == (rt.lib.BG_OK, False)
    assert lib.bg_rasterize_backward_depth(rt.ctx.handle, None, C.byref(again.state), again.out_img.data_ptr(), None,
                                           v_out.data_ptr(), v_d.data_ptr(), bg, 0, v_out.data_ptr(), n,
                                           v_out.data_ptr()) == rt.lib.BG_ERR_NULL


def test_depth_forward_backward_under_cuda_graph(rt):
    cam, tr, sh, op = synthetic_scene(30_000, 320, 240, k=4, seed=0xDE0500)
    d = rt.ctx.device
    ttr, tsh, top = _dev(rt, tr, sh, op)
    v_out, v_d = _dev(rt, random_v_output(240, 320), _v_depth(240, 320))

    def step():
        out = rt.R.render_splats(rt.ctx, cam, (320, 240), ttr, tsh, top, render_depth=True)
        vc, vz = rt.R.rasterize_bwd_depth(out, v_out, v_d)
        return out, vz, rt.R.project_bwd(out, ttr, tsh, top, vc, v_z=vz)

    out_e, vz_e, g_e = step()
    img_e, depth_e, vz_e, vt_e = out_e.out_img.clone(), out_e.depth.clone(), vz_e.clone(), g_e[0].clone()
    side = torch.cuda.Stream(d)
    side.wait_stream(torch.cuda.current_stream(d))
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream(d).wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out_g, vz_g, g_g = step()
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out_g.out_img, img_e) and torch.equal(out_g.depth, depth_e)
    _grad_close(vz_g.cpu().numpy(), vz_e.cpu().numpy(), name="v_z graph vs eager")
    _grad_close(g_g[0].cpu().numpy(), vt_e.cpu().numpy(), name="v_transforms graph vs eager")
