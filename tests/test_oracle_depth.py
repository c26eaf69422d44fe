"""The oracle's accumulated depth D = sum_i vis_i z_i (DESIGN.md section 4.6) and its joint colour + depth adjoint.

D is pinned against a float64 numpy restatement of the blend and against closed forms (one splat, an opaque front
splat, the convex-combination bound); the adjoint against central finite differences with the smooth alpha cutoff,
on the scenes, eps and tolerances of test_oracle_finite_diff.py."""
import os

import numpy as np
import pytest

from brush_b200.camera import Camera, build_uniforms
from oracle import oracle as orc
from oracle import oracle_depth as orcd
from scenes import finite_diff_base_scene, golden_case, splitmix64, synthetic_scene


def _np_blend(res):
    """float64 restatement of the hard-cutoff blend from the oracle's projected rows and sorted depths.
    Returns D, alpha, and per pixel the smallest / largest z among the blended splats (inf / -inf if none)."""
    h, w = res.h, res.w
    D = np.zeros((h, w)); A = np.zeros((h, w))
    zmin = np.full((h, w), np.inf); zmax = np.full((h, w), -np.inf)
    proj = res.projected.astype(np.float64)
    z_all = res.depths_sorted.astype(np.float64)
    ly, lx = np.mgrid[0:16, 0:16]
    for ty in range(res.tiles_y):
        for tx in range(res.tiles_x):
            lo, hi = (int(v) for v in res.tile_offsets[ty, tx])
            if hi <= lo:
                continue
            px, py = tx * 16 + lx.ravel(), ty * 16 + ly.ravel()
            ins = (px < w) & (py < h)
            px, py = px[ins], py[ins]
            ids = res.cgid_from_isect[lo:hi].astype(np.int64)
            p = proj[ids]
            dx = p[:, 0:1] - (px[None] + 0.5)
            dy = p[:, 1:2] - (py[None] + 0.5)
            sigma = 0.5 * (p[:, 2:3] * dx * dx + p[:, 4:5] * dy * dy) + p[:, 3:4] * dx * dy
            alpha = np.minimum(0.999, p[:, 5:6] * np.exp(-sigma))
            acts = (sigma >= 0) & (alpha >= 1.0 / 255.0)
            f = np.where(acts, 1.0 - alpha, 1.0)
            t_before = np.concatenate([np.ones((1, f.shape[1])), np.cumprod(f, 0)[:-1]], 0)
            stops = acts & (t_before * (1.0 - alpha) <= 1e-4)
            first_stop = np.where(stops.any(0), stops.argmax(0), len(ids))
            blended = acts & (np.arange(len(ids))[:, None] < first_stop[None])
            vis = np.where(blended, alpha * t_before, 0.0)
            z = z_all[ids][:, None]
            D[py, px] = (vis * z).sum(0)
            A[py, px] = 1.0 - np.prod(np.where(blended, 1.0 - alpha, 1.0), 0)
            zmin[py, px] = np.where(blended, z, np.inf).min(0)
            zmax[py, px] = np.where(blended, z, -np.inf).max(0)
    return D, A, zmin, zmax


def _render(cam, w, h, tr, sh, op, rpass=orc.PASS_BACKWARD, mip=False, bg=(0.0, 0.0, 0.0)):
    return orc.render_forward(build_uniforms(cam, w, h), w, h, tr, sh, op, mip=mip, bg=bg, rpass=rpass)


@pytest.mark.parametrize("name", ["tiny_case", "basic_case", "mix_case"])
def test_depth_matches_float64_restatement_on_golden_scenes(golden_dir, name):
    cam, tr, sh, op, _, (w, h) = golden_case(os.path.join(golden_dir, f"{name}.safetensors"))
    r = _render(cam, w, h, tr, sh, op)
    D = orcd.render_depth(r)
    D64, A64, _, _ = _np_blend(r)
    zmax = float(r.depths_sorted.max()) if r.num_visible else 1.0
    assert np.abs(A64 - r.out_img[..., 3]).max() < 1e-4   # the restatement blends what the oracle blends
    err = np.abs(D.astype(np.float64) - D64)
    bad = err > 1e-5 * zmax + 1e-4 * np.abs(D64)
    # an alpha within float rounding of a threshold may fall on the other side (a "threshold flip")
    assert bad.mean() <= 2e-3, f"{bad.sum()} pixels outside tolerance, max err {err.max():.3e}"
    if bad.any():
        assert err[bad].max() <= 1.5 / 255 * 1.5 * zmax
    assert (D > 0).any() and np.isfinite(D).all()


def _one_splat(z, log_scale=-1.0, raw_opac=2.0, x=0.0, y=0.0):
    tr = np.array([[x, y, z, 1.0, 0.0, 0.0, 0.0, log_scale, log_scale, log_scale]], np.float32)
    return tr, np.full((1, 1, 3), 0.5, np.float32), np.array([raw_opac], np.float32)


def test_single_splat_depth_is_alpha_times_z():
    w = h = 32
    cam = Camera(position=(0.0, 0.0, 0.0), rotation=(0.0, 0.0, 0.0, 1.0), fov_x=0.8, fov_y=0.8)
    tr, sh, op = _one_splat(3.0, log_scale=-1.5)
    r = _render(cam, w, h, tr, sh, op)
    D = orcd.render_depth(r)
    a = r.out_img[..., 3]
    z = np.float32(r.depths_sorted[0])
    assert (a > 0).any() and (a == 0).any()
    # D = fl(z * alpha_i); the image's alpha is 1 - fl(1 - alpha_i), which is alpha_i exactly when alpha_i >= 1/2
    hi = a >= 0.5
    assert hi.any()
    np.testing.assert_array_equal(D[hi], (z * a)[hi])
    np.testing.assert_allclose(D, z * a, rtol=0, atol=float(z) * 2.0 ** -24)
    assert (D[a == 0] == 0).all()


def test_opaque_front_splat_gives_its_depth():
    """A front splat near the alpha cap (0.999) leaves T ~ 1e-3; an opaque splat behind it then stops the pixel and is
    not blended, so the expected depth D / alpha is the front splat's z at every pixel."""
    w = h = 32
    cam = Camera(position=(0.0, 0.0, 0.0), rotation=(0.0, 0.0, 0.0, 1.0), fov_x=0.8, fov_y=0.8)
    t1, s1, o1 = _one_splat(2.0, log_scale=3.0, raw_opac=12.0)
    t2, s2, o2 = _one_splat(5.0, log_scale=3.0, raw_opac=12.0)
    r = _render(cam, w, h, np.concatenate([t2, t1]), np.concatenate([s2, s1]), np.concatenate([o2, o1]))
    assert r.num_visible == 2
    D = orcd.render_depth(r)
    a = r.out_img[..., 3]
    assert a.min() > 0.99
    np.testing.assert_allclose(D.astype(np.float64) / a, 2.0, rtol=1e-6)


def test_depth_is_a_convex_combination_of_blended_depths():
    w, h = 96, 64
    cam, tr, sh, op = synthetic_scene(4000, w, h, k=1, seed=0xDE9001)
    r = _render(cam, w, h, tr, sh, op)
    D = orcd.render_depth(r).astype(np.float64)
    _, A64, zmin, zmax = _np_blend(r)
    a = r.out_img[..., 3].astype(np.float64)
    same = (np.abs(A64 - a) < 1e-6) & np.isfinite(zmin)   # pixels where the restatement blends the same splats
    assert same.mean() > 0.5
    slack = 1e-5 * zmax[same]
    assert (a[same] * zmin[same] - slack <= D[same]).all()
    assert (D[same] <= a[same] * zmax[same] + slack).all()
    assert (D[~np.isfinite(zmin) & (a == 0)] == 0).all()


def _loss_and_render(cam, w, h, tr, sh, op, wd, wi):
    r = _render(cam, w, h, tr, sh, op, rpass=orc.PASS_BACKWARD_SMOOTH)
    D = orcd.render_depth(r)
    loss = float((D.astype(np.float64) * wd).sum())
    if wi is not None:
        loss += float((r.out_img.astype(np.float64) * wi).sum())
    return loss, r, D


def _fd_check(cam, w, h, tr, sh, op, wd, wi, cases, eps=3e-4, rel=0.01, abs_tol=5e-5):
    _, r, D = _loss_and_render(cam, w, h, tr, sh, op, wd, wi)
    v_out = wi if wi is not None else np.zeros((h, w, 4), np.float32)
    vc, vz = orcd.rasterize_backward_depth(r, v_out, wd, out_depth=D)
    vt, _, vo, _ = orcd.project_backward_depth(r, vc, vz)
    fails = []
    for kind, s, c in cases:
        def pert(dv):
            t2, o2 = tr.copy(), op.copy()
            if kind == "t":
                t2[s, c] += dv
            else:
                o2[s] += dv
            return _loss_and_render(cam, w, h, t2, sh, o2, wd, wi)[0]
        num = (pert(eps) - pert(-eps)) / (2 * eps)
        an = vt[s, c] if kind == "t" else vo[s]
        tol = abs_tol + rel * max(abs(num), abs(an), 1e-8)
        if abs(num - an) > tol:
            fails.append(f"{kind}[{s},{c}] num {num:.6f} an {an:.6f}")
    assert not fails, "\n".join(fails)


# means, quaternion, log-scales, opacity
CASES = [("t", 0, 0), ("t", 0, 1), ("t", 0, 2), ("t", 1, 2), ("t", 2, 0), ("t", 0, 3), ("t", 1, 5), ("t", 2, 6),
         ("t", 0, 7), ("t", 1, 8), ("t", 3, 9), ("op", 0, 0), ("op", 2, 0)]


def _depth_weights(w, h, seed=0xDE17):
    return (splitmix64(seed, h * w).reshape(h, w) / (h * w)).astype(np.float32)


def test_finite_difference_weighted_depth_loss():
    cam, tr, sh, op = finite_diff_base_scene()
    _fd_check(cam, 32, 32, tr, sh, op, _depth_weights(32, 32), None, CASES)


def test_finite_difference_image_plus_depth_loss():
    cam, tr, sh, op = finite_diff_base_scene()
    wi = splitmix64(0x51ED, 48 * 40 * 4).reshape(40, 48, 4).astype(np.float32) / (48 * 40)
    _fd_check(cam, 48, 40, tr, sh, op, _depth_weights(48, 40), wi, CASES, rel=0.02, abs_tol=1e-4)


def test_finite_difference_depth_offcentre_rotated_camera():
    _, tr, sh, op = finite_diff_base_scene()
    cam = Camera(position=(0.4, -0.2, -3.2), rotation=(0.05, -0.08, 0.03, 0.995), fov_x=0.7, fov_y=0.5, center_uv=(0.45, 0.55))
    wi = np.full((36, 48, 4), 1.0 / (36 * 48 * 4), np.float32)
    _fd_check(cam, 48, 36, tr, sh, op, _depth_weights(48, 36), wi, CASES, rel=0.02, abs_tol=1e-4)


def test_zero_depth_gradient_is_the_colour_adjoint():
    cam, tr, sh, op = synthetic_scene(3000, 96, 64, k=1, seed=0xDE9002)
    r = _render(cam, 96, 64, tr, sh, op, bg=(0.1, 0.2, 0.3))
    v_out = splitmix64(0xDE9003, 64 * 96 * 4).reshape(64, 96, 4).astype(np.float32)
    vc, vz = orcd.rasterize_backward_depth(r, v_out, np.zeros((64, 96), np.float32))
    np.testing.assert_array_equal(vc, orc.rasterize_backward(r, v_out))
    assert (vz == 0).all()
