"""The blend backward's two-splat rounds (blend_bwd.cu): the loop evaluates splats j and j+1 of a batch in list order,
reduce-scatters their sums together and flushes both with one RED per owning lane; an odd batch ends on a null row.

Hand-built scenes put every splat over every pixel of a 40x36 image (edge tiles on the right and bottom), so each
warp's batches hold exactly min(n - 32 b, 32) live rows: 1, 2, 31, 32, 33 and 64 splats cover the odd tail, full
pairs and a second batch.  The SH DC alternates so that a colour channel is clamped in one splat of each pair and
not in the other.  Opaque variants make pixels stop on the first splat of a pair (alpha 0.97: T reaches 1e-4 on the
third splat) or on the second (alpha 0.99: on the second).  Every case runs with DEPTH as well, the translucent
ones with the smooth cutoff.
Gradients are checked against the float64 restatement of tests/blend_ref.py and against the CPU oracle, and the
counting variant's walk counts against the restatement's.

A non-finite upstream gradient over odd batches must leave the flush on real ids (the null row carries the last
row's id): the call completes without a CUDA error and the context renders correctly afterwards.  And the walk of
bench.py's scenes is pinned: the counting variant's counts on configs [1] and [3] are the ones the one-splat-per-round
kernel produced before the two-splat rounds (the walk itself did not change).
"""
import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from blend_ref import reference_for  # noqa: E402
from scenes import random_v_output, splitmix64  # noqa: E402
from test_gpu_blend_opaque import COLS  # noqa: E402
from test_gpu_parity import _check_forward_exact, _grad_close  # noqa: E402

BG = (0.1, 0.2, 0.3)
W, H = 40, 36


@pytest.fixture(scope="module")
def rt():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import brush_b200.render as R
    from brush_b200.camera import Camera, build_uniforms
    from oracle import oracle as orc
    from oracle import oracle_depth as orcd

    class RT:
        pass

    r = RT()
    r.R, r.orc, r.orcd, r.build_uniforms, r.Camera = R, orc, orcd, build_uniforms, Camera
    r.ctx = R.RenderContext(max_splats=1 << 12, max_w=64, max_h=64, max_intersections=1 << 16)
    yield r
    r.ctx.close()


def _scene(rt, n, alpha):
    """n large splats straight ahead at depths 2..3 (list order = index order), each covering the whole image."""
    fov_x = math.radians(60.0)
    focal = 0.5 * W / math.tan(fov_x / 2)
    fov_y = 2.0 * math.atan(0.5 * H / focal)
    cam = rt.Camera(position=(0.0, 0.0, 0.0), rotation=(0.0, 0.0, 0.0, 1.0), fov_x=fov_x, fov_y=fov_y)
    r = splitmix64(0xB1D0 + n + int(alpha * 1000), n * 4).reshape(n, 4)
    z = 2.0 + np.arange(n) / max(n, 1)
    means = np.stack([(r[:, 0] - 0.5) * 0.1 * z, (r[:, 1] - 0.5) * 0.1 * z, z], 1)
    quats = np.tile([0.0, 0.0, 0.0, 1.0], (n, 1))
    log_scales = np.log(np.full((n, 3), 3.0))
    tr = np.concatenate([means, quats, log_scales], 1).astype(np.float32)
    sh = np.empty((n, 1, 3), np.float32)
    even = np.arange(n) % 2 == 0
    sh[:, 0, 0] = np.where(even, -2.2, 0.8)   # red clamped (c < 0) in the first splat of each pair only
    sh[:, 0, 1] = np.where(even, 0.6, -2.2)   # green in the second only
    sh[:, 0, 2] = 0.3 + r[:, 2]
    op = np.full(n, math.log(alpha / (1.0 - alpha)), np.float32)
    return cam, tr, sh, op


def _dev(rt, *arrs):
    return tuple(torch.from_numpy(np.ascontiguousarray(x)).to(rt.ctx.device) for x in arrs)


@pytest.mark.parametrize("n,alpha", [(1, 0.05), (2, 0.05), (31, 0.05), (32, 0.05), (33, 0.05), (64, 0.05),
                                     (7, 0.97), (7, 0.99), (33, 0.97), (33, 0.99)])
@pytest.mark.parametrize("depth", [False, True])
def test_pairs_vs_reference(rt, n, alpha, depth):
    cam, tr, sh, op = _scene(rt, n, alpha)
    o = rt.orc.render_forward(rt.build_uniforms(cam, W, H), W, H, tr, sh, op, bg=BG)
    assert o.num_visible == n
    v_out = random_v_output(H, W)
    v_d = splitmix64(0xDE0002, H * W).reshape(H, W).astype(np.float32) if depth else None
    r = reference_for(o, BG, z=depth, v_output=v_out, v_depth=v_d)
    if alpha > 0.5:
        assert r.n_stop >= 0.5 * W * H, r.n_stop    # most pixels stop, on the splat the opacity picks
    else:
        assert r.n_stop == 0 and r.n_blend == n * W * H

    ttr, tsh, top = _dev(rt, tr, sh, op)
    out = rt.R.render_splats(rt.ctx, cam, (W, H), ttr, tsh, top, background=BG, render_depth=depth)
    _check_forward_exact(rt, out, o)
    if not depth:
        st = rt.R.blend_stats(out, *_dev(rt, v_out))
        fb = r.flip_bound
        assert abs(st["pairs_live"] - r.n_blend) <= fb, (st, r.n_blend)
        assert abs(st["pairs_stopping"] - r.n_stop) <= fb, (st, r.n_stop)
        assert abs(st["warp_splat_iterations"] - r.n_acted_blocks) <= fb, (st, r.n_acted_blocks)
        if alpha < 0.5:   # every row is live for each of the 5 x 5 warps whose 8x8 block reaches into the image
            assert st["warp_splat_iterations"] == 25 * n, st

    if depth:
        vc, vz = rt.R.rasterize_bwd_depth(out, *_dev(rt, v_out, v_d))
        ovc, ovz = rt.orcd.rasterize_backward_depth(o, v_out, v_d)
    else:
        vc, vz = rt.R.rasterize_bwd(out, *_dev(rt, v_out)), None
        ovc, ovz = rt.orc.rasterize_backward(o, v_out), None
    vc_np = vc.cpu().numpy()[:n]
    assert np.isfinite(vc_np).all()
    keep = np.ones(n, bool)
    keep[r.ambiguous_splats] = False
    # (the symmetric footprints cancel most of each conic and position sum, so the float32 sums are held to the
    # element-wise tolerance of test_gpu_parity.py rather than to a multiple of the oracle's own error)
    for col, nm in enumerate(COLS):
        _grad_close(vc_np[keep, col], r.v_combined[keep, col], name=nm + " vs float64")
        _grad_close(vc_np[:, col], ovc[:, col], name=nm)
    if depth:
        vz_np = vz.cpu().numpy()[:n]
        _grad_close(vz_np[keep], r.v_z[keep], name="v_z vs float64")
        _grad_close(vz_np, ovz, name="v_z")
    # the clamped channel's gradient is exactly zero in the splat where it is clamped
    assert (vc_np[0::2, 5] == 0).all() and (vc_np[1::2, 6] == 0).all()


@pytest.mark.parametrize("n", [1, 2, 31, 33])
def test_pairs_smooth_cutoff(rt, n):
    cam, tr, sh, op = _scene(rt, n, 0.05)
    o = rt.orc.render_forward(rt.build_uniforms(cam, W, H), W, H, tr, sh, op, bg=BG, rpass=rt.R.PASS_BACKWARD_SMOOTH)
    ttr, tsh, top = _dev(rt, tr, sh, op)
    out = rt.R.render_splats(rt.ctx, cam, (W, H), ttr, tsh, top, background=BG, rpass=rt.R.PASS_BACKWARD_SMOOTH)
    _check_forward_exact(rt, out, o)
    v_out = random_v_output(H, W)
    vc = rt.R.rasterize_bwd(out, *_dev(rt, v_out), smooth_cutoff=True).cpu().numpy()[:n]
    ovc = rt.orc.rasterize_backward(o, v_out)
    for col, nm in enumerate(COLS):
        _grad_close(vc[:, col], ovc[:, col], name=nm)


@pytest.mark.parametrize("depth", [False, True])
def test_nan_upstream_gradient_over_odd_batches(rt, depth):
    """33 and 7 splats: odd batches of 1 and 7 rows.  A NaN in v_output (and in v_depth) under one pixel of every warp
    of the first tile makes every sum of those warps NaN, the null rows' included."""
    for n in (33, 7):
        cam, tr, sh, op = _scene(rt, n, 0.05)
        ttr, tsh, top = _dev(rt, tr, sh, op)
        out = rt.R.render_splats(rt.ctx, cam, (W, H), ttr, tsh, top, background=BG, render_depth=depth)
        v_out = random_v_output(H, W)
        v_d = splitmix64(0xDE0003, H * W).reshape(H, W).astype(np.float32)
        for y, x in ((0, 0), (0, 8), (8, 0), (8, 8)):
            v_out[y, x, 0] = np.nan
            v_d[y, x] = np.nan
        if depth:
            vc, vz = rt.R.rasterize_bwd_depth(out, *_dev(rt, v_out, v_d))
        else:
            vc = rt.R.rasterize_bwd(out, *_dev(rt, v_out))
        torch.cuda.synchronize()
        assert vc.shape[0] >= n and np.isnan(vc.cpu().numpy()[:n]).any()
    # the same context, clean inputs: still the oracle's gradients
    cam, tr, sh, op = _scene(rt, 33, 0.05)
    o = rt.orc.render_forward(rt.build_uniforms(cam, W, H), W, H, tr, sh, op, bg=BG)
    ttr, tsh, top = _dev(rt, tr, sh, op)
    out = rt.R.render_splats(rt.ctx, cam, (W, H), ttr, tsh, top, background=BG)
    _check_forward_exact(rt, out, o)
    v_out = random_v_output(H, W)
    vc = rt.R.rasterize_bwd(out, *_dev(rt, v_out)).cpu().numpy()[:33]
    ovc = rt.orc.rasterize_backward(o, v_out)
    for col, nm in enumerate(COLS):
        _grad_close(vc[:, col], ovc[:, col], name=nm)


# bench.py CONFIGS[1] and [3]: (n, w, h, seed, scale shift, K) -> counting variant's (warp-splat iterations, live pairs,
# stopping pairs); None where not pinned
WALKS = [((1_000_000, 1920, 1080, 0xB2000001, 0.0, 16), (2_461_709, 108_409_235, 2_073_600)),
         ((1_000_000, 1920, 1080, 0xB2000001, 0.0, 1), (2_476_313, 109_131_128, 2_073_600)),
         ((4_000_000, 3840, 2160, 0xB2000003, -math.log(2.0), 16), (9_926_192, 437_502_423, None))]


@pytest.mark.parametrize("scene,counts", WALKS)
def test_bench_scene_walk_counts(scene, counts):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import brush_b200.render as R
    from scenes import synthetic_scene

    n, w, h, seed, shift, k = scene
    cam, tr, sh, op = synthetic_scene(n, w, h, k=k, seed=seed, scale_shift=shift)
    ctx = R.RenderContext(n, w, h, 0)
    try:
        ttr, tsh, top = (torch.from_numpy(x).to(ctx.device) for x in (tr, sh, op))
        out = R.render_splats(ctx, cam, (w, h), ttr, tsh, top)
        st = R.blend_stats(out, torch.from_numpy(random_v_output(h, w)).to(ctx.device))
    finally:
        ctx.close()
    got = (st["warp_splat_iterations"], st["pairs_live"], st["pairs_stopping"])
    assert all(want is None or g == want for g, want in zip(got, counts)), (got, counts)
