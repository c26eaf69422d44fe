"""The forward blend's staging ring (blend_fwd.cu): one producer warp stages each batch of a tile's list once into a
ring of FWD_RING slots that the four pixel warps share, and keeps staging while any of them still blends.

The scenes stress the ring's hand-over: warps of one tile retiring many batches apart, every warp retiring in the
first batch, lists shorter than, equal to and one past a batch and the ring, empty tiles, right and bottom edge
tiles whose warps lie wholly outside the image, and a tile list of more than 10 000 entries.  Each render is checked
against the CPU oracle (projected rows, lists, trimmed ends, visible marks) and, for the near-opaque scenes, against
the float64 restatement of tests/blend_ref.py, including the walked and acted counts of the hand-off words through the
backward's counting variant.  The packed forward (PASS_FORWARD), DEPTH and the smooth cutoff run the same ring.
"""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from blend_ref import opaque_scene, reference_for  # noqa: E402
from scenes import random_v_output, synthetic_scene  # noqa: E402
from test_gpu_blend_opaque import _img_vs_ref  # noqa: E402
from test_gpu_parity import _check_forward_exact, _img_close  # noqa: E402

BG = (0.1, 0.2, 0.3)
RING_ROWS = 4 * 32   # FWD_RING slots of one 32-row batch


@pytest.fixture(scope="module")
def rt():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import brush_b200.render as R
    from brush_b200.camera import build_uniforms
    from oracle import oracle as orc

    class RT:
        pass

    r = RT()
    r.R, r.orc, r.build_uniforms = R, orc, build_uniforms
    r.ctx = R.RenderContext(max_splats=1 << 17, max_w=512, max_h=512, max_intersections=1 << 22)
    yield r
    r.ctx.close()


def _dev(rt, *arrs):
    return tuple(torch.from_numpy(np.ascontiguousarray(x)).to(rt.ctx.device) for x in arrs)


def _render(rt, cam, w, h, tr, sh, op, **kw):
    ttr, tsh, top = _dev(rt, tr, sh, op)
    return rt.R.render_splats(rt.ctx, cam, (w, h), ttr, tsh, top, background=BG, **kw)


def _packed_matches(rt, cam, w, h, tr, sh, op, img):
    """The packed forward blends the same rows in the same order: its bytes are the f32 image's, quantised."""
    out = _render(rt, cam, w, h, tr, sh, op, rpass=rt.R.PASS_FORWARD)
    packed = out.out_img.cpu().numpy().view(np.uint8).reshape(h, w, 4).astype(np.int32)
    want = np.clip(img * np.float32(255.0), 0.0, 255.0).astype(np.uint8).astype(np.int32)
    # (the two passes may round rgb + T bg with and without a fused multiply-add: a byte may truncate one lower)
    assert np.abs(packed - want).max() <= 1
    assert (packed == want).mean() > 0.999


# n, w, h: sizes whose right and bottom tiles keep only their left / top 8x8 blocks inside the image.  n_front None:
# warps of one tile retire many batches apart; 3000 large opaque front splats: every warp of many tiles retires in the
# first batch of a long list.
@pytest.mark.parametrize("n,w,h,depth,n_front", [(20_000, 200, 152, False, None), (16_000, 264, 120, True, None),
                                                 (20_000, 200, 152, False, 3000)])
def test_opaque_edges_and_retirement(rt, n, w, h, depth, n_front):
    kw = {} if n_front is None else {"n_front": n_front}
    cam, tr, sh, op = opaque_scene(0x57A6E0 + n + w, n, w, h, **kw)
    o = rt.orc.render_forward(rt.build_uniforms(cam, w, h), w, h, tr, sh, op, bg=BG)
    r = reference_for(o, BG, z=depth)
    if n_front is None:
        assert (r.walked.max(1) - r.walked.min(1)).max() >= 8
    else:
        assert ((r.walked.max(1) == 1) & (r.list_len > 4 * 32)).sum() >= 10
    assert w % 16 == 8 and h % 16 == 8
    ok = ~r.ambiguous
    out = _render(rt, cam, w, h, tr, sh, op, render_depth=depth)
    _check_forward_exact(rt, out, o)
    img = out.out_img.cpu().numpy()
    _img_vs_ref(img, r.img, np.repeat(ok[..., None], 4, -1))
    if depth:
        _img_vs_ref(out.depth.cpu().numpy(), r.depth, ok)
    else:
        st = rt.R.blend_stats(out, *_dev(rt, random_v_output(h, w)))
        assert abs(st["warp_splat_iterations"] - r.n_acted_blocks) <= r.flip_bound
        assert abs(st["pairs_live"] - r.n_blend) <= r.flip_bound
        _packed_matches(rt, cam, w, h, tr, sh, op, img)


@pytest.mark.parametrize("n,seed", [(1, 1), (31, 2), (32, 3), (33, 4), (RING_ROWS - 1, 5), (RING_ROWS + 1, 6),
                                    (RING_ROWS, 7)])
def test_short_lists(rt, n, seed):
    """Splats large enough to cover most of the 32x32 image: n bounds every tile's list length, around the batch and
    ring boundaries."""
    w, h = 32, 32
    cam, tr, sh, op = synthetic_scene(n, w, h, k=1, seed=0x5700 + seed, scale_shift=4.0)
    o = rt.orc.render_forward(rt.build_uniforms(cam, w, h), w, h, tr, sh, op, bg=BG)
    out = _render(rt, cam, w, h, tr, sh, op)
    _check_forward_exact(rt, out, o)
    _img_close(out.out_img.cpu().numpy(), o.out_img)
    _packed_matches(rt, cam, w, h, tr, sh, op, out.out_img.cpu().numpy())


def test_empty_tiles(rt):
    """A few small splats in a large image: most tiles have an empty list."""
    w, h = 256, 200
    cam, tr, sh, op = synthetic_scene(12, w, h, k=1, seed=0x57E0)
    o = rt.orc.render_forward(rt.build_uniforms(cam, w, h), w, h, tr, sh, op, bg=BG)
    lens = o.tile_offsets_untrimmed[..., 1] - o.tile_offsets_untrimmed[..., 0]
    assert (lens == 0).mean() > 0.5
    out = _render(rt, cam, w, h, tr, sh, op)
    _check_forward_exact(rt, out, o)
    _img_close(out.out_img.cpu().numpy(), o.out_img)


@pytest.mark.parametrize("smooth,depth", [(False, False), (True, False), (False, True)])
def test_long_list(rt, smooth, depth):
    """Translucent splats large enough to cover the 48x48 image: tile lists above 10 000 entries, walked to the end
    by warps that never saturate.  Also the smooth cutoff and DEPTH on the same lists."""
    w, h, n = 48, 48, 64_000
    cam, tr, sh, op = synthetic_scene(n, w, h, k=1, seed=0x57106, scale_shift=3.0)
    op = np.full_like(op, -5.0)   # opacity ~0.0067: far from saturating
    rpass = rt.R.PASS_BACKWARD_SMOOTH if smooth else rt.R.PASS_BACKWARD
    o = rt.orc.render_forward(rt.build_uniforms(cam, w, h), w, h, tr, sh, op, bg=BG, rpass=rpass)
    lens = o.tile_offsets_untrimmed[..., 1] - o.tile_offsets_untrimmed[..., 0]
    assert lens.max() >= 10_000
    out = _render(rt, cam, w, h, tr, sh, op, rpass=rpass, render_depth=depth)
    _check_forward_exact(rt, out, o)
    _img_close(out.out_img.cpu().numpy(), o.out_img)
    if depth:
        r = reference_for(o, BG, z=True)
        _img_vs_ref(out.depth.cpu().numpy(), r.depth, ~r.ambiguous)
