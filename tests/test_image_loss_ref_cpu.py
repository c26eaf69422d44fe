"""The float64 image-loss restatement (tests/image_loss_ref.py) checked on the CPU, before it judges the GPU kernels:
against the C oracle over the shapes and value regimes of tests/test_gpu_image_loss.py, and its gradient against
central differences of its own map at corner, edge and interior pixels.

The oracle runs the loss in f32 with the kernels' decode and accumulation order, so the two agree to f32 rounding.
Measured here, in units of |l1_w| + |ssim_w| on the map and of the gradient scale (max |grad|, but at least
max(dl) * (|l1_w| + |ssim_w|), which keeps the tie cases -- gradient ~0 -- on an absolute footing): at most 2.3e-6 and
1.3e-6 up to 300 x 500, outside the near-tie pixels where the L1 sign itself is a rounding decision.  The constant-block
regime is the exception, at 4.3e-4 and 4.1e-4: inside a constant block sigma^2 = E[x^2] - mu^2 cancels to f32 noise of
about 1e-7, which is 1e-4 of C2 = 9e-4 and moves the SSIM ratio by that much.  The bounds below are 4x the measured
errors."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

from image_loss_ref import decode_gt, gt_effective, loss_and_grad, loss_map, pack_rgba, taps  # noqa: E402
from oracle import oracle as orc  # noqa: E402

REGIMES = ("uniform", "wide", "ties", "const", "alpha0")


def make_case(h, w, channels, regime, seed, bg=None, mask=False):
    """(pred [C',h,w] f32 with C' = 4, packed GT [h,w] u32) for one value regime.  Shared with the GPU tests.
    uniform: pred in [0, 1]; wide: pred in [-0.5, 3]; ties: pred equals the decoded GT (alpha 255 there, so the
    composite is exact) on the left half; const: pred and GT constant on 16 x 16 blocks; alpha0: GT alpha 0 on
    24 x 24 blocks of a 48 x 48 checkerboard."""
    rng = np.random.default_rng(seed)
    alpha = channels == 4 or mask or bg is not None
    gt8 = rng.integers(0, 256, (h, w, 4), dtype=np.uint32)
    if not alpha:
        gt8[..., 3] = 255
    pred = rng.uniform(0.0, 1.0, (4, h, w)).astype(np.float32)
    if regime == "wide":
        pred = rng.uniform(-0.5, 3.0, (4, h, w)).astype(np.float32)
    elif regime == "const":
        by, bx = (np.arange(h) // 16)[:, None], (np.arange(w) // 16)[None, :]
        blk = by * 1000 + bx
        _, inv = np.unique(blk, return_inverse=True)
        inv = inv.reshape(h, w)
        nb = inv.max() + 1
        pred = rng.uniform(0.0, 1.0, (4, nb)).astype(np.float32)[:, inv]
        gt8 = rng.integers(0, 256, (nb, 4), dtype=np.uint32)[inv]
        if not alpha:
            gt8[..., 3] = 255
    elif regime == "alpha0":
        zero = ((np.arange(h)[:, None] // 24 + np.arange(w)[None, :] // 24) % 2) == 0
        gt8[..., 3] = np.where(zero, 0, gt8[..., 3])
    packed = pack_rgba(gt8)
    if regime == "ties":
        half = np.zeros((h, w), bool)
        half[:, : max(1, w // 2)] = True
        gt8[..., 3] = np.where(half, 255, gt8[..., 3])
        packed = pack_rgba(gt8)
        rgb, a = decode_gt(packed)
        pred[:3] = np.where(half[None], rgb, pred[:3])
        pred[3] = np.where(half, a, pred[3])
    return pred, packed


def near_ties(pred_chw, packed, bg):
    """Colour pixels whose L1 sign is a rounding decision: |pred - gt_eff| within a few f32 ulps but not exactly 0."""
    d = np.abs(pred_chw[:3].astype(np.float64) - gt_effective(packed, bg))
    scale = np.maximum(np.abs(pred_chw[:3]).astype(np.float64), 1.0)
    return (d > 0) & (d <= 4.0 * np.finfo(np.float32).eps * scale)


SHAPES = [(1, 1), (1, 17), (17, 1), (5, 11), (11, 5), (16, 33), (33, 16), (42, 43), (53, 52), (73, 74), (74, 73),
          (106, 107), (300, 500)]


@pytest.mark.parametrize("h,w", SHAPES)
@pytest.mark.parametrize("regime", REGIMES)
def test_reference_matches_oracle(h, w, regime):
    i = SHAPES.index((h, w)) + REGIMES.index(regime)
    channels = (3, 4)[i % 2]
    bg = (0.2, 0.4, 0.6) if i % 3 == 1 else None
    mask = i % 3 == 2 or regime == "alpha0"
    l1_w, ssim_w = ((0.8, -0.2), (1.0, 0.0), (0.0, 1.0))[i % 3]
    pred, packed = make_case(h, w, channels, regime, 1000 + i, bg, mask)
    pred_c = np.ascontiguousarray(pred[:channels])
    dl = np.random.default_rng(i).uniform(0.1, 1.0, (channels, h, w)).astype(np.float32)
    ref_map, ref_g = loss_and_grad(pred_c, packed, dl, l1_w, ssim_w, bg, mask)
    om = orc.image_loss_forward(pred_c, packed, l1_w, ssim_w, bg=bg, mask=mask)
    og = orc.image_loss_backward(pred_c, packed, dl, l1_w, ssim_w, bg=bg, mask=mask)
    map_tol, grad_tol = (2e-3, 2e-3) if regime == "const" else (1e-5, 5e-6)
    assert np.abs(om - ref_map).max() <= map_tol * (abs(l1_w) + abs(ssim_w))
    ok = np.ones_like(ref_g, bool)
    ok[:3] &= ~near_ties(pred_c, packed, bg)
    assert np.abs(og - ref_g)[ok].max() <= grad_tol * grad_scale(ref_g, dl, l1_w, ssim_w)


def grad_scale(ref_g, dl, l1_w, ssim_w):
    """max |grad|, but at least the L1 term's own size max(dl) * (|l1_w| + |ssim_w|)."""
    return max(float(np.abs(ref_g).max()), float(np.max(dl)) * (abs(l1_w) + abs(ssim_w)))


def test_reference_gradient_matches_central_differences():
    h, w = 23, 29
    bg = (0.1, 0.5, 0.9)
    pred, packed = make_case(h, w, 4, "wide", 7, bg, True)
    pred64 = pred.astype(np.float64)
    dl = np.random.default_rng(3).uniform(0.2, 1.0, (4, h, w))
    p = torch.tensor(pred64, requires_grad=True)
    (loss_map(p, packed, 0.8, -0.2, bg, True) * torch.from_numpy(dl)).sum().backward()
    g = p.grad.numpy()
    eps = 1e-6
    for (c, y, x) in [(0, 0, 0), (1, 0, w - 1), (2, h - 1, 0), (0, h - 1, w - 1), (1, 0, 14), (2, 11, 0), (0, 12, 13),
                      (1, 7, 20), (3, 5, 5)]:
        vals = []
        for s in (1.0, -1.0):
            q = pred64.copy()
            q[c, y, x] += s * eps
            vals.append(float((loss_map(torch.from_numpy(q), packed, 0.8, -0.2, bg, True).numpy() * dl).sum()))
        num = (vals[0] - vals[1]) / (2.0 * eps)
        assert abs(num - g[c, y, x]) <= 1e-5 * max(1.0, abs(num)), (c, y, x, num, g[c, y, x])


def test_taps_and_decode_conventions():
    w = taps()
    assert abs(float(w.sum()) - 1.0) < 1e-15 and torch.equal(w, w.flip(0))
    k = np.arange(256, dtype=np.uint32)
    rgb, a = decode_gt(k | (k << 8) | (k << 16) | (k << 24))
    assert rgb.dtype == np.float32 and np.array_equal(rgb[0], k.astype(np.float32) * np.float32(1.0 / 255.0))
    assert a[255] == np.float32(1.0) and a[0] == 0.0
    # the kernels' decode is not k / 255 for every byte
    assert (k.astype(np.float32) * np.float32(1.0 / 255.0) != k.astype(np.float32) / np.float32(255.0)).any()
