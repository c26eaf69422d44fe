"""Float64 restatement of the L1 + SSIM image loss (brush_b200/csrc/loss.cu, oracle/orc_loss_optim.c), written from the
formulas rather than from either implementation: torch float64, the separable 11-tap Gaussian window (sigma = 1.5, exact
float64 taps) as two conv2d passes, and autograd for the gradient.

The conventions are the kernels':
- the GT is decoded as f32(k) * f32(1 / 255), rounded to f32 (not k / 255: the two differ in the last bit for about half
  of the byte values, which flips the L1 sign wherever pred equals the decoded GT);
- compositing is gt_c + (1 - gt_a) * bg in float64 from the f32-decoded values; outside the image pred reads 0 and the
  GT reads 0, i.e. bg when compositing (the window of a border pixel sees the background);
- sign(0) = 0 for the L1 term; the SSIM value is clamped to [-1, 1] and its gradient is zero only strictly outside
  that range; max(0, sigma^2) clamps the value but never zeroes the variance derivative;
- with the mask, both the map and the chain are multiplied by the GT alpha;
- channel 3 (when present) is |pred.a - gt.a|, alpha-weighted under the mask, with no window.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

C1 = 1e-4
C2 = 9e-4
INV_255_F32 = np.float32(1.0) / np.float32(255.0)


def taps() -> torch.Tensor:
    x = torch.arange(11, dtype=torch.float64) - 5.0
    w = torch.exp(-x * x / (2.0 * 1.5 * 1.5))
    return w / w.sum()


def pack_rgba(rgba8: np.ndarray) -> np.ndarray:
    """[h,w,4] integer bytes -> [h,w] uint32 packed little-endian rgba8 (the kernels' GT layout)."""
    b = rgba8.astype(np.uint32)
    return (b[..., 0] | (b[..., 1] << 8) | (b[..., 2] << 16) | (b[..., 3] << 24)).astype(np.uint32)


def decode_gt(packed: np.ndarray):
    """packed [h,w] uint32 -> (rgb [3,h,w], alpha [h,w]) as float32, decoded exactly as the kernels do."""
    p = packed.astype(np.uint32)
    rgb = np.stack([((p >> (8 * c)) & 0xFF).astype(np.float32) * INV_255_F32 for c in range(3)])
    alpha = ((p >> 24) & 0xFF).astype(np.float32) * INV_255_F32
    return rgb, alpha


def gt_effective(packed: np.ndarray, bg=None) -> np.ndarray:
    """The GT each colour channel is compared with, [3,h,w] float64 (composited over bg when bg is given)."""
    rgb, alpha = decode_gt(packed)
    g = rgb.astype(np.float64)
    if bg is not None:
        b = np.asarray(bg, np.float32).astype(np.float64)
        g = g + (1.0 - alpha.astype(np.float64))[None] * b[:, None, None]
    return g


def _blur_valid(t: torch.Tensor) -> torch.Tensor:
    """[k,h+10,w+10] -> [k,h,w]: the separable window over an already padded stack."""
    k = t.shape[0]
    w = taps().to(t.device)
    t = F.conv2d(t[None], w.view(1, 1, 1, 11).expand(k, 1, 1, 11), groups=k)
    return F.conv2d(t, w.view(1, 1, 11, 1).expand(k, 1, 11, 1), groups=k)[0]


def _pass_clamp_min0(v: torch.Tensor) -> torch.Tensor:
    return v + (v.clamp_min(0.0) - v).detach()


def _ssim_clamp(s: torch.Tensor) -> torch.Tensor:
    inside = (s >= -1.0) & (s <= 1.0)
    return torch.where(inside, s, s.detach().clamp(-1.0, 1.0))


def loss_map(pred: torch.Tensor, packed: np.ndarray, l1_w: float, ssim_w: float, bg=None, mask: bool = False) -> torch.Tensor:
    """pred [C,h,w] float64 (C = 3 or 4, may require grad) -> the loss map [C,h,w] float64."""
    dev = pred.device
    nch = pred.shape[0]
    _, alpha = decode_gt(packed)
    ga = torch.from_numpy(alpha.astype(np.float64)).to(dev)
    y = torch.from_numpy(gt_effective(packed, bg)).to(dev)
    x = pred[:3]
    pad_bg = [0.0] * 3 if bg is None else [float(v) for v in np.asarray(bg, np.float32)]
    xp = F.pad(x, (5, 5, 5, 5))
    yp = torch.stack([F.pad(y[c], (5, 5, 5, 5), value=pad_bg[c]) for c in range(3)])
    m = _blur_valid(torch.cat([xp, xp * xp, yp, yp * yp, xp * yp]))
    mu1, ex2, mu2, ey2, exy = m[0:3], m[3:6], m[6:9], m[9:12], m[12:15]
    s1 = _pass_clamp_min0(ex2 - mu1 * mu1)
    s2 = _pass_clamp_min0(ey2 - mu2 * mu2)
    s12 = exy - mu1 * mu2
    ssim = ((2.0 * mu1 * mu2 + C1) * (2.0 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s1 + s2 + C2))
    out = [float(np.float32(l1_w)) * (x - y).abs() + float(np.float32(ssim_w)) * _ssim_clamp(ssim)]
    if nch == 4:
        out.append((pred[3] - ga).abs()[None])
    out = torch.cat(out)
    if mask:
        out = out * ga[None]
    return out


def loss_and_grad(pred_chw: np.ndarray, packed: np.ndarray, dl_dmap, l1_w: float, ssim_w: float, bg=None, mask: bool = False,
                  device="cpu"):
    """pred_chw [C,h,w] float32 -> (map [C,h,w], dL/dpred [C,h,w]) as float64 numpy, for L = sum(dl_dmap * map).
    dl_dmap: [C,h,w] array, or one constant per channel."""
    p = torch.tensor(np.asarray(pred_chw, np.float32).astype(np.float64), device=device, requires_grad=True)
    m = loss_map(p, packed, l1_w, ssim_w, bg, mask)
    dl = np.asarray(dl_dmap, np.float32).astype(np.float64)
    if dl.ndim == 1:
        dl = dl[:, None, None]
    (m * torch.from_numpy(dl).to(device)).sum().backward()
    return m.detach().cpu().numpy(), p.grad.cpu().numpy()


def weighted_sum(lmap: np.ndarray, chain) -> float:
    """sum_c chain[c] * sum(map[c]) in float64 (the loss scalar of the fused kernel and of the train step)."""
    return float(sum(float(np.float32(chain[c])) * float(lmap[c].astype(np.float64).sum()) for c in range(lmap.shape[0])))
