"""Float64 restatements of the bilateral grid of DESIGN.md section 4.11: slice, slice backward and the TV regulariser.

  torch_*  through torch.nn.functional.grid_sample (bilinear, border, align_corners) and autograd
  np_*     explicit trilinear interpolation and its adjoint written out in numpy

grid: [L, H, W, 12] (row-major 3x4 affine per cell); img, v_out: [h, w, 4].
"""
import numpy as np

L, H, W = 8, 16, 16
LUMA = np.array([0.299, 0.587, 0.114])


def identity(views=1):
    g = np.zeros((views, L, H, W, 12))
    g[..., 0] = g[..., 5] = g[..., 10] = 1.0
    return g


def lattice(h, w, img):
    """(gx, gy, gz, gray) per pixel, float64."""
    px = np.arange(w, dtype=np.float64)[None, :]
    py = np.arange(h, dtype=np.float64)[:, None]
    gx = np.broadcast_to((px + 0.5) / w * (W - 1), (h, w))
    gy = np.broadcast_to((py + 0.5) / h * (H - 1), (h, w))
    gray = img[..., 0:3] @ LUMA
    gz = np.clip(gray, 0.0, 1.0) * (L - 1)
    return gx, gy, gz, gray


def _cells(g, n):
    i0 = np.minimum(np.floor(g).astype(np.int64), n - 2)
    return i0, g - i0


def np_coeffs(grid, img):
    """A [h, w, 12], and dA/dgz [h, w, 12]."""
    h, w = img.shape[:2]
    gx, gy, gz, _ = lattice(h, w, img)
    x0, fx = _cells(gx, W)
    y0, fy = _cells(gy, H)
    z0, fz = _cells(gz, L)
    a = np.zeros((h, w, 12))
    da = np.zeros((h, w, 12))
    for dz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                wxy = (fx if dx else 1 - fx) * (fy if dy else 1 - fy)
                c = grid[z0 + dz, y0 + dy, x0 + dx]
                a += (wxy * (fz if dz else 1 - fz))[..., None] * c
                da += (wxy * (1.0 if dz else -1.0))[..., None] * c
    return a, da


def np_slice(grid, img):
    a, _ = np_coeffs(grid, img)
    m = a.reshape(*a.shape[:2], 3, 4)
    out = np.empty_like(img, dtype=np.float64)
    out[..., 0:3] = np.einsum("hwij,hwj->hwi", m[..., 0:3], img[..., 0:3]) + m[..., 3]
    out[..., 3] = img[..., 3]
    return out


def np_slice_backward(grid, img, v_out):
    """(v_img [h,w,4], v_grid [L,H,W,12])."""
    h, w = img.shape[:2]
    a, da = np_coeffs(grid, img)
    m, dm = a.reshape(h, w, 3, 4), da.reshape(h, w, 3, 4)
    c, v = img[..., 0:3], v_out[..., 0:3]
    _, _, _, gray = lattice(h, w, img)
    v_img = np.empty((h, w, 4))
    v_img[..., 0:3] = np.einsum("hwij,hwi->hwj", m[..., 0:3], v)
    dz = np.einsum("hwi,hwi->hw", v, np.einsum("hwij,hwj->hwi", dm[..., 0:3], c) + dm[..., 3])
    inside = (gray > 0) & (gray < 1)
    v_img[..., 0:3] += np.where(inside, dz * (L - 1), 0.0)[..., None] * LUMA
    v_img[..., 3] = v_out[..., 3]
    g = np.concatenate([v[..., :, None] * c[..., None, :], v[..., :, None]], axis=-1).reshape(h, w, 12)
    gx, gy, gz, _ = lattice(h, w, img)
    x0, fx = _cells(gx, W)
    y0, fy = _cells(gy, H)
    z0, fz = _cells(gz, L)
    v_grid = np.zeros((L, H, W, 12))
    for dzz in (0, 1):
        for dy in (0, 1):
            for dx in (0, 1):
                wgt = (fx if dx else 1 - fx) * (fy if dy else 1 - fy) * (fz if dzz else 1 - fz)
                np.add.at(v_grid, (z0 + dzz, y0 + dy, x0 + dx), wgt[..., None] * g)
    return v_img, v_grid


def tv_counts():
    return 12 * (L - 1) * H * W, 12 * L * (H - 1) * W, 12 * L * H * (W - 1)


def np_tv(grid):
    """(TV(grid), dTV/dgrid) for one grid [L,H,W,12]."""
    pz, py, px = tv_counts()
    val, grad = 0.0, np.zeros_like(grid)
    for axis, p in ((0, pz), (1, py), (2, px)):
        d = np.diff(grid, axis=axis)
        val += float((d * d).sum()) / p
        pad_lo = [(0, 0)] * 4
        pad_hi = [(0, 0)] * 4
        pad_lo[axis] = (1, 0)
        pad_hi[axis] = (0, 1)
        grad += 2.0 / p * (np.pad(d, pad_lo) - np.pad(d, pad_hi))
    return val, grad


def torch_slice(grid, img):
    """grid, img: float64 torch tensors (may require grad); the grid_sample statement of the slice."""
    import torch
    import torch.nn.functional as F
    h, w = img.shape[:2]
    dev = img.device
    gx = (torch.arange(w, dtype=torch.float64, device=dev) + 0.5) / w
    gy = (torch.arange(h, dtype=torch.float64, device=dev) + 0.5) / h
    gray = img[..., 0] * 0.299 + img[..., 1] * 0.587 + img[..., 2] * 0.114
    gz = gray.clamp(0.0, 1.0)
    coords = torch.stack([gx[None, :].expand(h, w), gy[:, None].expand(h, w), gz], dim=-1) * 2.0 - 1.0
    g5 = grid.permute(3, 0, 1, 2)[None]                                  # [1, 12, L, H, W]
    a = F.grid_sample(g5, coords[None, None], mode="bilinear", padding_mode="border", align_corners=True)
    a = a[0, :, 0].permute(1, 2, 0).reshape(h, w, 3, 4)                 # [h, w, 3, 4]
    rgb = torch.einsum("hwij,hwj->hwi", a[..., 0:3], img[..., 0:3]) + a[..., 3]
    return torch.cat([rgb, img[..., 3:4]], dim=-1)


def torch_slice_backward(grid, img, v_out):
    import torch
    g = torch.tensor(grid, dtype=torch.float64, requires_grad=True)
    x = torch.tensor(img, dtype=torch.float64, requires_grad=True)
    out = torch_slice(g, x)
    out.backward(torch.tensor(v_out, dtype=torch.float64))
    return x.grad.numpy(), g.grad.numpy()


def torch_tv(grid):
    import torch
    g = torch.tensor(grid, dtype=torch.float64, requires_grad=True)
    pz, py, px = tv_counts()
    val = (torch.diff(g, dim=0) ** 2).sum() / pz + (torch.diff(g, dim=1) ** 2).sum() / py + (torch.diff(g, dim=2) ** 2).sum() / px
    val.backward()
    return float(val.detach()), g.grad.numpy()


def kink_mask(img, tol=1e-6):
    """Pixels where the slice is not differentiable in the colour, within tol: gray at a clamp (0 or 1) or at a level
    boundary of the z lattice."""
    gray = img[..., 0:3].astype(np.float64) @ LUMA
    gz = gray * (L - 1)
    near_level = np.abs(gz - np.round(gz)) < tol * (L - 1)
    return near_level | (np.abs(gray) < tol) | (np.abs(gray - 1.0) < tol)


def random_grid(rng, scale=0.3):
    return identity()[0] + rng.normal(0.0, scale, (L, H, W, 12))


def adam_ref(p, g, m, v, t, lr, beta1=0.9, beta2=0.999, eps=1e-15):
    """The project's Adam in float64 (AdamScaled, first step initialising the moments from g alone)."""
    m = g * (1 - beta1) if t == 1 else m * beta1 + g * (1 - beta1)
    v = g * g * (1 - beta2) if t == 1 else v * beta2 + g * g * (1 - beta2)
    p = p - lr * (m / (1 - beta1 ** t)) / (np.sqrt(v / (1 - beta2 ** t)) + eps)
    return p, m, v
