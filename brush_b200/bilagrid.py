"""Per-view appearance compensation (DESIGN.md section 4.11): one bilateral grid of 3x4 affine colour transforms per
training view (Wang et al., "Bilateral Guided Radiance Field Processing", SIGGRAPH 2024), sliced between the render and
the loss, learned with the splats and not part of the model: evaluation and export render without it.

  BilateralGrids          grids [views, L, H, W, 12] at identity, their Adam moments, each view's own step count
  slice / slice_backward  bg_bilagrid_slice / bg_bilagrid_slice_backward
  update                  bg_bilagrid_update: TV gradient and value, then Adam on one view's grid
  apply_bilateral_grid    a training view's render as the model explains it (the raw render sliced by its grid)
  bilagrid_lr             the learning-rate schedule: warm-up over 1000 steps, then exponential decay
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from .render import RenderContext, _stream_ptr

L, H, W = _lib.BILAGRID_L, _lib.BILAGRID_H, _lib.BILAGRID_W


def bilagrid_lr(lr0: float, n: int, total_train_iters: int) -> float:
    """lr(n) = lr0 * (0.01 + 0.99 * min(n - 1, 1000) / 1000) * 0.01 ** ((n - 1) / total_train_iters), n 1-based (the
    warm-up and decay gsplat uses for its grids)."""
    return lr0 * (0.01 + 0.99 * min(n - 1, 1000) / 1000.0) * 0.01 ** ((n - 1) / float(total_train_iters))


def identity_grids(num_views: int, device) -> torch.Tensor:
    """[views, L, H, W, 12], every cell M = I, b = 0."""
    eye = torch.tensor([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], dtype=torch.float32, device=device)
    return eye.repeat(num_views, L, H, W, 1).contiguous()


class BilateralGrids:
    """The grids of all training views, their Adam moments and the host-side per-view step counts.  A view's grid
    changes only in the steps that render that view."""

    def __init__(self, num_views: int, device):
        if num_views < 1:
            raise ValueError("BilateralGrids needs at least one view")
        self.num_views = int(num_views)
        self.grids = identity_grids(self.num_views, device)
        self.m = torch.zeros_like(self.grids)
        self.v = torch.zeros_like(self.grids)
        self.steps = [0] * self.num_views
        self.v_grid = torch.zeros((L, H, W, 12), dtype=torch.float32, device=self.grids.device)
        self.tv_loss = torch.zeros(1, dtype=torch.float32, device=self.grids.device)

    def check_view(self, view: int) -> int:
        if not 0 <= view < self.num_views:
            raise ValueError(f"view index {view} outside 0..{self.num_views - 1}")
        return int(view)

    def step_args(self, view: int, lr: float, tv_weight: float) -> "_lib.BgBilagridStep":
        """Counts one more step of `view` and returns its BgBilagridStep (tv_loss_out -> self.tv_loss)."""
        view = self.check_view(view)
        self.steps[view] += 1
        a = _lib.BgBilagridStep()
        a.grid, a.m, a.v = (t[view].data_ptr() for t in (self.grids, self.m, self.v))
        a.step, a.lr, a.tv_weight = self.steps[view], float(lr), float(tv_weight)
        a.tv_loss_out = self.tv_loss.data_ptr()
        return a


def _check(t: torch.Tensor, name: str, shape, device) -> torch.Tensor:
    """t must be a contiguous float32 tensor of `shape` on `device`: the kernels take its data pointer as such."""
    if (not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or tuple(t.shape) != tuple(shape) or not t.is_contiguous()
            or t.device != device):
        got = (tuple(t.shape), t.dtype, str(t.device)) if isinstance(t, torch.Tensor) else type(t)
        raise ValueError(f"{name} must be a contiguous float32 tensor {list(shape)} on {device}, got {got}")
    return t


def _img(t: torch.Tensor, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or t.dim() != 3 or not t.is_cuda:
        raise ValueError(f"{name} must be a contiguous float32 CUDA tensor [h, w, 4]")
    return _check(t, name, (t.shape[0], t.shape[1], 4), t.device)


def _grid(t: torch.Tensor, name: str, device) -> torch.Tensor:
    return _check(t, name, (L, H, W, 12), device)


def _disjoint(a: torch.Tensor, b: torch.Tensor, what: str) -> None:
    a0, b0 = a.data_ptr(), b.data_ptr()
    if a0 < b0 + b.numel() * 4 and b0 < a0 + a.numel() * 4:
        raise ValueError(f"{what} must not overlap")


def slice(ctx: RenderContext, grid: torch.Tensor, img: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """grid [L,H,W,12], img [h,w,4] -> (M c + b, alpha) [h,w,4]."""
    _img(img, "img")
    _grid(grid, "grid", img.device)
    out = torch.empty_like(img) if out is None else _check(out, "out", img.shape, img.device)
    _disjoint(out, img, "out and img")
    h, w = img.shape[0], img.shape[1]
    _lib.check(_lib.load().bg_bilagrid_slice(ctx.handle, _stream_ptr(ctx.device), grid.data_ptr(), img.data_ptr(), h, w,
                                             out.data_ptr()), "bg_bilagrid_slice")
    return out


def slice_backward(ctx: RenderContext, grid: torch.Tensor, img: torch.Tensor, v_out: torch.Tensor,
                   v_img: Optional[torch.Tensor] = None, v_grid: Optional[torch.Tensor] = None):
    """(dL/dimg, dL/dgrid) from dL/dout.  v_img may be v_out (in place); v_grid is overwritten."""
    _img(img, "img")
    _grid(grid, "grid", img.device)
    _check(v_out, "v_out", img.shape, img.device)
    v_img = torch.empty_like(v_out) if v_img is None else _check(v_img, "v_img", img.shape, img.device)
    v_grid = torch.empty((L, H, W, 12), dtype=torch.float32, device=img.device) if v_grid is None else _grid(v_grid, "v_grid", img.device)
    _disjoint(v_img, img, "v_img and img")
    if v_img.data_ptr() != v_out.data_ptr():
        _disjoint(v_img, v_out, "v_img and v_out (other than the same tensor)")
    h, w = img.shape[0], img.shape[1]
    _lib.check(_lib.load().bg_bilagrid_slice_backward(ctx.handle, _stream_ptr(ctx.device), grid.data_ptr(), img.data_ptr(),
                                                      v_out.data_ptr(), h, w, v_img.data_ptr(), v_grid.data_ptr()),
               "bg_bilagrid_slice_backward")
    return v_img, v_grid


def update(ctx: RenderContext, grids: BilateralGrids, view: int, v_grid: torch.Tensor, lr: float, tv_weight: float) -> torch.Tensor:
    """TV then Adam on the grid of `view` (its step count advances); v_grid gets the TV gradient added.  Returns the
    device scalar tv_weight * TV(grid) before the update: a view of a buffer that the next update of ANY view overwrites
    (clone it to keep it)."""
    _grid(v_grid, "v_grid", grids.grids.device)
    a = grids.step_args(view, lr, tv_weight)
    _lib.check(_lib.load().bg_bilagrid_update(ctx.handle, _stream_ptr(ctx.device), C.byref(a), v_grid.data_ptr()),
               "bg_bilagrid_update")
    return grids.tv_loss[0]


def apply_bilateral_grid(ctx: RenderContext, out_img: torch.Tensor, grids: BilateralGrids, view: int) -> torch.Tensor:
    """A training view's render [h,w,4] as the model explains it: sliced by the view's grid."""
    return slice(ctx, grids.grids[grids.check_view(view)], out_img)
