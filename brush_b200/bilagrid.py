"""Per-view appearance compensation (DESIGN.md section 4.11): one bilateral grid of 3x4 affine colour transforms per
training view (Wang et al., "Bilateral Guided Radiance Field Processing", SIGGRAPH 2024), sliced between the render and
the loss, learned with the splats and not part of the model: evaluation and export render without it.

  BilateralGrids          grids [views, L, H, W, 12] at identity, their Adam moments, each view's own step count
  slice / slice_backward  bg_bilagrid_slice / bg_bilagrid_slice_backward
  update                  bg_bilagrid_update: TV gradient and value, then Adam on one view's grid
  update_views            bg_bilagrid_update_views: the same for several gradient slots in one launch, a view's slots summed
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
    """The grids of all training views, their Adam moments and the per-view step counts.  A view's grid changes only in
    the steps that render that view, and its count is the number of those steps.

    The counts are kept twice: `steps`, a host list that the single-view steps advance, and `device_steps`, int32
    [views] that the multi-view steps advance on the device (a rank does not know the other ranks' views).  Each copy is
    brought up to date from the other only when a step of the other kind ran since: a 4 * views byte transfer when the
    path changes, none in a steady run of either."""

    def __init__(self, num_views: int, device):
        if num_views < 1:
            raise ValueError("BilateralGrids needs at least one view")
        self.num_views = int(num_views)
        self.grids = identity_grids(self.num_views, device)
        self.m = torch.zeros_like(self.grids)
        self.v = torch.zeros_like(self.grids)
        self._steps = [0] * self.num_views
        self._device_steps = torch.zeros(self.num_views, dtype=torch.int32, device=self.grids.device)
        self._current = "both"   # which copy of the counts is up to date: "host", "device" or "both"
        self.v_grid = torch.zeros((L, H, W, 12), dtype=torch.float32, device=self.grids.device)
        self.tv_loss = torch.zeros(1, dtype=torch.float32, device=self.grids.device)
        self.views_tv_loss = torch.zeros(16, dtype=torch.float32, device=self.grids.device)

    @property
    def steps(self) -> list:
        """Each view's step count, as a host list (read back once after multi-view steps)."""
        if self._current == "device":
            self._steps = [int(x) for x in self._device_steps.tolist()]
            self._current = "both"
        return self._steps

    @property
    def device_steps(self) -> torch.Tensor:
        """Each view's step count, int32 [views] on the device (written once after single-view steps).  Whoever reads it
        for a step that advances it on the device calls advance_on_device() first."""
        if self._current == "host":
            self._device_steps.copy_(torch.tensor(self._steps, dtype=torch.int32))
            self._current = "both"
        return self._device_steps

    def advance_on_device(self) -> torch.Tensor:
        """device_steps, marked as the only up-to-date copy: the caller's step advances it on the device."""
        t = self.device_steps
        self._current = "device"
        return t

    def check_view(self, view: int) -> int:
        if not 0 <= view < self.num_views:
            raise ValueError(f"view index {view} outside 0..{self.num_views - 1}")
        return int(view)

    def step_args(self, view: int, lr: float, tv_weight: float) -> "_lib.BgBilagridStep":
        """Counts one more step of `view` and returns its BgBilagridStep (tv_loss_out -> self.tv_loss)."""
        view = self.check_view(view)
        steps = self.steps
        steps[view] += 1
        self._current = "host"
        a = _lib.BgBilagridStep()
        a.grid, a.m, a.v = (t[view].data_ptr() for t in (self.grids, self.m, self.v))
        a.step, a.lr, a.tv_weight = steps[view], float(lr), float(tv_weight)
        a.tv_loss_out = self.tv_loss.data_ptr()
        return a

    def views_args(self, view_index, lr: float, tv_weight: float, tv_out: torch.Tensor):
        """The BgBilagridViews of a step (or an update) whose counts advance on the device; view_index: the local views'
        training-view indices (None for bg_bilagrid_update_views).  Returns it with the host array it points into."""
        a = _lib.BgBilagridViews()
        a.grids, a.m, a.v = self.grids.data_ptr(), self.m.data_ptr(), self.v.data_ptr()
        a.steps = self.advance_on_device().data_ptr()
        a.num_views = self.num_views
        idx = None
        if view_index is not None:
            idx = (C.c_uint32 * len(view_index))(*[self.check_view(v) for v in view_index])
            a.view_index = idx
        a.lr, a.tv_weight = float(lr), float(tv_weight)
        a.tv_loss_out = tv_out.data_ptr()
        return a, idx


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


def update_views(ctx: RenderContext, grids: BilateralGrids, slot_view, v_grids: torch.Tensor, lr: float,
                 tv_weight: float) -> torch.Tensor:
    """One update of every view named in slot_view (1..16 training-view indices, one per gradient slot of v_grids
    [slots, L, H, W, 12]): a view's slots summed in slot order (into its first slot), TV, then Adam with the view's count
    + 1, bit-identical to update() given that sum; each named view's count advances by one.  Returns the device [slots]
    TV values (every slot of a view gets its view's value)."""
    slot_view = [grids.check_view(v) for v in slot_view]
    if not 1 <= len(slot_view) <= 16:
        raise ValueError("update_views takes 1..16 slots")
    dev = grids.grids.device
    _check(v_grids, "v_grids", (len(slot_view), L, H, W, 12), dev)
    sv = torch.tensor(slot_view, dtype=torch.int32, device=dev)
    tv = torch.empty(len(slot_view), dtype=torch.float32, device=dev)
    a, _ = grids.views_args(None, lr, tv_weight, tv)
    _lib.check(_lib.load().bg_bilagrid_update_views(ctx.handle, _stream_ptr(ctx.device), C.byref(a), len(slot_view), sv.data_ptr(),
                                                    v_grids.data_ptr()), "bg_bilagrid_update_views")
    return tv


def apply_bilateral_grid(ctx: RenderContext, out_img: torch.Tensor, grids: BilateralGrids, view: int) -> torch.Tensor:
    """A training view's render [h,w,4] as the model explains it: sliced by the view's grid."""
    return slice(ctx, grids.grids[grids.check_view(view)], out_img)
