"""Host mirror of brush_loss::image_loss over the C ABI.

  image_loss_forward / image_loss_backward <- LossOps (brush-loss/src/lib.rs:718-733)
  image_loss                               <- image_loss (lib.rs:1075-1104) with autograd glue
  ImageLossConfig                          <- lib.rs:698-712

`pred` is the rasterizer's [h,w,C'] image (C' >= channels, typically the [h,w,4] render output);
it is consumed in place through strides instead of being permuted to CHW as the reference does.
The loss map and dl_dmap are dense [channels,h,w], as in the reference kernels.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional, Tuple

import torch

from . import _lib
from .render import RenderContext, _stream_ptr


@dataclass
class ImageLossConfig:
    l1_weight: float
    ssim_weight: float
    composite_bg: Optional[Tuple[float, float, float]] = None
    mask: bool = False


def _strides_hwc(pred: torch.Tensor):
    if pred.dim() != 3 or pred.dtype != torch.float32 or not pred.is_cuda:
        raise TypeError("pred must be a float32 CUDA tensor [h, w, c]")
    sy, sx, sc = pred.stride()
    return sc, sy, sx


def _bg_ptr(cfg: ImageLossConfig):
    if cfg.composite_bg is None:
        return None
    return (C.c_float * 3)(*[float(b) for b in cfg.composite_bg])


def image_loss_forward(ctx: RenderContext, pred_hwc: torch.Tensor, gt_packed: torch.Tensor, channels: int,
                       cfg: ImageLossConfig) -> torch.Tensor:
    lib = _lib.load()
    h, w = pred_hwc.shape[0], pred_hwc.shape[1]
    if gt_packed.shape != (h, w):
        raise ValueError("gt_packed height/width must match pred")
    sc, sy, sx = _strides_hwc(pred_hwc)
    out = torch.empty((channels, h, w), dtype=torch.float32, device=pred_hwc.device)
    _lib.check(lib.bg_image_loss_forward(ctx.handle, _stream_ptr(ctx.device), pred_hwc.data_ptr(), gt_packed.data_ptr(),
                                         channels, h, w, sc, sy, sx, cfg.l1_weight, cfg.ssim_weight, _bg_ptr(cfg),
                                         int(cfg.mask), out.data_ptr()), "bg_image_loss_forward")
    return out


def image_loss_backward(ctx: RenderContext, pred_hwc: torch.Tensor, gt_packed: torch.Tensor, dl_dmap: torch.Tensor,
                        channels: int, cfg: ImageLossConfig, out_hwc: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Returns dL/dpred with the layout (and strides) of pred_hwc; channels beyond `channels` stay zero."""
    lib = _lib.load()
    h, w = pred_hwc.shape[0], pred_hwc.shape[1]
    sc, sy, sx = _strides_hwc(pred_hwc)
    if out_hwc is None:
        out_hwc = torch.zeros_like(pred_hwc)
    if out_hwc.stride() != pred_hwc.stride():
        raise ValueError("out_hwc must have the strides of pred_hwc")
    dl_dmap = dl_dmap.contiguous()
    _lib.check(lib.bg_image_loss_backward(ctx.handle, _stream_ptr(ctx.device), pred_hwc.data_ptr(), gt_packed.data_ptr(),
                                          dl_dmap.data_ptr(), channels, h, w, sc, sy, sx, cfg.l1_weight, cfg.ssim_weight,
                                          _bg_ptr(cfg), int(cfg.mask), out_hwc.data_ptr()), "bg_image_loss_backward")
    return out_hwc


def image_loss_fused(ctx: RenderContext, pred_hwc: torch.Tensor, gt_packed: torch.Tensor, channels: int,
                     cfg: ImageLossConfig, chain_per_channel, out_hwc: Optional[torch.Tensor] = None,
                     weights: Optional[torch.Tensor] = None):
    """Train-path fusion (bg_image_loss_fused): for a loss that is a weighted mean of the map
    (train.rs:254-260) returns (dL/dpred [h,w,c'], loss scalar tensor) in one kernel pass.
    chain_per_channel[c] = dL/dmap of channel c; loss = sum_c chain[c] * sum(map[c]).
    weights: chain_per_channel as a device tensor, for callers that capture the call in a CUDA graph (no host copy inside)."""
    lib = _lib.load()
    h, w = pred_hwc.shape[0], pred_hwc.shape[1]
    if gt_packed.shape != (h, w):
        raise ValueError("gt_packed height/width must match pred")
    sc, sy, sx = _strides_hwc(pred_hwc)
    if out_hwc is None:
        out_hwc = torch.zeros_like(pred_hwc) if pred_hwc.shape[2] > channels else torch.empty_like(pred_hwc)
    n_part = int(lib.bg_image_loss_num_partials(channels, h, w))
    partials = torch.empty((channels, n_part // channels), dtype=torch.float32, device=pred_hwc.device)
    chain = (C.c_float * channels)(*[float(x) for x in chain_per_channel])
    _lib.check(lib.bg_image_loss_fused(ctx.handle, _stream_ptr(ctx.device), pred_hwc.data_ptr(), gt_packed.data_ptr(),
                                       channels, h, w, sc, sy, sx, cfg.l1_weight, cfg.ssim_weight, _bg_ptr(cfg),
                                       int(cfg.mask), chain, out_hwc.data_ptr(), partials.data_ptr()),
               "bg_image_loss_fused")
    if weights is None:
        weights = torch.tensor([float(x) for x in chain_per_channel], dtype=torch.float32, device=pred_hwc.device)
    loss = (partials.sum(dim=1) * weights).sum()
    return out_hwc, loss


def depth_loss_fused(ctx: RenderContext, pred_hwc: torch.Tensor, depth: torch.Tensor, target: torch.Tensor, chain: float,
                     out_hwc: torch.Tensor, v_depth: Optional[torch.Tensor] = None):
    """Depth-supervision term (bg_depth_loss_fused, DESIGN.md section 4.7) of a depth render: pred_hwc = out_img [h,w,4],
    depth = D [h,w], target = t [h,w] (valid where finite and > 0), chain = w_d / |valid pixels|.  ADDS dL/dalpha to
    out_hwc[...,3] in place on the active pixels and returns (v_depth [h,w], L_d scalar tensor)."""
    lib = _lib.load()
    h, w = pred_hwc.shape[0], pred_hwc.shape[1]
    for t, name, shape in ((pred_hwc, "pred_hwc", (h, w, 4)), (out_hwc, "out_hwc", (h, w, 4)), (depth, "depth", (h, w)),
                           (target, "target", (h, w))):
        if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous() or tuple(t.shape) != shape:
            raise ValueError(f"{name} must be a contiguous float32 CUDA tensor of shape {shape}")
    if v_depth is None:
        v_depth = torch.empty((h, w), dtype=torch.float32, device=pred_hwc.device)
    partials = torch.empty(int(lib.bg_depth_loss_num_partials(h, w)), dtype=torch.float32, device=pred_hwc.device)
    _lib.check(lib.bg_depth_loss_fused(ctx.handle, _stream_ptr(ctx.device), pred_hwc.data_ptr(), depth.data_ptr(),
                                       target.data_ptr(), h, w, float(chain), out_hwc.data_ptr(), v_depth.data_ptr(),
                                       partials.data_ptr()), "bg_depth_loss_fused")
    return v_depth, partials.sum() * float(chain)


class _ImageLoss(torch.autograd.Function):
    @staticmethod
    def forward(fctx, pred_hwc, gt_packed, ctx, channels, cfg):
        fctx.ctx, fctx.channels, fctx.cfg = ctx, channels, cfg
        fctx.save_for_backward(pred_hwc, gt_packed)
        return image_loss_forward(ctx, pred_hwc, gt_packed, channels, cfg).permute(1, 2, 0)

    @staticmethod
    def backward(fctx, dl_dmap_hwc):
        pred, gt = fctx.saved_tensors
        g = image_loss_backward(fctx.ctx, pred, gt, dl_dmap_hwc.permute(2, 0, 1).contiguous(), fctx.channels, fctx.cfg)
        return g, None, None, None, None


def image_loss(ctx: RenderContext, pred_hwc: torch.Tensor, gt_packed: torch.Tensor, cfg: ImageLossConfig,
               channels: int = 3) -> torch.Tensor:
    """L1 + SSIM loss map [h, w, channels] (lib.rs:1075-1104)."""
    return _ImageLoss.apply(pred_hwc, gt_packed, ctx, channels, cfg)
