"""Evaluation metrics (SURVEY 8f N3): eval_stats <- brush-train/src/eval.rs:22-61.

Render on black with the float output, round-trip through 8 bit, PSNR from the L1 map squared
(|a-b|^2 == (a-b)^2), SSIM as the mean of the SSIM map -- both through bg_image_loss_forward.  With a ground-truth depth
map, the depth metrics over the active pixels of DESIGN.md section 4.7 (valid target, alpha >= 1/255)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from .dataset import ALPHA_MASKED, view_to_packed_data
from .loss import ImageLossConfig, image_loss_forward
from .render import PASS_BACKWARD, RenderContext, RenderOutput, render_splats


@dataclass
class EvalSample:
    rendered: torch.Tensor     # [H,W,3] after the 8-bit round trip
    psnr: torch.Tensor         # scalar
    ssim: torch.Tensor         # scalar
    render_aux: RenderOutput
    depth_abs_rel: Optional[torch.Tensor] = None    # mean |ed - t| / t over the active pixels (ed = D / alpha)
    depth_rmse: Optional[torch.Tensor] = None       # sqrt(mean (ed - t)^2) over the active pixels, scene units
    depth_coverage: Optional[torch.Tensor] = None   # |active| / |valid|

    def save_to_disk(self, path: str) -> None:
        """eval.rs:66-81: the rendered image (already on the 8-bit grid) as an 8-bit RGB file; parent directories are
        created."""
        import os
        from PIL import Image
        img = (self.rendered.detach().clamp(0.0, 1.0) * 255.0).round().to(torch.uint8).cpu().numpy()
        os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
        Image.fromarray(img, "RGB").save(path)


def eval_stats(ctx: RenderContext, splats, camera, gt_image: np.ndarray, alpha_mode: str = ALPHA_MASKED,
               render_mip: bool = False, gt_depth: Optional[np.ndarray] = None) -> EvalSample:
    """splats: train.Splats (a min-scale floor is folded in, as in render_splats, gaussian_splats.rs:379-384).
    render_mip: the splats' render mode -- evaluation renders with the filter the model is trained with
    (gaussian_splats.rs:395: `splats.render_mip`).  gt_image: [H,W,3] or [H,W,4] u8; an alpha channel goes through
    view_to_packed_data(alpha_mode) like a training view (eval.rs:31).  gt_depth: optional f32 [H,W] depth target
    (SceneView.load_depth); adds the depth metrics, which are NaN when no pixel is active."""
    h, w = gt_image.shape[0], gt_image.shape[1]
    packed, _ = view_to_packed_data(gt_image, alpha_mode)
    gt = torch.from_numpy(packed).to(ctx.device)
    transforms, raw_opac = splats.folded(ctx)
    out = render_splats(ctx, camera, (w, h), transforms, splats.sh_coeffs, raw_opac, mip=render_mip,
                        background=(0.0, 0.0, 0.0), rpass=PASS_BACKWARD, render_depth=gt_depth is not None)
    rgb = torch.round(out.out_img[..., 0:3] * 255.0) / 255.0            # eval.rs:41-42
    rgb = rgb.contiguous()
    l1 = image_loss_forward(ctx, rgb, gt, 3, ImageLossConfig(1.0, 0.0, None, False))
    mse = l1.pow(2).mean()
    psnr = torch.log(1.0 / mse) * 10.0 / float(np.log(10.0))
    ssim = image_loss_forward(ctx, rgb, gt, 3, ImageLossConfig(0.0, 1.0, None, False)).mean()
    sample = EvalSample(rendered=rgb, psnr=psnr, ssim=ssim, render_aux=out)
    if gt_depth is not None:
        if tuple(gt_depth.shape) != (h, w):
            raise ValueError(f"gt_depth must be [{h},{w}], got {tuple(gt_depth.shape)}")
        t = torch.from_numpy(np.ascontiguousarray(gt_depth, np.float32)).to(ctx.device).double()
        a = out.out_img[..., 3]
        valid = torch.isfinite(t) & (t > 0)
        active = valid & (a >= np.float32(1.0 / 255.0))
        ed = (out.depth / a.clamp_min(1e-30)).double()
        err = (ed - t)[active]
        cnt = active.sum()
        nan = torch.tensor(float("nan"), dtype=torch.float64, device=ctx.device)
        sample.depth_abs_rel = (err.abs() / t[active]).mean() if bool(cnt > 0) else nan
        sample.depth_rmse = err.pow(2).mean().sqrt() if bool(cnt > 0) else nan
        nv = valid.sum()
        sample.depth_coverage = cnt.double() / nv.double() if bool(nv > 0) else nan
    return sample
