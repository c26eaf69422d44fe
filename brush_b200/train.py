"""Host mirror of brush-train's per-step path over the C ABI.

  TrainConfig         <- brush-train/src/config.rs:5-132 (the fields the step uses, same defaults)
  Splats              <- brush-render/src/gaussian_splats.rs:57-74 (packed [N,10] / [N,K,3] / [N])
  SceneBatch          <- brush-dataset/src/scene.rs:138-162
  SplatTrainer.step   <- brush-train/src/train.rs:176-429
  bounds_from_pos / BoundingBox.median_size <- splat_init.rs:130-160, bounding_box.rs:23-29

Per step: render forward -> fused L1+SSIM loss -> loss backward -> rasterize/project backward ->
[optional gradient all-reduce hook for view-sharded data parallelism] -> Adam on the three parameter
tensors -> refine statistics + mean noise.  All device work goes through libbrush_b200.so; torch
provides memory, streams and (for N>1) torch.distributed.

  SplatTrainer.refine <- brush-train/src/train.rs:431-893 (prune / resample / force-split / grow / split /
                         opacity decay / bounds) through bg_refine + bg_bounds_percentile (csrc/refine.cu): flag scans,
                         row compaction, Efraimidis-Spirakis keys + the radix sort instead of a host readback into
                         rand::sample_weighted (multinomial.rs:1-26); the counts are the only readback.

  Splats.min_scale / set_view_cams <- the Mip-Splatting 3D-filter floor: compute_min_scale (train.rs:102-125),
                         fold_min_scale / bake_min_scale (gaussian_splats.rs:86-111, 245-252); the floor is folded
                         into scales/opacity for every render, its gradient chained back in place, baked at the
                         start of refine() and recomputed at its end while progress < 0.9 (train.rs:437, 641-647).

Out of scope here: LPIPS.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field
from typing import Callable, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .camera import Camera
from .loss import ImageLossConfig, depth_loss_fused, image_loss_fused
from .render import (PASS_BACKWARD, RenderContext, _stream_ptr, project_bwd, project_bwd_factored, rasterize_bwd,
                     rasterize_bwd_depth, render_splats, sh_grad_from_views)


@dataclass
class TrainConfig:
    total_train_iters: int = 30000
    lr_mean: float = 2e-5
    lr_mean_end: float = 2e-7
    mean_noise_weight: float = 50.0
    lr_coeffs_dc: float = 2e-3
    lr_coeffs_sh_scale: float = 10.0
    lr_opac: float = 0.012
    lr_scale: float = 5e-3
    lr_rotation: float = 2e-3
    ssim_weight: float = 0.2
    opac_decay: float = 0.004
    max_splats: int = 10_000_000
    refine_every: int = 200
    growth_grad_threshold: float = 0.0025
    growth_select_fraction: float = 0.25
    growth_stop_iter: int = 15000
    split_at_screen_size: float = 0.5
    match_alpha_weight: float = 0.1
    background_color: Sequence[float] = (0.0, 0.0, 0.0)
    background_noise_strength: float = 0.1
    render_mip: bool = False
    # depth supervision (DESIGN.md section 4.7): weight of the L1 term on the expected depth of views that carry a depth
    # map; 0 leaves the step exactly as without it.  Keyword-only, so the positional order of every other field and the
    # trailing seed + LOD fields stay as they were.
    depth_loss_weight: float = field(default=0.0, kw_only=True)
    seed: int = 0  # the reference uses an unseeded rand::rng(); a shared seed keeps DP ranks identical
    # LOD baking (config.rs:108-125): after the main run, lod_levels times score, keep lod_decimation_keep % of the splats
    # and retrain lod_refine_steps steps on images scaled by lod_image_scale % per level
    lod_levels: int = 0
    lod_refine_steps: int = 5000
    lod_decimation_keep: int = 50
    lod_image_scale: int = 50

    def __post_init__(self):
        if not (math.isfinite(self.depth_loss_weight) and self.depth_loss_weight >= 0.0):
            raise ValueError(f"depth_loss_weight must be finite and >= 0, got {self.depth_loss_weight}")
        if self.lod_levels < 0:
            raise ValueError("lod_levels must be >= 0")
        for name in ("lod_decimation_keep", "lod_image_scale"):
            if not 1 <= getattr(self, name) <= 100:
                raise ValueError(f"{name} is a percentage in 1..100, got {getattr(self, name)}")
        if self.lod_levels > 0 and self.lod_refine_steps <= 0:
            raise ValueError("lod_refine_steps must be > 0 when lod_levels > 0")

    def total_iters(self) -> int:
        """config.rs:141-143: the main run plus every LOD refine phase."""
        return self.total_train_iters + self.lod_levels * self.lod_refine_steps


@dataclass
class Splats:
    transforms: torch.Tensor      # [N,10]
    sh_coeffs: torch.Tensor       # [N,K,3]
    raw_opacities: torch.Tensor   # [N]
    min_scale: Optional[torch.Tensor] = None   # [N] world-space scale floor (gaussian_splats.rs:73), a constant

    def num_splats(self) -> int:
        return self.transforms.shape[0]

    def folded(self, ctx: RenderContext):
        """(transforms, raw_opacities) as the renderer must see them (gaussian_splats.rs:212-223, 379-384)."""
        if self.min_scale is None:
            return self.transforms, self.raw_opacities
        return fold_min_scale(ctx, self.transforms, self.raw_opacities, self.min_scale)

    def bake_min_scale(self, ctx: RenderContext) -> None:
        """Splats::bake_min_scale (gaussian_splats.rs:245-252): fold permanently, in place, and drop the floor."""
        if self.min_scale is not None:
            fold_min_scale(ctx, self.transforms, self.raw_opacities, self.min_scale, out=(self.transforms, self.raw_opacities))
            self.min_scale = None


def fold_min_scale(ctx: RenderContext, transforms, raw_opac, f, out=None):
    lib = _lib.load()
    n = transforms.shape[0]
    t_out, o_out = out if out is not None else (torch.empty_like(transforms), torch.empty_like(raw_opac))
    _lib.check(lib.bg_fold_min_scale_forward(ctx.handle, _stream_ptr(ctx.device), n, transforms.data_ptr(), raw_opac.data_ptr(),
                                             f.data_ptr(), t_out.data_ptr(), o_out.data_ptr()), "bg_fold_min_scale_forward")
    return t_out, o_out


def fold_min_scale_backward(ctx: RenderContext, transforms, raw_opac, f, v_transforms, v_raw_opac) -> None:
    """In place: gradients w.r.t. the folded values -> w.r.t. the learned ones."""
    lib = _lib.load()
    _lib.check(lib.bg_fold_min_scale_backward(ctx.handle, _stream_ptr(ctx.device), transforms.shape[0], transforms.data_ptr(),
                                              raw_opac.data_ptr(), f.data_ptr(), v_transforms.data_ptr(),
                                              v_raw_opac.data_ptr()), "bg_fold_min_scale_backward")


def compute_min_scale(ctx: RenderContext, transforms, view_cams: torch.Tensor, factor: float) -> Optional[torch.Tensor]:
    """compute_min_scale (train.rs:102-125).  view_cams: device [views,4] = (x, y, z, focal_px)."""
    if factor <= 0.0 or view_cams is None or view_cams.shape[0] == 0:
        return None
    lib = _lib.load()
    f = torch.empty(transforms.shape[0], dtype=torch.float32, device=transforms.device)
    _lib.check(lib.bg_compute_min_scale(ctx.handle, _stream_ptr(ctx.device), transforms.shape[0], transforms.data_ptr(),
                                        view_cams.data_ptr(), view_cams.shape[0], float(factor), f.data_ptr()),
               "bg_compute_min_scale")
    return f


@dataclass
class SceneBatch:
    img_packed: torch.Tensor      # [H,W] int32 (rgba8 little endian); host (pinned) or device
    camera: Camera
    has_alpha: bool = False
    masked_alpha: bool = False    # AlphaMode::Masked
    depth: Optional[torch.Tensor] = None   # [H,W] f32 metric camera-space z target, 0 = no measurement; host (pinned) or device
    depth_count: int = 0                    # valid pixels of `depth` (finite and > 0), counted on the host

    def img_size(self):
        return int(self.img_packed.shape[0]), int(self.img_packed.shape[1])


@dataclass
class BoundingBox:
    center: np.ndarray
    extent: np.ndarray

    def median_size(self) -> float:
        """bounding_box.rs:23-29: twice the middle extent, ordered by f32::total_cmp (a NaN extent sorts last instead of
        breaking the comparison)."""
        def key(x):
            b = int(np.float32(x).view(np.int32))
            return b ^ (((b >> 31) & 0xFFFFFFFF) >> 1)
        e = sorted((float(x) for x in self.extent), key=key)
        return e[1] * 2.0


def bounds_from_pos(percentile: float, means: np.ndarray) -> BoundingBox:
    """splat_init.rs:130-160."""
    cols = []
    for a in range(3):
        v = means[:, a]
        v = np.sort(v[np.isfinite(v)])
        if v.size == 0:
            return BoundingBox(np.zeros(3, np.float32), np.ones(3, np.float32))
        n = v.size
        lo = int((np.float32(1.0) - np.float32(percentile)) / np.float32(2.0) * np.float32(n))   # all in f32, like the reference
        hi = min(n - 1, int((np.float32(1.0) + np.float32(percentile)) / np.float32(2.0) * np.float32(n)))
        cols.append((v[lo], v[hi]))
    mn = np.array([c[0] for c in cols], np.float32)
    mx = np.array([c[1] for c in cols], np.float32)
    return BoundingBox((mx + mn) / 2.0, (mx - mn) / 2.0)


@dataclass
class RefineStats:
    """brush-train/src/msg.rs RefineStats."""
    num_added: int
    num_split_oversized: int
    num_split_high_grad: int
    num_pruned: int
    num_pruned_non_finite: int
    total_splats: int


MIN_SCALE_FREEZE_FRAC = 0.9   # train.rs:37
MIN_SCALE_FACTOR = 0.1        # train.rs:44
MIN_OPACITY = 1.0 / 255.0
BOUND_PERCENTILE = 0.8
FRAC_1_SQRT_2 = 0.7071067811865476


def bounds_from_pos_device(ctx: RenderContext, percentile: float, transforms: torch.Tensor) -> BoundingBox:
    """splat_init.rs:130-160 on the device (bg_bounds_percentile: three radix sorts, six scalars read back).
    transforms: [n,10] (the means are its first three columns)."""
    lib = _lib.load()
    n = int(transforms.shape[0])
    if n == 0:
        return BoundingBox(np.zeros(3, np.float32), np.ones(3, np.float32))
    need = int(lib.bg_refine_workspace_bytes(n))
    ws = torch.empty(need, dtype=torch.uint8, device=ctx.device)
    out = (C.c_float * 6)()
    _lib.check(lib.bg_bounds_percentile(ctx.handle, _stream_ptr(ctx.device), n, transforms.data_ptr(), float(percentile), ws.data_ptr(),
                                        need, out), "bg_bounds_percentile")
    mm = np.array(list(out), np.float32).reshape(3, 2)
    if not np.isfinite(mm).all():
        return BoundingBox(np.zeros(3, np.float32), np.ones(3, np.float32))
    return BoundingBox((mm[:, 1] + mm[:, 0]) / 2.0, (mm[:, 1] - mm[:, 0]) / 2.0)


@dataclass
class TrainStepStats:
    num_visible_event: object
    lr_mean: float
    loss: torch.Tensor  # lazy device scalar (msg.rs:16-27); image loss + depth loss
    depth_loss: Optional[torch.Tensor] = None   # the depth term alone (None when the batch carries no depth)


class SplatTrainer:
    def __init__(self, config: TrainConfig, ctx: RenderContext, bounds: BoundingBox,
                 grad_hook: Optional[Callable[[Sequence[torch.Tensor]], None]] = None):
        self.config = config
        self.ctx = ctx
        self.bounds = bounds
        self.lr_mean_decay = (config.lr_mean_end / config.lr_mean) ** (1.0 / config.total_train_iters)
        self.ssim_enabled = config.ssim_weight > 0.0
        self.step_count = 0
        self.grad_hook = grad_hook  # called with the gradient tensors before Adam (DP all-reduce)
        self._state = None
        self._v_output = None
        self._v_output_ch = 0
        # ctx may be None for refine()-only use (pure tensor logic, runs on whatever device the splats are on)
        self._gen = torch.Generator(device=ctx.device if ctx is not None else "cpu")
        self._gen.manual_seed(config.seed)
        self._host_rng = np.random.default_rng(config.seed)
        self.view_cams: Optional[torch.Tensor] = None
        self._views_buf = None
        self._views_ws = None
        self._views_loss = None
        self._dp_comm = None
        self._dp_group = None
        self._fused_ws = None
        self._fused_loss = None
        self._fused_depth_loss = None
        self._v_output_depth = None

    def set_view_cams(self, view_cams) -> None:
        """train.rs:172-174.  view_cams: sequence of ((x, y, z), focal_px) of the training views."""
        rows = [[float(c[0][0]), float(c[0][1]), float(c[0][2]), float(c[1])] for c in view_cams]
        dev = self.ctx.device if self.ctx is not None else "cpu"
        self.view_cams = torch.tensor(rows, dtype=torch.float32, device=dev).reshape(-1, 4) if rows else None

    # -- optimizer state (train.rs:300-326, adam_scaled.rs)
    def _ensure_state(self, s: Splats):
        if self._state is not None:
            return
        n, k = s.num_splats(), s.sh_coeffs.shape[1]
        dev = s.transforms.device
        z = lambda *shape: torch.zeros(shape, dtype=torch.float32, device=dev)
        scales = np.ones(k, np.float32)
        scales[1:] = np.float32(1.0) / np.float32(self.config.lr_coeffs_sh_scale)
        self._state = dict(
            m_t=z(n, 10), v_t=z(n, 10), m_sh=z(n, k, 3), v_sh=z(n), m_o=z(n), v_o=z(n),
            sh_lr_scale=torch.from_numpy(np.repeat(scales, 3)).to(dev),
            t_lr=torch.zeros(10, dtype=torch.float32, device=dev),
            refine_norm=z(n), vis_weight=z(n), max_screen=z(n),
        )

    def _adam(self, p, g, m, v, lr, scale, reduce_v):
        lib = _lib.load()
        rows = p.shape[0]
        cols = p.numel() // max(rows, 1)
        _lib.check(lib.bg_adam_step(self.ctx.handle, _stream_ptr(self.ctx.device), p.data_ptr(), g.data_ptr(), m.data_ptr(),
                                    v.data_ptr(), rows, cols, scale.data_ptr() if scale is not None else None,
                                    float(lr), 0.9, 0.999, 1e-15, self.step_count, int(reduce_v)), "bg_adam_step")

    def sample_background(self):
        base = np.asarray(self.config.background_color, np.float32)
        s = self.config.background_noise_strength
        if s <= 0.0:
            return tuple(float(x) for x in np.clip(base, 0.0, 1.0))
        noise = self._host_rng.uniform(-s, s, 3).astype(np.float32)
        return tuple(float(x) for x in np.clip(base + noise, 0.0, 1.0))

    def _depth_term(self, batch: SceneBatch) -> bool:
        """Whether this step runs the depth term (DESIGN.md section 4.7): a positive weight and a map with valid pixels."""
        return self.config.depth_loss_weight > 0.0 and batch.depth is not None and batch.depth_count > 0

    def _depth_target(self, batch: SceneBatch) -> torch.Tensor:
        img_h, img_w = batch.img_size()
        t = batch.depth.to(self.ctx.device, non_blocking=True)
        if t.dtype != torch.float32 or tuple(t.shape) != (img_h, img_w) or not t.is_contiguous():
            raise ValueError(f"SceneBatch.depth must be a contiguous float32 [{img_h},{img_w}] tensor")
        return t

    def _depth_chain(self, batch: SceneBatch) -> float:
        return float(np.float32(self.config.depth_loss_weight) / np.float32(batch.depth_count))   # w_d / |valid|, in f32

    def step(self, batch: SceneBatch, splats: Splats) -> TrainStepStats:
        if self._depth_term(batch):
            return self._step_depth(batch, splats)
        cfg = self.config
        self._ensure_state(splats)
        st = self._state
        self.step_count += 1
        img_h, img_w = batch.img_size()
        dev = self.ctx.device
        gt_packed = batch.img_packed.to(dev, non_blocking=True)           # H2D upload (train.rs:197-198)
        background = self.sample_background()
        median_scale = self.bounds.median_size()

        r_transforms, r_raw_opac = splats.folded(self.ctx)   # 3D-filter floor folded in (bwd/burn_glue.rs:260-270)
        out = render_splats(self.ctx, batch.camera, (img_w, img_h), r_transforms, splats.sh_coeffs,
                            r_raw_opac, mip=cfg.render_mip, background=background, rpass=PASS_BACKWARD)
        # loss config (train.rs:220-249)
        l1_w, ssim_w = (1.0 - cfg.ssim_weight, -cfg.ssim_weight) if self.ssim_enabled else (1.0, 0.0)
        do_alpha_match = batch.has_alpha and not batch.masked_alpha and cfg.match_alpha_weight > 0.0
        composite = background if (batch.has_alpha and any(b != 0.0 for b in background)) else None
        lcfg = ImageLossConfig(l1_w, ssim_w, composite, batch.masked_alpha)
        channels = 4 if do_alpha_match else 3
        # loss = mean over [h,w,3] (+ alpha mean * weight) (train.rs:254-260): dL/dmap is one constant per
        # channel, so value and gradient come from the fused kernel in one pass.
        npx = float(img_h * img_w)
        chain = [1.0 / (3.0 * npx)] * 3 + ([cfg.match_alpha_weight / npx] if do_alpha_match else [])
        if self._v_output is None or self._v_output.shape != out.out_img.shape or self._v_output_ch != channels:
            self._v_output = torch.zeros_like(out.out_img)   # channel 3 stays zero unless alpha matching
            self._v_output_ch = channels
        v_output, loss = image_loss_fused(self.ctx, out.out_img, gt_packed, channels, lcfg, chain, self._v_output)
        v_combined = rasterize_bwd(out, v_output)
        v_t, v_sh, v_o, v_r = project_bwd(out, r_transforms, splats.sh_coeffs, r_raw_opac, v_combined)
        if splats.min_scale is not None:
            fold_min_scale_backward(self.ctx, splats.transforms, splats.raw_opacities, splats.min_scale, v_t, v_o)
        if self.grad_hook is not None:
            self.grad_hook((v_t, v_sh, v_o, v_r, out.visible, out.max_radius))

        lr_mean = self._apply_updates(splats, v_t, v_sh, v_o, v_r, out.visible, out.max_radius, median_scale)
        depth_loss = torch.zeros((), dtype=torch.float32, device=dev) if batch.depth is not None else None
        return TrainStepStats(num_visible_event=out, lr_mean=lr_mean, loss=loss, depth_loss=depth_loss)

    def _step_depth(self, batch: SceneBatch, splats: Splats) -> TrainStepStats:
        """step() with the depth term: depth render -> image loss -> depth loss (adds dL/dalpha to v_output[...,3]) ->
        depth rasterize backward -> projection backward with v_z; the floor backward, the hook and the update as in step()."""
        cfg = self.config
        self._ensure_state(splats)
        self.step_count += 1
        img_h, img_w = batch.img_size()
        dev = self.ctx.device
        gt_packed = batch.img_packed.to(dev, non_blocking=True)
        target = self._depth_target(batch)
        background = self.sample_background()
        median_scale = self.bounds.median_size()

        r_transforms, r_raw_opac = splats.folded(self.ctx)
        out = render_splats(self.ctx, batch.camera, (img_w, img_h), r_transforms, splats.sh_coeffs,
                            r_raw_opac, mip=cfg.render_mip, background=background, rpass=PASS_BACKWARD, render_depth=True)
        l1_w, ssim_w = (1.0 - cfg.ssim_weight, -cfg.ssim_weight) if self.ssim_enabled else (1.0, 0.0)
        do_alpha_match = batch.has_alpha and not batch.masked_alpha and cfg.match_alpha_weight > 0.0
        composite = background if (batch.has_alpha and any(b != 0.0 for b in background)) else None
        lcfg = ImageLossConfig(l1_w, ssim_w, composite, batch.masked_alpha)
        channels = 4 if do_alpha_match else 3
        npx = float(img_h * img_w)
        chain = [1.0 / (3.0 * npx)] * 3 + ([cfg.match_alpha_weight / npx] if do_alpha_match else [])
        # a buffer of its own: the depth term writes channel 3, which the plain step's buffer keeps at zero
        if self._v_output_depth is None or self._v_output_depth.shape != out.out_img.shape:
            self._v_output_depth = torch.zeros_like(out.out_img)
        elif channels == 3:
            self._v_output_depth[..., 3].zero_()
        v_output, loss = image_loss_fused(self.ctx, out.out_img, gt_packed, channels, lcfg, chain, self._v_output_depth)
        v_depth, depth_loss = depth_loss_fused(self.ctx, out.out_img, out.depth, target, self._depth_chain(batch), v_output)
        v_combined, v_z = rasterize_bwd_depth(out, v_output, v_depth)
        v_t, v_sh, v_o, v_r = project_bwd(out, r_transforms, splats.sh_coeffs, r_raw_opac, v_combined, v_z=v_z)
        if splats.min_scale is not None:
            fold_min_scale_backward(self.ctx, splats.transforms, splats.raw_opacities, splats.min_scale, v_t, v_o)
        if self.grad_hook is not None:
            self.grad_hook((v_t, v_sh, v_o, v_r, out.visible, out.max_radius))

        lr_mean = self._apply_updates(splats, v_t, v_sh, v_o, v_r, out.visible, out.max_radius, median_scale)
        return TrainStepStats(num_visible_event=out, lr_mean=lr_mean, loss=loss + depth_loss, depth_loss=depth_loss)


    # ------------------------------------------------------------------------------------------------
    def step_fused(self, batch: SceneBatch, splats: Splats) -> TrainStepStats:
        """The same step through ONE ABI call (bg_train_step): every launch of the step is issued by the library on
        the current stream, scratch comes from a workspace allocated once.  No min-scale floor, no gradient hook.
        A batch that carries depth goes through bg_train_step_depth (the depth term of DESIGN.md section 4.7)."""
        if splats.min_scale is not None or self.grad_hook is not None:
            raise ValueError("step_fused handles the plain single-view step; use step() with a scale floor or a gradient hook")
        cfg = self.config
        self._ensure_state(splats)
        self.step_count += 1
        img_h, img_w = batch.img_size()
        dev = self.ctx.device
        lib = _lib.load()
        gt_packed = batch.img_packed.to(dev, non_blocking=True)
        background = self.sample_background()
        median_scale = self.bounds.median_size()
        n, k = splats.num_splats(), splats.sh_coeffs.shape[1]
        with_depth = batch.depth is not None
        need = int((lib.bg_train_step_depth_workspace_bytes if with_depth else lib.bg_train_step_workspace_bytes)(n, k, img_w, img_h))
        if self._fused_ws is None or self._fused_ws.numel() < need:
            self._fused_ws = torch.empty(need, dtype=torch.uint8, device=dev)
            self._fused_loss = torch.zeros(1, dtype=torch.float32, device=dev)
        a, lr_mean = self._fused_args(batch, splats, gt_packed, background, median_scale, self._fused_ws, need)
        a.loss_out = self._fused_loss.data_ptr()
        if not with_depth:
            _lib.check(lib.bg_train_step(self.ctx.handle, _stream_ptr(dev), C.byref(a)), "bg_train_step")
            return TrainStepStats(num_visible_event=None, lr_mean=lr_mean, loss=self._fused_loss[0])
        # bg_train_step_depth runs bg_train_step itself when the term is off (weight 0 or no valid pixel)
        if self._fused_depth_loss is None:
            self._fused_depth_loss = torch.zeros(1, dtype=torch.float32, device=dev)
        ds = _lib.BgDepthSupervision()
        target = self._depth_target(batch) if self._depth_term(batch) else None
        ds.target = target.data_ptr() if target is not None else None
        ds.weight, ds.valid_count = float(cfg.depth_loss_weight), int(batch.depth_count)
        ds.depth_loss_out = self._fused_depth_loss.data_ptr()
        _lib.check(lib.bg_train_step_depth(self.ctx.handle, _stream_ptr(dev), C.byref(a), C.byref(ds)), "bg_train_step_depth")
        self._fused_keepalive = target
        return TrainStepStats(num_visible_event=None, lr_mean=lr_mean, loss=self._fused_loss[0],
                              depth_loss=self._fused_depth_loss[0])

    def _fused_args(self, batch: SceneBatch, splats: Splats, gt_packed, background, median_scale, ws, need):
        """BgTrainStepArgs of step_fused for the current step_count (loss_out left unset)."""
        cfg, st = self.config, self._state
        img_h, img_w = batch.img_size()
        n, k = splats.num_splats(), splats.sh_coeffs.shape[1]
        from .camera import build_uniforms
        a = _lib.BgTrainStepArgs()
        a.cam = _lib.camera_struct(build_uniforms(batch.camera, img_w, img_h))
        a.w, a.h, a.n, a.k, a.mip = img_w, img_h, n, k, int(cfg.render_mip)
        for i in range(3):
            a.background[i] = float(background[i])
        a.transforms, a.sh, a.raw_opac = splats.transforms.data_ptr(), splats.sh_coeffs.data_ptr(), splats.raw_opacities.data_ptr()
        a.m_t, a.v_t, a.m_sh, a.v_sh, a.m_o, a.v_o = (st[x].data_ptr() for x in ("m_t", "v_t", "m_sh", "v_sh", "m_o", "v_o"))
        a.refine_norm, a.vis_weight, a.max_screen = (st[x].data_ptr() for x in ("refine_norm", "vis_weight", "max_screen"))
        a.gt_packed = gt_packed.data_ptr()
        a.l1_weight, a.ssim_weight = (1.0 - cfg.ssim_weight, -cfg.ssim_weight) if self.ssim_enabled else (1.0, 0.0)
        do_alpha_match = batch.has_alpha and not batch.masked_alpha and cfg.match_alpha_weight > 0.0
        comp = batch.has_alpha and any(b != 0.0 for b in background)
        a.has_composite_bg = int(comp)
        for i in range(3):
            a.composite_bg[i] = float(background[i])
        a.mask, a.channels, a.alpha_weight = int(batch.masked_alpha), (4 if do_alpha_match else 3), float(cfg.match_alpha_weight)
        lr_mean = cfg.lr_mean * self.lr_mean_decay ** (self.step_count - 1) * float(median_scale)
        a.lr_mean, a.lr_rotation, a.lr_scale = float(np.float32(lr_mean)), cfg.lr_rotation, cfg.lr_scale
        a.lr_coeffs_dc, a.lr_coeffs_sh_scale, a.lr_opac = cfg.lr_coeffs_dc, cfg.lr_coeffs_sh_scale, cfg.lr_opac
        a.noise_scale = float(np.float32(lr_mean) * np.float32(cfg.mean_noise_weight))
        a.median_scale, a.seed, a.step = float(median_scale), int(cfg.seed), self.step_count
        a.workspace, a.workspace_bytes = ws.data_ptr(), need
        return a, lr_mean

    # ------------------------------------------------------------------------------------------------
    def step_views(self, batches: Sequence[SceneBatch], splats: Splats, group=None, chunks: int = 0,
                   distributed: Optional[bool] = None) -> TrainStepStats:
        """One optimizer step over several views (SURVEY 8e, BASELINE config [4]) through ONE ABI call
        (bg_train_step_views): the loss is the mean of the per-view losses, i.e. the step equals accumulating the
        views' gradients sequentially on one GPU.  Under torch.distributed every rank passes ITS views (the same count
        on every rank, global view index = rank * local + i); the library exchanges the SH-factored gradients over its
        own NCCL communicator (all-reduce SUM 48 N B, all-reduce MAX 8 N B, all-gather 12 local N B per rank), runs the SH
        part of the update pass under the all-reduces, and all ranks apply bit-identical updates.  At most 16 views per step in total.  All views of a
        step share the image size and the loss configuration.  distributed=False runs the step on this device alone even
        inside an initialised process group."""
        import torch.distributed as dist
        cfg = self.config
        self._ensure_state(splats)
        st = self._state
        dev = self.ctx.device
        lib = _lib.load()
        multi = dist.is_initialized() and dist.get_world_size(group) > 1 if distributed is None else bool(distributed)
        world = dist.get_world_size(group) if multi else 1
        local = len(batches)
        if local == 0 or local * world > 16:
            raise ValueError("step_views needs 1..16 views per step in total")
        if cfg.depth_loss_weight > 0.0 and any(b.depth is not None for b in batches):
            raise ValueError("step_views has no depth term: train views with depth through step() or step_fused()")
        if multi and (self._dp_comm is None or self._dp_group is not group):
            from .dp import DpComm
            self._dp_comm, self._dp_group = DpComm(self.ctx, group), group
        self.step_count += 1
        n, k = splats.num_splats(), splats.sh_coeffs.shape[1]
        img_h, img_w = batches[0].img_size()
        b0 = batches[0]
        for b in batches:
            if b.img_size() != (img_h, img_w) or (b.has_alpha, b.masked_alpha) != (b0.has_alpha, b0.masked_alpha):
                raise ValueError("the views of one step must share the image size and the alpha mode")
        need = int(lib.bg_train_step_views_workspace_bytes(n, k, img_w, img_h, local, world))
        if self._views_ws is None or self._views_ws.numel() < need:
            self._views_ws = torch.empty(need, dtype=torch.uint8, device=dev)
            self._views_loss = torch.zeros(1, dtype=torch.float32, device=dev)
        from .camera import build_uniforms
        background = self.sample_background()          # shared seed: identical on every rank
        median_scale = self.bounds.median_size()
        gts = [b.img_packed.to(dev, non_blocking=True) for b in batches]
        a = _lib.BgTrainViewsArgs()
        a.w, a.h, a.n, a.k, a.mip = img_w, img_h, n, k, int(cfg.render_mip)
        for i in range(3):
            a.background[i] = float(background[i])
            a.composite_bg[i] = float(background[i])
        a.local_views = local
        cams = (_lib.BgCamera * local)(*[_lib.camera_struct(build_uniforms(b.camera, img_w, img_h)) for b in batches])
        ptrs = (C.c_void_p * local)(*[g.data_ptr() for g in gts])
        a.cams, a.gt_packed = cams, ptrs
        a.transforms, a.sh, a.raw_opac = splats.transforms.data_ptr(), splats.sh_coeffs.data_ptr(), splats.raw_opacities.data_ptr()
        a.m_t, a.v_t, a.m_sh, a.v_sh, a.m_o, a.v_o = (st[x].data_ptr() for x in ("m_t", "v_t", "m_sh", "v_sh", "m_o", "v_o"))
        a.refine_norm, a.vis_weight, a.max_screen = (st[x].data_ptr() for x in ("refine_norm", "vis_weight", "max_screen"))
        a.min_scale = splats.min_scale.data_ptr() if splats.min_scale is not None else None
        a.l1_weight, a.ssim_weight = (1.0 - cfg.ssim_weight, -cfg.ssim_weight) if self.ssim_enabled else (1.0, 0.0)
        do_alpha_match = b0.has_alpha and not b0.masked_alpha and cfg.match_alpha_weight > 0.0
        a.has_composite_bg = int(b0.has_alpha and any(x != 0.0 for x in background))
        a.mask, a.channels, a.alpha_weight = int(b0.masked_alpha), (4 if do_alpha_match else 3), float(cfg.match_alpha_weight)
        lr_mean = cfg.lr_mean * self.lr_mean_decay ** (self.step_count - 1) * float(median_scale)
        a.lr_mean, a.lr_rotation, a.lr_scale = float(np.float32(lr_mean)), cfg.lr_rotation, cfg.lr_scale
        a.lr_coeffs_dc, a.lr_coeffs_sh_scale, a.lr_opac = cfg.lr_coeffs_dc, cfg.lr_coeffs_sh_scale, cfg.lr_opac
        a.noise_scale = float(np.float32(lr_mean) * np.float32(cfg.mean_noise_weight))
        a.median_scale, a.seed, a.step, a.chunks = float(median_scale), int(cfg.seed), self.step_count, int(chunks)
        a.workspace, a.workspace_bytes = self._views_ws.data_ptr(), need
        a.loss_out = self._views_loss.data_ptr()
        comm = self._dp_comm.handle if multi else None
        _lib.check(lib.bg_train_step_views(self.ctx.handle, comm, _stream_ptr(dev), C.byref(a)), "bg_train_step_views")
        self._views_keepalive = (gts, cams, ptrs)
        return TrainStepStats(num_visible_event=None, lr_mean=lr_mean, loss=self._views_loss[0])

    def _apply_updates(self, splats, v_t, v_sh, v_o, v_r, visible, max_radius, median_scale) -> float:
        """Adam on the three parameter tensors, refine statistics, mean noise (train.rs:300-416): ONE pass over the
        Gaussians (bg_train_update); the noise is the counter-based draw keyed by (seed, step), identical on every
        data-parallel rank and in bg_train_step."""
        cfg, st, dev = self.config, self._state, self.ctx.device
        lr_mean = cfg.lr_mean * self.lr_mean_decay ** (self.step_count - 1) * float(median_scale)
        n, k = splats.num_splats(), splats.sh_coeffs.shape[1]
        a = _lib.BgTrainUpdateArgs()
        a.n, a.k = n, k
        a.transforms, a.sh, a.raw_opac = splats.transforms.data_ptr(), splats.sh_coeffs.data_ptr(), splats.raw_opacities.data_ptr()
        a.m_t, a.v_t, a.m_sh, a.v_sh, a.m_o, a.v_o = (st[x].data_ptr() for x in ("m_t", "v_t", "m_sh", "v_sh", "m_o", "v_o"))
        a.refine_norm, a.vis_weight, a.max_screen = (st[x].data_ptr() for x in ("refine_norm", "vis_weight", "max_screen"))
        a.v_transforms, a.v_sh_grad, a.v_raw_opac = v_t.data_ptr(), v_sh.data_ptr(), v_o.data_ptr()
        a.v_refine, a.visible, a.max_radius = v_r.data_ptr(), visible.data_ptr(), max_radius.data_ptr()
        a.lr_mean, a.lr_rotation, a.lr_scale = float(np.float32(lr_mean)), cfg.lr_rotation, cfg.lr_scale
        a.lr_coeffs_dc, a.lr_coeffs_sh_scale, a.lr_opac = cfg.lr_coeffs_dc, cfg.lr_coeffs_sh_scale, cfg.lr_opac
        a.noise_scale = float(np.float32(lr_mean) * np.float32(cfg.mean_noise_weight))
        a.median_scale, a.seed, a.step = float(median_scale), int(cfg.seed), self.step_count
        _lib.check(_lib.load().bg_train_update(self.ctx.handle, _stream_ptr(dev), C.byref(a)), "bg_train_update")
        return lr_mean

    # ------------------------------------------------------------------------------------------------
    def refine(self, iteration: int, splats: Splats) -> RefineStats:
        """SplatTrainer::refine + refine_splats + prune_points (train.rs:431-893) through ONE ABI call (bg_refine):
        prune mask, row compaction, the two weighted samples without replacement, the force-split scan, the split itself
        and the opacity decay all run on the device; the only readback is the final counts.  Mutates `splats` (tensors
        are replaced: N changes) and the optimizer / refine-record state."""
        cfg = self.config
        if self._state is None:
            raise RuntimeError("Can only refine after optimizer is initialized")
        st = self._state
        dev = splats.transforms.device
        lib = _lib.load()
        # refine manipulates the canonical params: bake the current floor first (train.rs:432-437)
        if splats.min_scale is not None:
            splats.bake_min_scale(self.ctx)
        n0, k = splats.num_splats(), splats.sh_coeffs.shape[1]
        cap = max(n0, min(2 * n0, max(n0, int(cfg.max_splats))))
        z = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)
        out = dict(transforms=z(cap, 10), sh=z(cap, k, 3), raw_opac=z(cap), m_t=z(cap, 10), v_t=z(cap, 10), m_sh=z(cap, k, 3),
                   v_sh=z(cap), m_o=z(cap), v_o=z(cap))
        need = int(lib.bg_refine_workspace_bytes(n0))
        ws = torch.empty(need, dtype=torch.uint8, device=dev)
        a = _lib.BgRefineArgs()
        a.n, a.k, a.capacity = n0, k, cap
        a.transforms, a.sh, a.raw_opac = splats.transforms.data_ptr(), splats.sh_coeffs.data_ptr(), splats.raw_opacities.data_ptr()
        a.m_t, a.v_t, a.m_sh, a.v_sh, a.m_o, a.v_o = (st[x].data_ptr() for x in ("m_t", "v_t", "m_sh", "v_sh", "m_o", "v_o"))
        a.refine_norm, a.vis_weight, a.max_screen = (st[x].data_ptr() for x in ("refine_norm", "vis_weight", "max_screen"))
        a.transforms_out, a.sh_out, a.raw_opac_out = out["transforms"].data_ptr(), out["sh"].data_ptr(), out["raw_opac"].data_ptr()
        a.m_t_out, a.v_t_out, a.m_sh_out, a.v_sh_out, a.m_o_out, a.v_o_out = (out[x].data_ptr() for x in ("m_t", "v_t", "m_sh", "v_sh", "m_o", "v_o"))
        for i in range(3):
            a.bounds_center[i] = float(self.bounds.center[i])
        a.max_allowed = float(np.float32(np.max(self.bounds.extent)) * np.float32(100.0))
        a.split_at_screen_size, a.growth_grad_threshold = float(cfg.split_at_screen_size), float(cfg.growth_grad_threshold)
        a.growth_select_fraction, a.max_splats = float(cfg.growth_select_fraction), int(cfg.max_splats)
        a.growth_enabled = int(iteration < cfg.growth_stop_iter)
        train_t = min(max(iteration / float(cfg.total_train_iters), 0.0), 1.0)
        a.opac_decay_minus = float(cfg.opac_decay * (1.0 - train_t))
        a.seed, a.refine_index = int(cfg.seed), int(iteration)
        a.workspace, a.workspace_bytes = ws.data_ptr(), need
        rs = _lib.BgRefineStats()
        _lib.check(lib.bg_refine(self.ctx.handle, _stream_ptr(dev), C.byref(a), C.byref(rs)), "bg_refine")
        n_new = int(rs.total_splats)
        splats.transforms, splats.sh_coeffs, splats.raw_opacities = out["transforms"][:n_new], out["sh"][:n_new], out["raw_opac"][:n_new]
        for key in ("m_t", "v_t", "m_sh", "v_sh", "m_o", "v_o"):
            st[key] = out[key][:n_new]
        # bounds, refine record restart (train.rs:637-640, 442-445)
        self.bounds = bounds_from_pos_device(self.ctx, BOUND_PERCENTILE, splats.transforms)
        for key in ("refine_norm", "vis_weight", "max_screen"):
            st[key] = torch.zeros(n_new, dtype=torch.float32, device=dev)
        # fresh 3D-filter floor against the new positions / count (train.rs:641-647)
        progress = iteration / float(max(cfg.total_train_iters, 1))
        if progress < MIN_SCALE_FREEZE_FRAC and self.view_cams is not None:
            splats.min_scale = compute_min_scale(self.ctx, splats.transforms, self.view_cams, MIN_SCALE_FACTOR)
        return RefineStats(num_added=int(rs.num_added), num_split_oversized=int(rs.num_split_oversized),
                           num_split_high_grad=int(rs.num_split_high_grad), num_pruned=int(rs.num_pruned),
                           num_pruned_non_finite=int(rs.num_pruned_non_finite), total_splats=n_new)
