"""Training loop driver (SURVEY 8f N3): the schedule of brush-process/src/train_stream.rs:150-500 without its app plumbing
(message emitter, viewer slot, rerun).

  schedule predicates  <- train_stream.rs:318-326 (refine gating), :350-353 (eval cadence), :377-383 (export cadence)
  LOD schedule         <- train_stream.rs:221-225 (target level), :309-324 (phase-local refine gating), :351-352 (eval in
                          level 0 only), :381-393 (export cadence and names), :272 (image scale)
  train_loop           <- train_stream.rs:176-497: loader -> step -> refine -> eval -> export; at each LOD level boundary
                          (:227-291) export -> score -> decimate -> fresh trainer -> loader on downscaled images
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np


@dataclass
class ProcessConfig:                     # brush-process/src/config.rs (the fields the loop reads)
    eval_every: int = 1000
    export_every: int = 5000
    export_path: str = "."
    export_name: str = "export_{iter}.ply"
    start_iter: int = 0
    seed: int = 42
    eval_save_to_disk: bool = False     # the rendered eval images go to <export_path>/eval_<iter>/<image name>.png


def should_refine(it: int, refine_every: int, total_iters: int) -> bool:
    """train_stream.rs:318-326, for the step that just ran with 0-based index `it`."""
    progress = min(max(it / float(max(total_iters, 1)), 0.0), 1.0)
    return it > 0 and it % refine_every == 0 and progress <= 0.95


def should_eval(done: int, eval_every: int, total_iters: int) -> bool:
    """train_stream.rs:350-353, `done` = number of finished iterations."""
    return done % eval_every == 0 or done == total_iters


def should_export(done: int, export_every: int, total_iters: int) -> bool:
    """train_stream.rs:377-383 (no LOD phases)."""
    return done % export_every == 0 or done == total_iters


def lod_level(it: int, total_train_iters: int, lod_levels: int, lod_refine_steps: int) -> int:
    """train_stream.rs:221-225: the level that the step with 0-based index `it` trains (0 = the main run)."""
    if lod_levels == 0 or it < total_train_iters:
        return 0
    return min((it - total_train_iters) // lod_refine_steps + 1, lod_levels)


def lod_phase(it: int, level: int, total_train_iters: int, lod_refine_steps: int) -> Tuple[int, int]:
    """train_stream.rs:309-318: (phase_iter, phase_total) of step `it` in `level`."""
    if level == 0:
        return it, total_train_iters
    return (it - total_train_iters) % lod_refine_steps, lod_refine_steps


def should_refine_lod(it: int, level: int, refine_every: int, total_train_iters: int, lod_refine_steps: int) -> bool:
    """train_stream.rs:319-324: refine gating on the phase-local iteration and progress (refine itself still receives
    the global iteration)."""
    phase_iter, phase_total = lod_phase(it, level, total_train_iters, lod_refine_steps)
    return should_refine(phase_iter, refine_every, phase_total)


def should_eval_lod(done: int, level: int, eval_every: int, total_train_iters: int) -> bool:
    """train_stream.rs:351-352: evaluations belong to level 0."""
    return level == 0 and should_eval(done, eval_every, total_train_iters)


def should_export_lod(done: int, level: int, export_every: int, total_iters: int, lod_levels: int) -> bool:
    """train_stream.rs:381-385: level 0 at export_every multiples (and at the last step when there are no LOD levels),
    a LOD level at the last step only.  total_iters = TrainConfig.total_iters()."""
    if level == 0:
        return done % export_every == 0 or (done == total_iters and lod_levels == 0)
    return done == total_iters


def lod_export_name(export_name: str, level: int, iteration: int, lod_refine_steps: int) -> str:
    """train_stream.rs:233-241, 386-393: level 0 writes export_name with {iter} = iteration; level n inserts "_lod{n}"
    before ".ply" and puts lod_refine_steps in {iter}."""
    if level == 0:
        return export_name.replace("{iter}", str(iteration))
    return export_name.replace(".ply", f"_lod{level}.ply").replace("{iter}", str(lod_refine_steps))


def lod_image_scale(level: int, lod_image_scale_pct: int) -> float:
    """train_stream.rs:272: (lod_image_scale / 100).powi(level) in f32 (powi by squaring, as compiler-rt's __powisf2)."""
    r, a, b = np.float32(1.0), np.float32(lod_image_scale_pct) / np.float32(100.0), int(level)
    while True:
        if b & 1:
            r = np.float32(r * a)
        b >>= 1
        if b == 0:
            return float(r)
        a = np.float32(a * a)


def train_loop(ctx, splats, train_views: Sequence, eval_views: Sequence, config, process: Optional[ProcessConfig] = None,
               on_step: Optional[Callable] = None, alpha_mode: str = "masked") -> List[dict]:
    """Runs config.total_iters() steps (the main run, then config.lod_levels LOD levels); returns the evaluation records.
    `splats`: train.Splats on ctx's device, updated in place (refine and decimation replace its tensors); views:
    dataset.SceneView lists."""
    import torch
    from . import ply
    from .dataset import SceneLoader
    from .eval import eval_stats
    from .lod import compute_pup_scores, decimate_to_count, lod_target_count
    from .train import BOUND_PERCENTILE, SplatTrainer, bounds_from_pos_device
    process = process or ProcessConfig()
    from PIL import Image
    loader = SceneLoader(train_views, alpha_mode, seed=process.seed)
    trainer = SplatTrainer(config, ctx, bounds_from_pos_device(ctx, BOUND_PERCENTILE, splats.transforms))
    # refine grows the model up to config.max_splats: the context must have been created for it (the reference sizes
    # its buffers per render; here capacity is fixed at bg_ctx_create)
    cap = min(int(config.max_splats), max(int(ctx.max_splats), 0))
    if ctx.max_splats < min(config.max_splats, splats.num_splats()):
        raise ValueError(f"render context holds {ctx.max_splats} splats, the model already has {splats.num_splats()}")
    if cap < config.max_splats:
        import dataclasses
        config = dataclasses.replace(config, max_splats=cap)     # never grow past what the context can render
        trainer.config = config
    view_cams = []
    for v in train_views:                                   # (position, focal in px at native resolution): the 3D filter
        with Image.open(v.image_path) as im:                # header only: no decode
            iw, ih = im.size
        view_cams.append((v.camera.position, float(v.camera.focal(iw, ih)[0])))
    trainer.set_view_cams(view_cams)
    total = config.total_train_iters
    total_all = config.total_iters()
    steps = config.lod_refine_steps
    level = 0
    evals: List[dict] = []
    last_out = None

    def check_overflow():
        # a view whose tile list exceeds the arena is rendered with the overflowing intersections dropped: never silently
        if last_out is not None and last_out.intersection_overflow:
            raise RuntimeError("intersection arena overflow: create the RenderContext with a larger max_intersections "
                               f"(num_intersections {last_out.num_intersections})")

    def export(name: str):
        t_fold, o_fold = splats.folded(ctx)                # export.rs:183: the floor is folded into a COPY, never stored
        data = ply.splat_to_ply(t_fold.cpu().numpy(), splats.sh_coeffs.cpu().numpy(), o_fold.cpu().numpy(),
                                render_mip=config.render_mip)
        os.makedirs(process.export_path, exist_ok=True)
        with open(os.path.join(process.export_path, name), "wb") as f:
            f.write(data)

    for it in range(process.start_iter, total_all):
        target = lod_level(it, total, config.lod_levels, steps)
        if target > level:                                  # train_stream.rs:227-291
            check_overflow()
            export(lod_export_name(process.export_name, level, it, steps))
            keep = lod_target_count(splats.num_splats(), config.lod_decimation_keep)
            scores = compute_pup_scores(ctx, splats, train_views, alpha_mode, mip=config.render_mip)
            kept = decimate_to_count(ctx, splats, scores, keep)
            splats.transforms, splats.sh_coeffs, splats.raw_opacities, splats.min_scale = (
                kept.transforms, kept.sh_coeffs, kept.raw_opacities, kept.min_scale)
            level = target
            trainer = SplatTrainer(config, ctx, bounds_from_pos_device(ctx, BOUND_PERCENTILE, splats.transforms))
            trainer.set_view_cams(view_cams)
            if config.lod_image_scale < 100:               # a rebuild at 100 % would only drop the warm batch cache
                loader.close()
                loader = SceneLoader(train_views, alpha_mode, seed=process.seed,
                                     image_scale=lod_image_scale(level, config.lod_image_scale))
            last_out = None
        stats = trainer.step(loader.next_batch(), splats)
        if stats.num_visible_event is not None:
            last_out = stats.num_visible_event
        refine = None
        if should_refine_lod(it, level, config.refine_every, total, steps):
            check_overflow()                                # refine synchronises anyway
            refine = trainer.refine(it, splats)
        done = it + 1
        if on_step is not None:
            on_step(done, stats, refine)
        if eval_views and should_eval_lod(done, level, process.eval_every, total):
            check_overflow()
            psnr, ssim, dm = [], [], []
            for v in eval_views:
                gt = v.load_image()                        # view.image.load(): a mask file, if any, is the alpha channel
                gt_depth = v.load_depth() if v.depth_path is not None else None
                s = eval_stats(ctx, splats, v.camera, gt, alpha_mode, render_mip=config.render_mip, gt_depth=gt_depth)
                psnr.append(float(s.psnr)); ssim.append(float(s.ssim))
                if gt_depth is not None:
                    dm.append((float(s.depth_abs_rel), float(s.depth_rmse), float(s.depth_coverage)))
                if process.eval_save_to_disk:              # train_stream.rs:543-550
                    s.save_to_disk(os.path.join(process.export_path, f"eval_{done}", f"{v.img_name()}.png"))
            rec = {"iter": done, "psnr": float(np.mean(psnr)), "ssim": float(np.mean(ssim)), "splats": splats.num_splats()}
            if dm:                                         # only when the eval views carry depth (means over those views)
                for key, col in zip(("depth_abs_rel", "depth_rmse", "depth_coverage"), np.array(dm, np.float64).T):
                    rec[key] = float(np.mean(col))
            evals.append(rec)
        if should_export_lod(done, level, process.export_every, total_all, config.lod_levels):
            export(lod_export_name(process.export_name, level, done, steps))
    torch.cuda.synchronize(ctx.device)
    check_overflow()
    loader.close()
    return evals
