"""Host-side mirror of the reference's render operators over the C ABI.

  render_splats / RenderOutput  <- SplatOps::render, RenderOutput, RenderAux
                                   (brush-render/src/lib.rs:54-77, render_aux.rs:16-81)
  rasterize_bwd / project_bwd   <- SplatBwdOps (brush-render/src/bwd/burn_glue.rs:62-92)
  RenderFunction                <- RenderBackwards (bwd/burn_glue.rs:121-182): autograd glue
  render_splats(render_depth=True), rasterize_bwd_depth, project_bwd(v_z=...), RenderDepthFunction,
  expected_depth                <- differentiable per-pixel depth (DESIGN.md section 4.6; no reference operator)

PyTorch supplies device memory and the current stream only; all compute goes through
libbrush_b200.so (brush_b200/_lib.py).  No CPU path exists.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import PASS_BACKWARD, PASS_BACKWARD_SMOOTH, PASS_FORWARD, PROJECTED_STRIDE, VCOMBINED_STRIDE
from .camera import Camera, ProjectUniforms, build_uniforms


class _DevView:
    """Zero-copy view of a raw device pointer through the CUDA array interface."""

    def __init__(self, ptr: int, shape, typestr: str):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False), "version": 2}


def _view(ptr, shape, typestr, device):
    n = 1
    for s in shape:
        n *= s
    if n == 0 or not ptr:
        dt = {"<f4": torch.float32, "<u4": torch.int32, "<i4": torch.int32}[typestr]
        return torch.empty(tuple(shape), dtype=dt, device=device)
    t = torch.as_tensor(_DevView(ptr, shape, "<i4" if typestr == "<u4" else typestr), device=device)
    return t


def _stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _f32c(t: torch.Tensor, name: str) -> torch.Tensor:
    if t.dtype != torch.float32 or not t.is_cuda:
        raise TypeError(f"{name} must be a float32 CUDA tensor")
    return t.contiguous()


class RenderContext:
    """Owns a BgContext (scratch arena).  One per logical task, as in the reference's threading contract."""

    def __init__(self, max_splats: int, max_w: int, max_h: int, max_intersections: int = 0, device: int = 0):
        lib = _lib.load()
        self.device = torch.device("cuda", device)
        self._h = C.c_void_p()
        _lib.check(lib.bg_ctx_create(device, max_splats, max_w, max_h, max_intersections, C.byref(self._h)), "bg_ctx_create")
        self.max_splats, self.max_w, self.max_h = max_splats, max_w, max_h

    @property
    def handle(self):
        return self._h

    def arena_bytes(self) -> int:
        return int(_lib.load().bg_ctx_arena_bytes(self._h))

    def close(self):
        if self._h:
            _lib.load().bg_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


@dataclass
class RenderOutput:
    """render_aux.rs:16-81.  `state` pointers live in the context arena until the next render on it."""

    out_img: torch.Tensor            # [h,w,4] f32, or [h,w] int32 (packed rgba8) for PASS_FORWARD
    visible: Optional[torch.Tensor]  # [n] f32 (None for PASS_FORWARD)
    max_radius: torch.Tensor         # [n] f32
    state: _lib.BgRenderState
    cam: _lib.BgCamera
    uniforms: ProjectUniforms
    background: Tuple[float, float, float]
    ctx: RenderContext
    _event: torch.cuda.Event = field(default=None, repr=False)
    depth: Optional[torch.Tensor] = None  # [h,w] f32 accumulated depth sum_i vis_i z_i (render_depth=True only)

    def _counters(self):
        if self._event is not None:
            self._event.synchronize()
        else:  # rendered while a CUDA graph was being captured: the values belong to the latest replay
            torch.cuda.synchronize(self.ctx.device)
        return self.state.counters_host

    @property
    def num_visible(self) -> int:
        return int(self._counters()[0])

    @property
    def num_intersections(self) -> int:
        return int(self._counters()[1])

    @property
    def intersection_overflow(self) -> int:
        return int(self._counters()[2])

    def validate_counts(self):
        """render_aux.rs:30-45"""
        nv, ni = self.num_visible, self.num_intersections
        assert nv <= self.state.n, f"num_visible ({nv}) > total_splats ({self.state.n})"
        assert ni <= nv * self.state.tiles_x * self.state.tiles_y

    # zero-copy views of the saved state (valid until the next render on the same context)
    def projected(self) -> torch.Tensor:
        return _view(self.state.projected, (self.num_visible, PROJECTED_STRIDE), "<f4", self.ctx.device)

    def global_from_compact_gid(self) -> torch.Tensor:
        return _view(self.state.global_from_compact_gid, (self.num_visible,), "<u4", self.ctx.device)

    def depths(self) -> torch.Tensor:
        return _view(self.state.depths, (self.num_visible,), "<f4", self.ctx.device)

    def compact_gid_from_isect(self) -> torch.Tensor:
        return _view(self.state.compact_gid_from_isect, (self.num_intersections,), "<u4", self.ctx.device)

    def tile_id_from_isect(self) -> torch.Tensor:
        return _view(self.state.tile_id_from_isect, (self.num_intersections,), "<u4", self.ctx.device)

    def tile_offsets(self) -> torch.Tensor:
        return _view(self.state.tile_offsets, (self.state.tiles_y, self.state.tiles_x, 2), "<u4", self.ctx.device)


def render_splats(ctx: RenderContext, camera, img_size, transforms: torch.Tensor, sh_coeffs: torch.Tensor,
                  raw_opacities: torch.Tensor, mip: bool = False, background=(0.0, 0.0, 0.0),
                  rpass: int = PASS_BACKWARD, render_depth: bool = False) -> RenderOutput:
    """<MainBackendBase as SplatOps>::render (render.rs:37-315).  img_size = (w, h).
    `camera` is a brush_b200.camera.Camera or prebuilt ProjectUniforms.
    render_depth: also return `depth`, the [h,w] accumulated depth sum_i alpha_i T_i z_i (z_i = camera-space z of the
    splat mean; no background term).  Needs an f32 pass (PASS_BACKWARD or PASS_BACKWARD_SMOOTH); expected_depth()
    turns it into the expected depth."""
    lib = _lib.load()
    w, h = int(img_size[0]), int(img_size[1])
    transforms = _f32c(transforms, "transforms")
    sh_coeffs = _f32c(sh_coeffs, "sh_coeffs")
    raw_opacities = _f32c(raw_opacities, "raw_opacities")
    # DimCheck (render.rs:61-64)
    n = transforms.shape[0]
    if transforms.dim() != 2 or transforms.shape[1] != 10:
        raise ValueError("transforms must be [D, 10]")
    if sh_coeffs.dim() != 3 or sh_coeffs.shape[0] != n or sh_coeffs.shape[2] != 3:
        raise ValueError("sh_coeffs must be [D, C, 3]")
    if raw_opacities.dim() != 1 or raw_opacities.shape[0] != n:
        raise ValueError("raw_opacities must be [D]")
    k = sh_coeffs.shape[1]
    uniforms = camera if isinstance(camera, ProjectUniforms) else build_uniforms(camera, w, h)
    cam = _lib.camera_struct(uniforms)
    dev = ctx.device
    bwd_info = rpass != PASS_FORWARD
    out_img = torch.empty((h, w, 4), dtype=torch.float32, device=dev) if bwd_info else torch.empty((h, w), dtype=torch.int32, device=dev)
    visible = torch.empty((n,), dtype=torch.float32, device=dev) if bwd_info else None
    max_radius = torch.empty((n,), dtype=torch.float32, device=dev)
    bg = (C.c_float * 3)(*[float(b) for b in background])
    st = _lib.BgRenderState()
    # the depth entry point takes the depth output right behind out_img
    depth = torch.empty((h, w), dtype=torch.float32, device=dev) if render_depth else None
    fn = "bg_render_forward_depth" if render_depth else "bg_render_forward"
    _lib.check(
        getattr(lib, fn)(ctx.handle, _stream_ptr(dev), C.byref(cam), w, h, n, k, transforms.data_ptr(), sh_coeffs.data_ptr(),
                         raw_opacities.data_ptr(), int(bool(mip)), bg, int(rpass), out_img.data_ptr(),
                         *((depth.data_ptr(),) if render_depth else ()), visible.data_ptr() if visible is not None else None,
                         max_radius.data_ptr(), C.byref(st)),
        fn)
    ev = None
    if not torch.cuda.is_current_stream_capturing():
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(dev))
    return RenderOutput(out_img=out_img, visible=visible, max_radius=max_radius, state=st, cam=cam, uniforms=uniforms,
                        background=tuple(float(b) for b in background), ctx=ctx, _event=ev, depth=depth)


def rasterize_bwd(out: RenderOutput, v_output: torch.Tensor, smooth_cutoff: Optional[bool] = None) -> torch.Tensor:
    """SplatBwdOps::rasterize_bwd (bwd/render_bwd.rs:22-99).  Returns v_combined [n, 10]
    (rows >= num_visible; rows past num_visible are zero)."""
    lib = _lib.load()
    v_output = _f32c(v_output, "v_output")
    st = out.state
    if tuple(v_output.shape) != (st.h, st.w, 4):
        raise ValueError("v_output must be [h, w, 4]")
    if smooth_cutoff is None:
        smooth_cutoff = st.pass_ == PASS_BACKWARD_SMOOTH
    rows = max(int(st.n), 1)
    v_combined = torch.empty((rows, VCOMBINED_STRIDE), dtype=torch.float32, device=out.ctx.device)
    bg = (C.c_float * 3)(*out.background)
    _lib.check(
        lib.bg_rasterize_backward(out.ctx.handle, _stream_ptr(out.ctx.device), C.byref(st), out.out_img.data_ptr(),
                                  v_output.data_ptr(), bg, int(bool(smooth_cutoff)), v_combined.data_ptr(), rows),
        "bg_rasterize_backward")
    return v_combined


def rasterize_bwd_depth(out: RenderOutput, v_output: torch.Tensor, v_depth: torch.Tensor):
    """Adjoint of a render_depth=True render: rasterize_bwd with the upstream gradient v_depth [h,w] of out.depth.
    Returns (v_combined [n,10], v_z [n]); v_z is indexed by compact id like v_combined and feeds project_bwd(v_z=...).
    `out` must still be its context's last render."""
    lib = _lib.load()
    v_output = _f32c(v_output, "v_output")
    v_depth = _f32c(v_depth, "v_depth")
    st = out.state
    if tuple(v_output.shape) != (st.h, st.w, 4):
        raise ValueError("v_output must be [h, w, 4]")
    if tuple(v_depth.shape) != (st.h, st.w):
        raise ValueError("v_depth must be [h, w]")
    if out.depth is None:
        raise ValueError("rasterize_bwd_depth needs a render_splats(..., render_depth=True) output")
    rows = max(int(st.n), 1)
    v_combined = torch.empty((rows, VCOMBINED_STRIDE), dtype=torch.float32, device=out.ctx.device)
    v_z = torch.empty((rows,), dtype=torch.float32, device=out.ctx.device)
    bg = (C.c_float * 3)(*out.background)
    _lib.check(
        lib.bg_rasterize_backward_depth(out.ctx.handle, _stream_ptr(out.ctx.device), C.byref(st), out.out_img.data_ptr(),
                                        out.depth.data_ptr(), v_output.data_ptr(), v_depth.data_ptr(), bg,
                                        int(st.pass_ == PASS_BACKWARD_SMOOTH), v_combined.data_ptr(), rows,
                                        v_z.data_ptr()),
        "bg_rasterize_backward_depth")
    return v_combined, v_z


def blend_stats(out: RenderOutput, v_output: torch.Tensor) -> dict:
    """Measurement aid (bg_debug_blend_stats): counters of the blend loop for `out` (a PASS_BACKWARD render that is
    still this context's last forward).  Synchronises the stream."""
    lib = _lib.load()
    v_output = _f32c(v_output, "v_output")
    st = out.state
    scratch = torch.empty((max(int(st.n), 1), VCOMBINED_STRIDE), dtype=torch.float32, device=out.ctx.device)
    scratch.zero_()
    res = (C.c_ulonglong * 4)()
    bg = (C.c_float * 3)(*out.background)
    _lib.check(lib.bg_debug_blend_stats(out.ctx.handle, _stream_ptr(out.ctx.device), C.byref(st), out.out_img.data_ptr(),
                                        v_output.data_ptr(), bg, scratch.data_ptr(), res), "bg_debug_blend_stats")
    it, live, stop, isect = (int(x) for x in res)
    return {"tile_list_entries": isect, "warp_splat_iterations": it, "pairs_evaluated": it * 64, "pairs_live": live,
            "pairs_stopping": stop, "lane_utilisation": (live / (it * 64)) if it else 0.0}


def project_bwd(out: RenderOutput, transforms, sh_coeffs, raw_opacities, v_combined, outputs=None, v_z=None):
    """SplatBwdOps::project_bwd (bwd/render_bwd.rs:102-171) -> (v_transforms, v_coeffs, v_raw_opac, v_refine_weight).
    `outputs`: optional preallocated (v_t [n,10], v_sh [n,k,3], v_o [n], v_r [n]) -- e.g. views of one flat
    buffer so that data-parallel training can all-reduce all gradients with a single collective.
    `v_z`: the depth gradient of rasterize_bwd_depth; its chain to the means is added to v_transforms[:, 0:3]."""
    lib = _lib.load()
    transforms = _f32c(transforms, "transforms")
    sh_coeffs = _f32c(sh_coeffs, "sh_coeffs")
    raw_opacities = _f32c(raw_opacities, "raw_opacities")
    v_combined = _f32c(v_combined, "v_combined")
    dev = out.ctx.device
    n, k = int(out.state.n), int(out.state.k)
    if outputs is not None:
        v_t, v_sh, v_o, v_r = outputs
        for t_, shp in ((v_t, (n, 10)), (v_sh, (n, k, 3)), (v_o, (n,)), (v_r, (n,))):
            if tuple(t_.shape) != shp or t_.dtype != torch.float32 or not t_.is_contiguous():
                raise ValueError("project_bwd outputs must be contiguous float32 tensors of the documented shapes")
    else:
        v_t = torch.empty((n, 10), dtype=torch.float32, device=dev)
        v_sh = torch.empty((n, k, 3), dtype=torch.float32, device=dev)
        v_o = torch.empty((n,), dtype=torch.float32, device=dev)
        v_r = torch.empty((n,), dtype=torch.float32, device=dev)
    if v_z is not None:
        v_z = _f32c(v_z, "v_z")
        if v_z.dim() != 1 or v_z.shape[0] < max(n, 1):
            raise ValueError("v_z must be [n] (as returned by rasterize_bwd_depth)")
    # the depth entry point takes v_z right behind v_combined
    fn = "bg_project_backward" if v_z is None else "bg_project_backward_depth"
    _lib.check(
        getattr(lib, fn)(out.ctx.handle, _stream_ptr(dev), C.byref(out.cam), C.byref(out.state), transforms.data_ptr(),
                         sh_coeffs.data_ptr(), raw_opacities.data_ptr(), v_combined.data_ptr(),
                         *(() if v_z is None else (v_z.data_ptr(),)), v_t.data_ptr(), v_sh.data_ptr(), v_o.data_ptr(),
                         v_r.data_ptr()),
        fn)
    return v_t, v_sh, v_o, v_r


def project_bwd_factored(out: RenderOutput, transforms, sh_coeffs, raw_opacities, v_combined, outputs=None):
    """bg_project_backward_factored: project_bwd with the view's SH gradient left in its rank-one form.
    Returns (v_transforms [n,10], v_color [n,3], v_raw_opac [n], v_refine_weight [n]); the dense
    v_sh = Y(dir) x v_color is rebuilt by sh_grad_from_views after the views' v_color rows are gathered."""
    lib = _lib.load()
    transforms = _f32c(transforms, "transforms")
    sh_coeffs = _f32c(sh_coeffs, "sh_coeffs")
    raw_opacities = _f32c(raw_opacities, "raw_opacities")
    v_combined = _f32c(v_combined, "v_combined")
    dev = out.ctx.device
    n = int(out.state.n)
    if outputs is not None:
        v_t, v_c, v_o, v_r = outputs
        for t_, shp in ((v_t, (n, 10)), (v_c, (n, 3)), (v_o, (n,)), (v_r, (n,))):
            if tuple(t_.shape) != shp or t_.dtype != torch.float32 or not t_.is_contiguous():
                raise ValueError("project_bwd_factored outputs must be contiguous float32 tensors of the documented shapes")
    else:
        v_t = torch.empty((n, 10), dtype=torch.float32, device=dev)
        v_c = torch.empty((n, 3), dtype=torch.float32, device=dev)
        v_o = torch.empty((n,), dtype=torch.float32, device=dev)
        v_r = torch.empty((n,), dtype=torch.float32, device=dev)
    _lib.check(
        lib.bg_project_backward_factored(out.ctx.handle, _stream_ptr(dev), C.byref(out.cam), C.byref(out.state),
                                         transforms.data_ptr(), sh_coeffs.data_ptr(), raw_opacities.data_ptr(),
                                         v_combined.data_ptr(), v_t.data_ptr(), v_c.data_ptr(), v_o.data_ptr(),
                                         v_r.data_ptr()),
        "bg_project_backward_factored")
    return v_t, v_c, v_o, v_r


def sh_grad_from_views(ctx: RenderContext, transforms, k: int, cam_positions, v_color_all, out_scale: float = 1.0,
                       out=None, view_stride: int = 0):
    """bg_sh_grad_from_views: v_sh [n,k,3] = out_scale * sum_v Y(dir(mean, cam_positions[v])) x v_color_all[v].
    cam_positions: sequence of `views` world-space camera positions; v_color_all: [views, n, 3], or with
    view_stride > 0 a [views, view_stride] buffer whose rows START with the view's [n,3] colours."""
    lib = _lib.load()
    transforms = _f32c(transforms, "transforms")
    v_color_all = _f32c(v_color_all, "v_color_all")
    views = int(v_color_all.shape[0])
    n = int(transforms.shape[0])
    if view_stride == 0 and (v_color_all.dim() != 3 or int(v_color_all.shape[1]) != n):
        raise ValueError("v_color_all must be [views, n, 3]")
    pos = [float(x) for p in cam_positions for x in p]
    if len(pos) != 3 * views:
        raise ValueError("cam_positions must hold one xyz per view of v_color_all")
    if out is None:
        out = torch.empty((n, k, 3), dtype=torch.float32, device=transforms.device)
    elif tuple(out.shape) != (n, k, 3) or out.dtype != torch.float32 or not out.is_contiguous():
        raise ValueError("out must be a contiguous float32 [n,k,3] tensor")
    arr = (C.c_float * len(pos))(*pos)
    _lib.check(lib.bg_sh_grad_from_views(ctx.handle, _stream_ptr(ctx.device), n, k, transforms.data_ptr(), arr, views,
                                         v_color_all.data_ptr(), int(view_stride), float(out_scale), out.data_ptr()),
               "bg_sh_grad_from_views")
    return out


class RenderFunction(torch.autograd.Function):
    """Autograd glue: forward = render, backward = rasterize_bwd + project_bwd (bwd/burn_glue.rs:121-182).
    The refine weight gradient is returned through the `refine_weight_holder` input, as in the reference."""

    @staticmethod
    def forward(fctx, transforms, sh_coeffs, raw_opacities, refine_weight_holder, ctx, camera, img_size, mip, background,
                rpass):
        out = render_splats(ctx, camera, img_size, transforms, sh_coeffs, raw_opacities, mip, background, rpass)
        fctx.out = out
        fctx.save_for_backward(transforms, sh_coeffs, raw_opacities)
        fctx.mark_non_differentiable(out.visible, out.max_radius)
        return out.out_img, out.visible, out.max_radius

    @staticmethod
    def backward(fctx, v_img, _v_vis, _v_rad):
        transforms, sh_coeffs, raw_opacities = fctx.saved_tensors
        out = fctx.out
        v_combined = rasterize_bwd(out, v_img.contiguous())
        v_t, v_sh, v_o, v_r = project_bwd(out, transforms, sh_coeffs, raw_opacities, v_combined)
        # refine_weight_holder is an [n] tensor here (torch requires matching shapes); its gradient is
        # v_refine_weight, exactly what the reference registers on its holder node.
        return v_t, v_sh, v_o, v_r, None, None, None, None, None, None


class RenderDepthFunction(torch.autograd.Function):
    """RenderFunction with the accumulated depth as a second differentiable output: forward returns
    (img, depth, visible, max_radius).  When no gradient reaches `depth`, backward is RenderFunction's."""

    @staticmethod
    def forward(fctx, transforms, sh_coeffs, raw_opacities, refine_weight_holder, ctx, camera, img_size, mip, background,
                rpass):
        out = render_splats(ctx, camera, img_size, transforms, sh_coeffs, raw_opacities, mip, background, rpass,
                            render_depth=True)
        fctx.out = out
        fctx.save_for_backward(transforms, sh_coeffs, raw_opacities)
        fctx.mark_non_differentiable(out.visible, out.max_radius)
        fctx.set_materialize_grads(False)
        return out.out_img, out.depth, out.visible, out.max_radius

    @staticmethod
    def backward(fctx, v_img, v_depth, _v_vis, _v_rad):
        transforms, sh_coeffs, raw_opacities = fctx.saved_tensors
        out = fctx.out
        if v_img is None:
            v_img = torch.zeros_like(out.out_img)
        if v_depth is None:
            v_combined, v_z = rasterize_bwd(out, v_img.contiguous()), None
        else:
            v_combined, v_z = rasterize_bwd_depth(out, v_img.contiguous(), v_depth.contiguous())
        v_t, v_sh, v_o, v_r = project_bwd(out, transforms, sh_coeffs, raw_opacities, v_combined, v_z=v_z)
        return v_t, v_sh, v_o, v_r, None, None, None, None, None, None


def expected_depth(img: torch.Tensor, depth: torch.Tensor, eps: float = 1e-10) -> torch.Tensor:
    """Expected depth D / alpha of a depth render (alpha = img[..., 3]); differentiable through both inputs.
    Pixels that nothing covers (alpha <= eps) divide by eps, giving ~0 since D is 0 there too."""
    return depth / img[..., 3].clamp_min(eps)


def radix_argsort(ctx: RenderContext, keys: torch.Tensor, values: torch.Tensor, sorting_bits: int):
    """brush_sort::radix_argsort (brush-sort/src/lib.rs:16-125).  int32/uint32-as-int32 CUDA tensors."""
    lib = _lib.load()
    if keys.shape != values.shape or keys.dim() != 1:
        raise ValueError("Input keys and values must have the same number of elements")
    if sorting_bits > 32:
        raise ValueError("Can only sort up to 32 bits")
    keys, values = keys.contiguous(), values.contiguous()
    ko, vo = torch.empty_like(keys), torch.empty_like(values)
    _lib.check(lib.bg_radix_argsort_u32(ctx.handle, _stream_ptr(ctx.device), keys.data_ptr(), values.data_ptr(),
                                        keys.shape[0], None, sorting_bits, ko.data_ptr(), vo.data_ptr()), "bg_radix_argsort_u32")
    return ko, vo


def prefix_sum(ctx: RenderContext, x: torch.Tensor) -> torch.Tensor:
    """brush_prefix_sum::prefix_sum (brush-prefix-sum/src/lib.rs:11-89): inclusive."""
    lib = _lib.load()
    x = x.contiguous()
    o = torch.empty_like(x)
    _lib.check(lib.bg_inclusive_scan_u32(ctx.handle, _stream_ptr(ctx.device), x.data_ptr(), x.shape[0], o.data_ptr()),
               "bg_inclusive_scan_u32")
    return o
