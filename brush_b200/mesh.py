"""Mesh export over the C ABI (DESIGN.md section 4.9; no reference operator): render depth and colour from the training
views, fuse them into a truncated signed distance field on the device, and extract the zero level set as a coloured
triangle mesh by marching tetrahedra.

  TsdfVolume.integrate   <- bg_tsdf_integrate: one view (a render_splats(..., render_depth=True, background=0) output)
  TsdfVolume.extract     <- bg_mesh_count (one readback) + bg_mesh_emit: TriangleMesh in the deterministic order of 4.9
  splats_to_mesh         <- the whole export: bounds, one render and one integration per view, the extraction
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .render import PASS_BACKWARD, RenderContext, RenderOutput, _stream_ptr, render_splats

MESH_BOUND_PERCENTILE = 0.98   # central per-axis box of the means ...
MESH_BOUND_MARGIN = 0.1        # ... grown by this fraction of its extent on every side
MAX_GRID_POINTS = (1 << 31) - 1


class TriangleMesh(NamedTuple):
    vertices: np.ndarray   # f32 [M, 3]
    colors: np.ndarray     # u8 [M, 3]
    faces: np.ndarray      # i32 [F, 3]; normals point toward free space (T >= 0)

    def to_ply(self) -> bytes:
        from .ply import mesh_to_ply
        return mesh_to_ply(self.vertices, self.colors, self.faces)


def grid_dims(lo, hi, resolution: int):
    """(h, dims): `resolution` points along the longest axis of [lo, hi], the same spacing along the others (at least 2
    points each)."""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    ext = hi - lo
    if not (np.isfinite(ext).all() and (ext > 0).all()) or resolution < 2:
        raise ValueError(f"mesh bounds must be a non-empty box and resolution >= 2 (lo={lo}, hi={hi}, resolution={resolution})")
    h = float(ext.max()) / (resolution - 1)
    dims = tuple(max(2, int(np.ceil(e / h - 1e-9)) + 1) for e in ext)
    return float(np.float32(h)), dims


class TsdfVolume:
    """A dense TSDF grid on ctx's device over [lo, hi]: `resolution` points along the longest axis, truncation
    trunc_voxels * h.  20 bytes per point, zeroed (unobserved) at creation."""

    def __init__(self, ctx: RenderContext, lo, hi, resolution: int = 512, trunc_voxels: float = 4.0):
        self.ctx = ctx
        self.h, self.dims = grid_dims(lo, hi, int(resolution))
        npts = self.dims[0] * self.dims[1] * self.dims[2]
        if npts > MAX_GRID_POINTS:
            raise ValueError(f"TSDF grid {self.dims} has {npts} points; at most 2^31 - 1 are supported")
        need = npts * 20 + _lib.load().bg_mesh_workspace_bytes(*self.dims)
        free, _ = torch.cuda.mem_get_info(ctx.device)
        if need > free:
            raise MemoryError(f"TSDF grid {self.dims} needs {need / 2**30:.2f} GiB with its extraction workspace; "
                              f"{free / 2**30:.2f} GiB are free on {ctx.device}: lower the resolution")
        self.origin = tuple(float(np.float32(x)) for x in np.asarray(lo, np.float64))
        self.trunc = float(np.float32(float(trunc_voxels) * self.h))
        dx, dy, dz = self.dims
        dev = ctx.device
        self.tsdf = torch.zeros((dz, dy, dx), dtype=torch.float32, device=dev)
        self.weight = torch.zeros((dz, dy, dx), dtype=torch.float32, device=dev)
        self.rgb = torch.zeros((dz, dy, dx, 3), dtype=torch.float32, device=dev)

    def grid_struct(self) -> _lib.BgTsdfGrid:
        g = _lib.BgTsdfGrid()
        for a in range(3):
            g.origin[a] = self.origin[a]
            g.dims[a] = self.dims[a]
        g.h, g.trunc = self.h, self.trunc
        g.tsdf, g.weight, g.rgb = self.tsdf.data_ptr(), self.weight.data_ptr(), self.rgb.data_ptr()
        return g

    def integrate(self, out: RenderOutput, camera=None, alpha_min: float = 0.5) -> None:
        """Fuses one render: `out` from render_splats(..., render_depth=True, background=(0, 0, 0)).  `camera` defaults to
        the render's own uniforms."""
        if out.depth is None or out.out_img.dim() != 3:
            raise ValueError("TsdfVolume.integrate needs a render_splats(..., render_depth=True) output")
        if any(b != 0.0 for b in out.background):
            raise ValueError("TsdfVolume.integrate needs a render on a black background (the colour is un-premultiplied)")
        cam = out.cam if camera is None else _lib.camera_struct(camera)
        h, w = int(out.depth.shape[0]), int(out.depth.shape[1])
        g = self.grid_struct()
        _lib.check(_lib.load().bg_tsdf_integrate(self.ctx.handle, _stream_ptr(self.ctx.device), C.byref(g), C.byref(cam), w, h,
                                                 out.out_img.data_ptr(), out.depth.data_ptr(), float(alpha_min)),
                   "bg_tsdf_integrate")

    def extract(self) -> TriangleMesh:
        lib = _lib.load()
        dev = self.ctx.device
        g = self.grid_struct()
        need = int(lib.bg_mesh_workspace_bytes(*self.dims))
        ws = torch.empty(need, dtype=torch.uint8, device=dev)
        nv, nt = C.c_uint32(), C.c_uint32()
        s = _stream_ptr(dev)
        _lib.check(lib.bg_mesh_count(self.ctx.handle, s, C.byref(g), ws.data_ptr(), need, C.byref(nv), C.byref(nt)), "bg_mesh_count")
        m, f = int(nv.value), int(nt.value)
        verts = torch.empty((m, 3), dtype=torch.float32, device=dev)
        cols = torch.empty((m, 3), dtype=torch.uint8, device=dev)
        faces = torch.empty((f, 3), dtype=torch.int32, device=dev)
        _lib.check(lib.bg_mesh_emit(self.ctx.handle, s, C.byref(g), ws.data_ptr(), need, m, f,
                                    verts.data_ptr() if m else None, cols.data_ptr() if m else None,
                                    faces.data_ptr() if f else None), "bg_mesh_emit")
        return TriangleMesh(verts.cpu().numpy(), cols.cpu().numpy(), faces.cpu().numpy())


def mesh_bounds(ctx: RenderContext, transforms: torch.Tensor):
    """Default bounds: the central 98 % per-axis box of the means, grown by 10 % of its extent on every side."""
    from .train import bounds_from_pos_device
    b = bounds_from_pos_device(ctx, MESH_BOUND_PERCENTILE, transforms)
    c, e = np.asarray(b.center, np.float64), np.asarray(b.extent, np.float64)
    ext = np.maximum(2.0 * e, 1e-6)
    return c - e - MESH_BOUND_MARGIN * ext, c + e + MESH_BOUND_MARGIN * ext


def splats_to_mesh(ctx: RenderContext, splats, views: Sequence, *, resolution: int = 512, bounds=None,
                   trunc_voxels: float = 4.0, alpha_min: float = 0.5, render_mip: bool = False,
                   max_resolution: Optional[int] = None) -> TriangleMesh:
    """splats: train.Splats (its floor folded in, as eval_stats renders); views: dataset.SceneView, each rendered at its
    loaded size (image_size(max_resolution)).  bounds = (lo, hi) overrides the default box."""
    transforms, raw_opac = splats.folded(ctx)
    lo, hi = bounds if bounds is not None else mesh_bounds(ctx, transforms)
    vol = TsdfVolume(ctx, lo, hi, resolution, trunc_voxels)
    for v in views:
        w, h = v.image_size(max_resolution)
        out = render_splats(ctx, v.camera, (w, h), transforms, splats.sh_coeffs, raw_opac, mip=render_mip,
                            background=(0.0, 0.0, 0.0), rpass=PASS_BACKWARD, render_depth=True)
        vol.integrate(out, alpha_min=alpha_min)
    return vol.extract()
