"""Mesh export over the C ABI (DESIGN.md section 4.9; no reference operator): render depth and colour from the training
views, fuse them into a truncated signed distance field on the device, and extract the zero level set as a coloured
triangle mesh by marching tetrahedra.

  TsdfVolume.integrate   <- bg_tsdf_integrate: one view (a render_splats(..., render_depth=True, background=0) output)
  TsdfVolume.extract     <- bg_mesh_count (one readback) + bg_mesh_emit: TriangleMesh in the deterministic order of 4.9
  SparseTsdfVolume       <- the same lattice in 8^3-point bricks near the surface (section 4.10): bg_sparse_tsdf_mark per
                            view, bg_sparse_tsdf_allocate once, bg_sparse_tsdf_integrate per view, bg_sparse_mesh_count /
                            bg_sparse_mesh_emit; the same mesh bit for bit
  splats_to_mesh         <- the whole export: bounds, one render and one integration per view, the extraction; on the
                            sparse grid (a marking pass over the views, then an integration pass) when the dense grid
                            cannot be built
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
        cam, w, h = _view_args(out, camera, "TsdfVolume.integrate")
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


def _view_args(out: RenderOutput, camera, who: str):
    """(BgCamera, w, h) of a render that the integration takes."""
    if out.depth is None or out.out_img.dim() != 3:
        raise ValueError(f"{who} needs a render_splats(..., render_depth=True) output")
    if any(b != 0.0 for b in out.background):
        raise ValueError(f"{who} needs a render on a black background (the colour is un-premultiplied)")
    cam = out.cam if camera is None else _lib.camera_struct(camera)
    return cam, int(out.depth.shape[1]), int(out.depth.shape[0])


def _check_free(ctx: RenderContext, need: int, what: str) -> None:
    free, _ = torch.cuda.mem_get_info(ctx.device)
    if need > free:
        raise MemoryError(f"{what} needs {need / 2**30:.2f} GiB; {free / 2**30:.2f} GiB are free on {ctx.device}: "
                          f"lower the resolution")


BRICK = 8                        # points per brick edge
MAX_SPARSE_BRICKS = (1 << 31) - 1
_MARK_BITMAP_OFFSET = 512        # the mark bitmap's byte offset in the grid workspace (csrc/api.cu, carve_sparse_ws)


class SparseTsdfVolume:
    """TsdfVolume's lattice stored only in the 8^3-point bricks within one brick of a point that some view updates with
    f < 0 (DESIGN.md section 4.10).  Every view is marked before the allocation and integrated after it; the extracted
    mesh equals the dense grid's bit for bit.  4 bytes per brick of the lattice for the brick map, 20 bytes per point of
    the allocated bricks."""

    def __init__(self, ctx: RenderContext, lo, hi, resolution: int = 512, trunc_voxels: float = 4.0):
        h, dims = grid_dims(lo, hi, int(resolution))
        origin = tuple(float(np.float32(x)) for x in np.asarray(lo, np.float64))
        self._setup(ctx, origin, h, dims, float(np.float32(float(trunc_voxels) * h)))

    @classmethod
    def on_lattice(cls, ctx: RenderContext, origin, h: float, dims, trunc: float) -> "SparseTsdfVolume":
        """A grid on an explicit lattice: point (i, j, k) at origin + (i, j, k) * h (f32 arithmetic)."""
        vol = cls.__new__(cls)
        vol._setup(ctx, tuple(float(np.float32(o)) for o in origin), float(np.float32(h)), tuple(int(d) for d in dims),
                   float(np.float32(trunc)))
        return vol

    def _setup(self, ctx, origin, h, dims, trunc):
        self.ctx, self.origin, self.h, self.dims, self.trunc = ctx, origin, h, dims, trunc
        self.brick_dims = tuple((d + BRICK - 1) // BRICK for d in dims)
        nb = self.brick_dims[0] * self.brick_dims[1] * self.brick_dims[2]
        if nb > MAX_SPARSE_BRICKS or max(dims) > (1 << 24):
            raise ValueError(f"sparse TSDF grid {dims} has {nb} bricks; at most 2^31 - 1 bricks and 2^24 points per axis "
                             f"are supported")
        self._ws_view = (0, 0)
        ws = int(_lib.load().bg_sparse_tsdf_workspace_bytes(*dims, 0, 0))
        _check_free(ctx, nb * 4 + ws, f"sparse TSDF grid {dims} ({nb} bricks)")
        self.brick_slot = torch.empty(nb, dtype=torch.int32, device=ctx.device)
        self.workspace = torch.zeros(ws, dtype=torch.uint8, device=ctx.device)
        self.num_bricks = None                           # set by allocate()
        self.tsdf = self.weight = self.rgb = None

    def grid_struct(self) -> _lib.BgSparseTsdfGrid:
        g = _lib.BgSparseTsdfGrid()
        for a in range(3):
            g.origin[a] = self.origin[a]
            g.dims[a] = self.dims[a]
        g.h, g.trunc = self.h, self.trunc
        g.brick_slot = self.brick_slot.data_ptr()
        g.workspace, g.workspace_bytes = self.workspace.data_ptr(), self.workspace.numel()
        if self.num_bricks:
            g.num_bricks = self.num_bricks
            g.tsdf, g.weight, g.rgb = self.tsdf.data_ptr(), self.weight.data_ptr(), self.rgb.data_ptr()
        return g

    def _fit_view(self, w: int, h: int) -> None:
        """Grows the workspace's pyramid part for a w x h view (its first part, the grid's state, is kept)."""
        need = int(_lib.load().bg_sparse_tsdf_workspace_bytes(*self.dims, w, h))
        if need > self.workspace.numel():
            ws = torch.zeros(need, dtype=torch.uint8, device=self.ctx.device)
            ws[:self.workspace.numel()].copy_(self.workspace)
            self.workspace = ws

    def mark(self, out: RenderOutput, camera=None, alpha_min: float = 0.5) -> None:
        """Marks the bricks that one render (as TsdfVolume.integrate takes it) updates with f < 0.  Every view is marked
        before allocate()."""
        if self.num_bricks is not None:
            raise RuntimeError("SparseTsdfVolume.mark after allocate(): a late brick would miss the earlier views")
        cam, w, h = _view_args(out, camera, "SparseTsdfVolume.mark")
        self._fit_view(w, h)
        g = self.grid_struct()
        _lib.check(_lib.load().bg_sparse_tsdf_mark(self.ctx.handle, _stream_ptr(self.ctx.device), C.byref(g), C.byref(cam), w, h,
                                                   out.out_img.data_ptr(), out.depth.data_ptr(), float(alpha_min)),
                   "bg_sparse_tsdf_mark")

    def allocate(self) -> int:
        """Allocates the marked bricks and their neighbours (one readback) and a zeroed pool for them; returns the count."""
        if self.num_bricks is not None:
            raise RuntimeError("SparseTsdfVolume.allocate runs once")
        lib, dev = _lib.load(), self.ctx.device
        n = C.c_uint32()
        g = self.grid_struct()
        _lib.check(lib.bg_sparse_tsdf_allocate(self.ctx.handle, _stream_ptr(dev), C.byref(g), C.byref(n)),
                   "bg_sparse_tsdf_allocate")
        nb = int(n.value)
        _check_free(self.ctx, nb * 512 * 20 + int(lib.bg_sparse_mesh_workspace_bytes(nb)),
                    f"sparse TSDF pool of {nb} bricks with its extraction workspace")
        self.tsdf = torch.zeros((nb, 512), dtype=torch.float32, device=dev)
        self.weight = torch.zeros((nb, 512), dtype=torch.float32, device=dev)
        self.rgb = torch.zeros((nb, 512, 3), dtype=torch.float32, device=dev)
        self.num_bricks = nb
        return nb

    def integrate(self, out: RenderOutput, camera=None, alpha_min: float = 0.5) -> None:
        """Fuses one render into the allocated bricks exactly as TsdfVolume.integrate fuses it into the dense grid."""
        if self.num_bricks is None:
            raise RuntimeError("SparseTsdfVolume.integrate before allocate(): mark every view, then allocate")
        cam, w, h = _view_args(out, camera, "SparseTsdfVolume.integrate")
        g = self.grid_struct()
        _lib.check(_lib.load().bg_sparse_tsdf_integrate(self.ctx.handle, _stream_ptr(self.ctx.device), C.byref(g), C.byref(cam),
                                                        w, h, out.out_img.data_ptr(), out.depth.data_ptr(), float(alpha_min)),
                   "bg_sparse_tsdf_integrate")

    def mark_bitmap(self) -> np.ndarray:
        """The marked bricks, bool [nbz, nby, nbx]."""
        nbx, nby, nbz = self.brick_dims
        nb = nbx * nby * nbz
        words = self.workspace[_MARK_BITMAP_OFFSET:_MARK_BITMAP_OFFSET + (nb + 31) // 32 * 4].cpu().numpy().view(np.uint32)
        bits = np.unpackbits(words.view(np.uint8), bitorder="little")[:nb]
        return bits.astype(bool).reshape(nbz, nby, nbx)

    def slots(self) -> np.ndarray:
        """brick_slot as u32 [nbz, nby, nbx] (0xFFFFFFFF: unallocated)."""
        nbx, nby, nbz = self.brick_dims
        return self.brick_slot.cpu().numpy().view(np.uint32).reshape(nbz, nby, nbx)

    def extract(self) -> TriangleMesh:
        if self.num_bricks is None:
            raise RuntimeError("SparseTsdfVolume.extract before allocate()")
        lib = _lib.load()
        dev = self.ctx.device
        g = self.grid_struct()
        need = int(lib.bg_sparse_mesh_workspace_bytes(self.num_bricks))
        ws = torch.empty(need, dtype=torch.uint8, device=dev)
        nv, nt = C.c_uint32(), C.c_uint32()
        s = _stream_ptr(dev)
        _lib.check(lib.bg_sparse_mesh_count(self.ctx.handle, s, C.byref(g), ws.data_ptr(), need, C.byref(nv), C.byref(nt)),
                   "bg_sparse_mesh_count")
        m, f = int(nv.value), int(nt.value)
        verts = torch.empty((m, 3), dtype=torch.float32, device=dev)
        cols = torch.empty((m, 3), dtype=torch.uint8, device=dev)
        faces = torch.empty((f, 3), dtype=torch.int32, device=dev)
        _lib.check(lib.bg_sparse_mesh_emit(self.ctx.handle, s, C.byref(g), ws.data_ptr(), need, m, f,
                                           verts.data_ptr() if m else None, cols.data_ptr() if m else None,
                                           faces.data_ptr() if f else None), "bg_sparse_mesh_emit")
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
    loaded size (image_size(max_resolution)).  bounds = (lo, hi) overrides the default box.  A grid too large for the
    dense TsdfVolume (over 2^31 - 1 points, or more than the free memory) is built as a SparseTsdfVolume, which renders
    the views twice (once to mark, once to integrate) and gives the mesh the dense grid would."""
    transforms, raw_opac = splats.folded(ctx)
    lo, hi = bounds if bounds is not None else mesh_bounds(ctx, transforms)

    def renders():
        for v in views:
            w, h = v.image_size(max_resolution)
            yield render_splats(ctx, v.camera, (w, h), transforms, splats.sh_coeffs, raw_opac, mip=render_mip,
                                background=(0.0, 0.0, 0.0), rpass=PASS_BACKWARD, render_depth=True)

    try:
        vol = TsdfVolume(ctx, lo, hi, resolution, trunc_voxels)
    except (ValueError, MemoryError):
        vol = SparseTsdfVolume(ctx, lo, hi, resolution, trunc_voxels)
        for out in renders():
            vol.mark(out, alpha_min=alpha_min)
        vol.allocate()
    for out in renders():
        vol.integrate(out, alpha_min=alpha_min)
    return vol.extract()
