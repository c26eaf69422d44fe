"""The sparse brick TSDF (DESIGN.md section 4.10) without a GPU: the candidate stage keeps every brick holding a near
point, the dilation covers every point within one lattice step of a near point, slots follow linear brick order, and
the C ABI's argument checks and struct layout."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import mesh_ref as mr
import sparse_mesh_ref as sr
from test_mesh_cpu import pinhole_camera, pinhole_maps, sphere_views

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


def _lattice(dims, lo=-1.3, hi=1.3):
    h = F((hi - lo) / (max(dims) - 1))
    return (F(lo),) * 3, h, F(4.0 * h)


def _poison(img, depth, seed):
    rng = np.random.default_rng(seed)
    sel = rng.random(depth.shape)
    depth[sel < 0.02] = np.nan
    depth[(sel >= 0.02) & (sel < 0.04)] = 0.0
    depth[(sel >= 0.04) & (sel < 0.05)] = np.inf
    img[(sel >= 0.05) & (sel < 0.07), 3] = 0.3                 # below alpha_min
    return img, depth


def _step_maps(cam, w, h, near_z, far_z, split=0.45):
    """A depth discontinuity over the whole frame, border pixels included: camera-space depth near_z left of the split
    column, far_z right of it, alpha 0.9 everywhere."""
    from brush_b200.camera import build_uniforms
    u = build_uniforms(cam, w, h)
    z = np.where(np.arange(w)[None, :] < int(split * w), near_z, far_z) * np.ones((h, 1))
    img = np.zeros((h, w, 4), F)
    img[..., :3] = 0.9 * 0.5
    img[..., 3] = 0.9
    return u, img, (0.9 * z).astype(F)


def _scenes():
    """(name, [(uniforms, img, depth)]) of pinhole views of the unit sphere and of depth steps around the lattice."""
    out = []
    views = []
    for k, pos in enumerate(sphere_views(8)):
        u, img, depth = pinhole_maps(pinhole_camera(pos), 96, 80)
        views.append((u, *_poison(img, depth, k)))
    out.append(("sphere_poisoned", views))
    # inside the lattice: bricks straddle the near plane z = 0.01
    views = []
    for k, pos in enumerate(sphere_views(4, radius=1.2)):
        u, img, depth = pinhole_maps(pinhole_camera(pos, fov=1.6), 96, 96)
        views.append((u, *_poison(img, depth, 10 + k)))
    out.append(("inside_near_plane", views))
    # close: the sphere covers the whole frame, so the band reaches the image border
    views = [pinhole_maps(pinhole_camera(pos, fov=0.6), 64, 48) for pos in sphere_views(3, radius=1.6)]
    out.append(("sphere_to_border", views))
    # depth steps across the frame
    views = []
    for k, pos in enumerate(sphere_views(3, radius=2.5)):
        views.append(_step_maps(pinhole_camera(pos), 80, 64, 1.7 + 0.1 * k, 2.9))
    out.append(("depth_steps", views))
    return out


@pytest.mark.parametrize("dims", [(37, 45, 50), (24, 24, 24)])
def test_candidates_keep_every_brick_with_a_near_point(dims):
    origin, h, trunc = _lattice(dims)
    for name, views in _scenes():
        kept = total = 0
        for u, img, depth in views:
            near = sr.near_points(origin, h, trunc, dims, u, img, depth)
            need = sr.bricks_of(near, dims)
            cand = sr.candidates(origin, h, trunc, dims, u, img, depth)
            missed = need & ~cand
            assert not missed.any(), (name, np.argwhere(missed)[:5])
            kept += int(cand.sum())
            total += cand.size
            assert near.any() or name == "depth_steps", name
        assert kept < total, name                                 # the test culls something
        # the distorted-model candidate set (whole image) contains the pinhole one
        u, img, depth = views[0]
        whole = sr.candidates(origin, h, trunc, dims, u, img, depth, pinhole=False)
        assert not (sr.candidates(origin, h, trunc, dims, u, img, depth) & ~whole).any()


def test_depth_steps_mark_both_sides_of_the_edge():
    dims = (40, 40, 40)
    origin, h, trunc = _lattice(dims)
    from brush_b200.camera import Camera
    from test_mesh_cpu import look_at_quat
    pos = (0.0, 0.0, -3.0)
    cam = Camera(position=pos, rotation=look_at_quat(pos), fov_x=0.9, fov_y=0.9)
    u, img, depth = _step_maps(cam, 96, 96, 2.6, 3.9)   # world planes z = -0.4 (left) and z = 0.9 (right)
    near = sr.near_points(origin, h, trunc, dims, u, img, depth)
    zs = mr.lattice(origin, h, dims)[..., 2][near]
    assert (np.abs(zs + 0.4) < 0.2).any() and (np.abs(zs - 0.9) < 0.2).any()
    assert not (sr.bricks_of(near, dims) & ~sr.candidates(origin, h, trunc, dims, u, img, depth)).any()


def test_dilation_covers_every_point_within_one_step_of_a_near_point():
    dims = (37, 45, 50)
    origin, h, trunc = _lattice(dims)
    near = np.zeros(dims[::-1], bool)
    for _, views in _scenes():
        for u, img, depth in views:
            near |= sr.near_points(origin, h, trunc, dims, u, img, depth)
    alloc = sr.dilate(sr.bricks_of(near, dims))
    k, j, i = np.nonzero(near)
    assert len(k) > 1000
    for dk in (-1, 0, 1):
        for dj in (-1, 0, 1):
            for di in (-1, 0, 1):
                kk, jj, ii = k + dk, j + dj, i + di
                ok = (kk >= 0) & (jj >= 0) & (ii >= 0) & (kk < dims[2]) & (jj < dims[1]) & (ii < dims[0])
                assert alloc[kk[ok] // 8, jj[ok] // 8, ii[ok] // 8].all()
    slots = sr.assign_slots(alloc)
    flat = slots.reshape(-1)
    assert (flat[alloc.reshape(-1)] == np.arange(alloc.sum())).all()
    assert (flat[~alloc.reshape(-1)] == sr.UNALLOCATED).all()


def test_final_negative_points_were_near_in_some_view():
    """A point whose fused T < 0 is near in at least one view (DESIGN.md section 4.10, fact 1)."""
    dims = (37, 45, 50)
    origin, h, trunc = _lattice(dims)
    g = mr.new_grid(dims)
    near = np.zeros(dims[::-1], bool)
    for _, views in _scenes():
        for u, img, depth in views:
            mr.integrate(g, origin, h, trunc, u.viewmat, u.fx, u.fy, u.cx, u.cy, img, depth, 0.5)
            near |= sr.near_points(origin, h, trunc, dims, u, img, depth)
    neg = (g["tsdf"] < 0) & (g["weight"] != 0)
    assert neg.any() and not (neg & ~near).any()
    # and the dense mesh only touches allocated bricks
    v, _, f = mr.extract(g, origin, h)
    alloc = sr.dilate(sr.bricks_of(near, dims))
    p = np.rint((v.astype(np.float64) - np.asarray(origin, np.float64)) / float(h) - 0.5).astype(np.int64)
    p = np.clip(p, 0, np.asarray(dims) - 1)
    assert len(f) > 0 and alloc[p[:, 2] // 8, p[:, 1] // 8, p[:, 0] // 8].all()


# ---------------------------------------------------------------------------------------------- C ABI
def _sparse_struct(dims=(64, 64, 64), h=0.1, trunc=0.4, slot=256, ws=512, ws_bytes=None, num_bricks=0, pool=0):
    from brush_b200 import _lib
    g = _lib.BgSparseTsdfGrid()
    for a in range(3):
        g.dims[a] = dims[a]
    g.h, g.trunc = h, trunc
    g.brick_slot = slot
    g.workspace = ws
    g.workspace_bytes = (int(_lib.load().bg_sparse_tsdf_workspace_bytes(*dims, 64, 64)) if ws_bytes is None else ws_bytes)
    g.num_bricks = num_bricks
    g.tsdf = g.weight = g.rgb = pool
    return g


def test_sparse_entry_points_reject_bad_arguments_before_any_cuda_call():
    from brush_b200 import _lib
    lib = _lib.load()
    fake_ctx = ctypes.create_string_buffer(4096)            # never dereferenced: every check here runs before the context is used
    ctx = ctypes.cast(fake_ctx, ctypes.c_void_p)
    cam = _lib.BgCamera()
    g = _sparse_struct()
    img, dep = 4096, 8192
    R = ctypes.byref
    for fn in (lib.bg_sparse_tsdf_mark, lib.bg_sparse_tsdf_integrate):
        assert fn(None, None, R(g), R(cam), 4, 4, img, dep, 0.5) == _lib.BG_ERR_NULL
        assert fn(ctx, None, None, R(cam), 4, 4, img, dep, 0.5) == _lib.BG_ERR_NULL
        assert fn(ctx, None, R(g), None, 4, 4, img, dep, 0.5) == _lib.BG_ERR_NULL
        assert fn(ctx, None, R(g), R(cam), 4, 4, None, dep, 0.5) == _lib.BG_ERR_NULL
        assert fn(ctx, None, R(_sparse_struct(slot=0)), R(cam), 4, 4, img, dep, 0.5) == _lib.BG_ERR_NULL
        assert fn(ctx, None, R(_sparse_struct(ws=0)), R(cam), 4, 4, img, dep, 0.5) == _lib.BG_ERR_NULL
        for bad in (_sparse_struct(dims=(0, 8, 8)), _sparse_struct(dims=(1 << 24 | 1, 8, 8)),
                    _sparse_struct(dims=(1 << 14, 1 << 14, 1 << 14), ws_bytes=1 << 40), _sparse_struct(h=0.0),
                    _sparse_struct(trunc=-1.0), _sparse_struct(h=float("nan")), _sparse_struct(slot=258),
                    _sparse_struct(ws=256 + 64)):
            assert fn(ctx, None, R(bad), R(cam), 4, 4, img, dep, 0.5) == _lib.BG_ERR_INVALID
        assert fn(ctx, None, R(g), R(cam), 0, 4, img, dep, 0.5) == _lib.BG_ERR_INVALID
        for a in (0.0, -1.0, 1.5, float("nan")):
            assert fn(ctx, None, R(g), R(cam), 4, 4, img, dep, a) == _lib.BG_ERR_INVALID
        assert fn(ctx, None, R(g), R(cam), 4, 4, img + 4, dep, 0.5) == _lib.BG_ERR_INVALID
        bad_cam = _lib.BgCamera()
        bad_cam.camera_model = 7
        assert fn(ctx, None, R(g), R(bad_cam), 4, 4, img, dep, 0.5) == _lib.BG_ERR_INVALID
    # the workspace must hold the view's pyramid (mark) or the grid's state (the other calls)
    need_view = int(lib.bg_sparse_tsdf_workspace_bytes(64, 64, 64, 128, 128))
    small = _sparse_struct(ws_bytes=need_view - 1)
    assert lib.bg_sparse_tsdf_mark(ctx, None, R(small), R(cam), 128, 128, img, dep, 0.5) == _lib.BG_ERR_CAPACITY
    need_state = int(lib.bg_sparse_tsdf_workspace_bytes(64, 64, 64, 0, 0))
    assert 0 < need_state < need_view
    n = ctypes.c_uint32(7)
    assert lib.bg_sparse_tsdf_allocate(ctx, None, R(_sparse_struct(ws_bytes=need_state - 1)), R(n)) == _lib.BG_ERR_CAPACITY
    assert n.value == 0
    assert lib.bg_sparse_tsdf_allocate(ctx, None, R(g), None) == _lib.BG_ERR_NULL
    assert lib.bg_sparse_tsdf_allocate(None, None, R(g), R(n)) == _lib.BG_ERR_NULL
    assert lib.bg_sparse_tsdf_allocate(ctx, None, R(_sparse_struct(dims=(8, 0, 8))), R(n)) == _lib.BG_ERR_INVALID
    # the pool
    assert lib.bg_sparse_tsdf_integrate(ctx, None, R(_sparse_struct(num_bricks=4)), R(cam), 4, 4, img, dep, 0.5) == _lib.BG_ERR_NULL
    assert lib.bg_sparse_tsdf_integrate(ctx, None, R(_sparse_struct(num_bricks=4, pool=258)), R(cam), 4, 4, img, dep,
                                        0.5) == _lib.BG_ERR_INVALID
    # extraction
    nv, nt = ctypes.c_uint32(7), ctypes.c_uint32(7)
    gp = _sparse_struct(num_bricks=4, pool=1024)
    need = int(lib.bg_sparse_mesh_workspace_bytes(4))
    assert need > 4 * 512 * 5 and lib.bg_sparse_mesh_workspace_bytes(8) > need
    assert lib.bg_sparse_mesh_count(ctx, None, R(gp), 256, need, None, R(nt)) == _lib.BG_ERR_NULL
    assert lib.bg_sparse_mesh_count(ctx, None, R(gp), None, need, R(nv), R(nt)) == _lib.BG_ERR_NULL
    assert lib.bg_sparse_mesh_count(ctx, None, R(gp), 256 + 4, need, R(nv), R(nt)) == _lib.BG_ERR_INVALID
    assert lib.bg_sparse_mesh_count(ctx, None, R(gp), 256, need - 1, R(nv), R(nt)) == _lib.BG_ERR_CAPACITY
    assert nv.value == 0 and nt.value == 0
    assert lib.bg_sparse_mesh_count(ctx, None, R(_sparse_struct(num_bricks=4)), 256, need, R(nv), R(nt)) == _lib.BG_ERR_NULL
    assert lib.bg_sparse_mesh_emit(None, None, R(gp), 256, need, 0, 0, None, None, None) == _lib.BG_ERR_NULL
    assert lib.bg_sparse_mesh_emit(ctx, None, R(gp), 256, need, 5, 0, None, None, None) == _lib.BG_ERR_NULL
    assert lib.bg_sparse_mesh_emit(ctx, None, R(gp), 256, need, 0, 5, None, None, None) == _lib.BG_ERR_NULL
    assert lib.bg_sparse_mesh_emit(ctx, None, R(gp), 256, need, 5, 5, 258, 512, 1024) == _lib.BG_ERR_INVALID
    assert lib.bg_sparse_mesh_emit(ctx, None, R(gp), 256, need - 1, 0, 0, None, None, None) == _lib.BG_ERR_CAPACITY


def test_sparse_grid_layout_matches_the_c_header(tmp_path):
    from brush_b200 import _lib
    fields = ["origin", "h", "dims", "trunc", "brick_slot", "workspace", "workspace_bytes", "num_bricks", "tsdf", "weight", "rgb"]
    prog = ['#include <stdio.h>', '#include <stddef.h>', '#include "brush_b200.h"', 'int main(void){',
            'printf("%zu", sizeof(BgSparseTsdfGrid));']
    prog += [f'printf(" %zu", offsetof(BgSparseTsdfGrid, {f}));' for f in fields]
    prog += ['printf("\\n"); return 0;}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(prog))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    tok = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert ctypes.sizeof(_lib.BgSparseTsdfGrid) == int(tok[0])
    for f, off in zip(fields, tok[1:]):
        assert getattr(_lib.BgSparseTsdfGrid, f).offset == int(off), f


def test_sparse_workspace_follows_bricks_not_points():
    from brush_b200 import _lib
    lib = _lib.load()
    small = int(lib.bg_sparse_tsdf_workspace_bytes(512, 512, 512, 0, 0))
    big = int(lib.bg_sparse_tsdf_workspace_bytes(2048, 2048, 2048, 0, 0))
    nb = 256 ** 3
    assert nb * 4 < big < nb * 5                             # the brick list and the bitmap: about 4.2 bytes per brick
    assert 60 < big / small < 68
    assert lib.bg_sparse_mesh_workspace_bytes(1000) < 1000 * 512 * 6
