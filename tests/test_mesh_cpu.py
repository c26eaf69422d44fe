"""Mesh export (DESIGN.md section 4.9) without a GPU: the numpy restatement (tests/mesh_ref.py) on analytic fields and on
an analytic sphere fused from ray-traced views, the PLY writer, and the C ABI's argument checks and struct layout."""
import ctypes
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import mesh_ref as mr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


# ---------------------------------------------------------------------------------------------- helpers shared with GPU tests
def analytic_grid(kind, dims, lo=-1.0, hi=1.0, trunc_voxels=4.0):
    """An exact field on a lattice centred on (lo + hi) / 2 that spans [lo, hi] along its shortest axis: T = clamp(sdf / trunc,
    -1, 1), weight 1, rgb the position mapped to [0, 1].  Returns (grid, origin, h, trunc)."""
    h = F((hi - lo) / max(min(dims) - 1, 1))
    origin = tuple(F((lo + hi) / 2 - (d - 1) * float(h) / 2) for d in dims)
    p = mr.lattice(origin, h, dims).astype(np.float64)
    if kind == "sphere":
        sdf = np.linalg.norm(p, axis=-1) - 0.7
    elif kind == "torus":
        q = np.hypot(p[..., 0], p[..., 1]) - 0.6
        sdf = np.hypot(q, p[..., 2]) - 0.25
    else:
        raise ValueError(kind)
    trunc = F(trunc_voxels * h)
    g = mr.new_grid(dims)
    g["tsdf"][...] = np.clip(sdf / trunc, -1, 1).astype(F)
    g["weight"][...] = 1.0
    g["rgb"][...] = np.clip((p + 1.0) / 2.0, 0, 1).astype(F)
    return g, origin, h, trunc


def analytic_volume(kind):
    return 4.0 / 3.0 * math.pi * 0.7 ** 3 if kind == "sphere" else 2.0 * math.pi ** 2 * 0.6 * 0.25 ** 2


def surface_distance(kind, v):
    v = v.astype(np.float64)
    if kind == "sphere":
        return np.abs(np.linalg.norm(v, axis=-1) - 0.7)
    q = np.hypot(v[:, 0], v[:, 1]) - 0.6
    return np.abs(np.hypot(q, v[:, 2]) - 0.25)


def mesh_topology(v, f):
    """(undirected edge -> count, directed edges unique, Euler characteristic over referenced vertices)."""
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    directed_unique = len(np.unique(e, axis=0)) == len(e)
    und, cnt = np.unique(np.sort(e, axis=1), axis=0, return_counts=True)
    chi = len(np.unique(f)) - len(und) + len(f)
    return cnt, directed_unique, chi


def signed_volume(v, f):
    a, b, c = (v[f[:, i]].astype(np.float64) for i in range(3))
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)


def look_at_quat(pos, target=(0.0, 0.0, 0.0)):
    """Camera rotation (x, y, z, w; local -> world) whose local +z looks from pos at target."""
    z = np.asarray(target, np.float64) - np.asarray(pos, np.float64)
    z /= np.linalg.norm(z)
    a = np.array([0.0, 1.0, 0.0]) if abs(z[1]) < 0.9 else np.array([1.0, 0.0, 0.0])
    x = np.cross(a, z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    m = np.stack([x, y, z], 1)
    w = math.sqrt(max(0.0, 1.0 + m[0, 0] + m[1, 1] + m[2, 2])) / 2.0
    if w > 1e-3:
        q = [(m[2, 1] - m[1, 2]) / (4 * w), (m[0, 2] - m[2, 0]) / (4 * w), (m[1, 0] - m[0, 1]) / (4 * w), w]
    else:                                               # 180 degree turns: largest diagonal
        i = int(np.argmax(np.diag(m)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = math.sqrt(max(0.0, 1.0 + m[i, i] - m[j, j] - m[k, k])) * 2.0
        q = [0.0, 0.0, 0.0, (m[k, j] - m[j, k]) / s]
        q[i], q[j], q[k] = s / 4.0, (m[j, i] + m[i, j]) / s, (m[k, i] + m[i, k]) / s
    q = np.asarray(q)
    return tuple(q / np.linalg.norm(q))


def sphere_views(n, radius=3.0, seed=0):
    """n camera positions on a sphere around the origin (Fibonacci spiral)."""
    i = np.arange(n) + 0.5
    phi = np.arccos(1 - 2 * i / n)
    th = math.pi * (1 + 5 ** 0.5) * i
    return np.stack([np.cos(th) * np.sin(phi), np.cos(phi), np.sin(th) * np.sin(phi)], 1) * radius


SPHERE_R = 1.0


def sphere_color(p):
    return np.clip(0.5 + 0.5 * p / SPHERE_R, 0.0, 1.0)


def trace_sphere(cam_pos, rays_world, cam_z, alpha=0.9):
    """Render maps of the analytic sphere for rays [H,W,3] (world, not normalised) from cam_pos: out_img [H,W,4] with
    premultiplied colour and alpha, D = alpha * (camera-space z of the hit).  Misses are black with alpha 0."""
    o = np.asarray(cam_pos, np.float64)
    d = rays_world / np.linalg.norm(rays_world, axis=-1, keepdims=True)
    b = d @ o
    c = o @ o - SPHERE_R ** 2
    disc = b * b - c
    hit = disc > 0
    t = -b - np.sqrt(np.where(hit, disc, 0.0))
    hit &= t > 0
    p = o + d * t[..., None]
    zc = (p - o) @ np.asarray(cam_z, np.float64)
    img = np.zeros(rays_world.shape[:2] + (4,), F)
    img[..., :3] = np.where(hit[..., None], alpha * sphere_color(p), 0.0)
    img[..., 3] = np.where(hit, alpha, 0.0)
    depth = np.where(hit, alpha * zc, 0.0).astype(F)
    return img, depth


def pinhole_maps(cam, w, h):
    """Ray-traced maps of the analytic sphere through the pixel centres of a pinhole camera.Camera."""
    from brush_b200.camera import build_uniforms
    u = build_uniforms(cam, w, h)
    xs, ys = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    dc = np.stack([(xs - u.cx) / u.fx, (ys - u.cy) / u.fy, np.ones_like(xs)], -1)
    vm = np.asarray(u.viewmat, np.float64).reshape(4, 3)
    r_w2c = vm[:3].T                                     # rows of the world -> camera rotation
    rays = dc @ r_w2c                                    # camera -> world: R^T d
    img, depth = trace_sphere(cam.position, rays, r_w2c[2])
    return u, img, depth


def pinhole_camera(pos, fov=0.9):
    from brush_b200.camera import Camera
    return Camera(position=tuple(float(x) for x in pos), rotation=look_at_quat(pos), fov_x=fov, fov_y=fov)


def fused_sphere_grid(dims, views=30, size=128, lo=-1.3, hi=1.3, poison=False):
    """The restatement's fusion of `views` ray-traced pinhole views of the unit sphere; returns (grid, origin, h, trunc,
    [(uniforms, img, depth)])."""
    h = F((hi - lo) / (max(dims) - 1))
    origin = (F(lo), F(lo), F(lo))
    trunc = F(4.0 * h)
    g = mr.new_grid(dims)
    maps = []
    for k, pos in enumerate(sphere_views(views)):
        if poison and k == 0:
            pos = pos * (1.2 / 3.0)                      # inside the grid: lattice points behind the camera
        u, img, depth = pinhole_maps(pinhole_camera(pos), size, size)
        if poison:
            rng = np.random.default_rng(k)
            sel = rng.random(depth.shape)
            depth[sel < 0.02] = np.nan
            depth[(sel >= 0.02) & (sel < 0.04)] = 0.0
            img[(sel >= 0.04) & (sel < 0.06), 3] = 0.3  # below alpha_min
        mr.integrate(g, origin, h, trunc, u.viewmat, u.fx, u.fy, u.cx, u.cy, img, depth, 0.5)
        maps.append((u, img, depth))
    return g, origin, h, trunc, maps


# ---------------------------------------------------------------------------------------------- restatement on exact fields
@pytest.mark.parametrize("kind", ["sphere", "torus"])
@pytest.mark.parametrize("dims", [(40, 40, 40), (37, 45, 50), (64, 33, 57)])
def test_analytic_field_mesh_is_closed_and_accurate(kind, dims):
    g, origin, h, _ = analytic_grid(kind, dims)
    v, c, f = mr.extract(g, origin, h)
    assert len(f) > 0
    cnt, directed_unique, chi = mesh_topology(v, f)
    assert (cnt == 2).all() and directed_unique
    assert chi == (2 if kind == "sphere" else 0)
    vol = signed_volume(v, f)
    assert vol > 0 and abs(vol / analytic_volume(kind) - 1.0) < 0.02
    assert surface_distance(kind, v).max() < h
    # colours: the interpolated position colour
    np.testing.assert_allclose(c.astype(np.float64) / 255.0, np.clip((v + 1.0) / 2.0, 0, 1), atol=1.0 / 255.0 + 1e-3)


def test_two_point_axis_and_odd_lattices():
    for dims in [(20, 2, 17), (2, 2, 2), (9, 1, 9), (1, 1, 1)]:
        g, origin, h, _ = analytic_grid("sphere", dims, lo=-0.9, hi=0.9)
        v, c, f = mr.extract(g, origin, h)
        if min(dims) < 2:
            assert len(f) == 0
        if len(f):
            cnt, directed_unique, _ = mesh_topology(v, f)
            assert (cnt <= 2).all() and directed_unique
            assert f.max() < len(v)


def test_empty_grids_give_no_triangles():
    g = mr.new_grid((17, 9, 12))
    assert len(mr.extract(g, (0, 0, 0), 0.1)[2]) == 0
    g["weight"][...] = 1.0
    g["tsdf"][...] = 0.5
    v, _, f = mr.extract(g, (0, 0, 0), 0.1)
    assert len(f) == 0 and len(v) == 0


def test_partly_observed_rim_keeps_edges_manifold():
    g, origin, h, _ = analytic_grid("sphere", (33, 30, 31))
    g["weight"][:, :, :12] = 0.0                         # cut the sphere open: unreferenced rim vertices are allowed
    v, _, f = mr.extract(g, origin, h)
    cnt, directed_unique, _ = mesh_topology(v, f)
    assert (cnt <= 2).all() and (cnt == 1).any() and directed_unique


# ---------------------------------------------------------------------------------------------- fusion of ray-traced views
def test_fused_sphere_zero_crossing_within_a_voxel():
    g, origin, h, _, _ = fused_sphere_grid((64, 64, 64))
    v, c, f = mr.extract(g, origin, h)
    d = np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - SPHERE_R)
    assert len(f) > 1000
    assert d.max() < h, (d.max(), h)
    cnt, directed_unique, chi = mesh_topology(v, f)
    assert directed_unique and (cnt == 2).all() and chi == 2
    err = np.abs(c.astype(np.float64) / 255.0 - sphere_color(v.astype(np.float64)))
    assert err.mean() < 0.02


def test_integration_skips_what_it_must():
    """Poisoned maps: NaN or zero depth, low alpha and points behind the camera update nothing; the rest does."""
    dims = (24, 24, 24)
    g, origin, h, trunc, maps = fused_sphere_grid(dims, views=1, poison=True)
    u, img, depth = maps[0]
    p = mr.lattice(origin, h, dims).reshape(-1, 3)
    vm = np.asarray(u.viewmat, F).reshape(4, 3)
    z = p @ vm[:3, 2].astype(np.float64) + vm[3, 2]
    assert (z < 0.01).any() and (g["weight"].reshape(-1)[z < 0.01] == 0).all()
    assert g["weight"].max() == 1.0 and (g["weight"] == 1.0).sum() > 20
    assert np.isfinite(g["tsdf"]).all() and np.isfinite(g["rgb"]).all()
    assert g["tsdf"].min() >= -1.0 and g["tsdf"].max() <= 1.0


# ---------------------------------------------------------------------------------------------- PLY
def parse_mesh_ply(data: bytes):
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").split("\n")
    assert head[0] == "ply" and head[1] == "format binary_little_endian 1.0"
    nv = int(next(l for l in head if l.startswith("element vertex")).split()[2])
    nf = int(next(l for l in head if l.startswith("element face")).split()[2])
    props = [l for l in head if l.startswith("property")]
    assert props == ["property float x", "property float y", "property float z", "property uchar red",
                     "property uchar green", "property uchar blue", "property list uchar int vertex_indices"]
    v = np.zeros((nv, 3), F)
    c = np.zeros((nv, 3), np.uint8)
    off = end
    for i in range(nv):
        v[i] = struct.unpack_from("<3f", data, off)
        c[i] = struct.unpack_from("<3B", data, off + 12)
        off += 15
    f = np.zeros((nf, 3), np.int64)
    for i in range(nf):
        n = data[off]
        assert n == 3
        f[i] = struct.unpack_from("<3i", data, off + 1)
        off += 13
    assert off == len(data)
    return v, c, f


def test_mesh_ply_bytes_round_trip():
    from brush_b200.ply import mesh_to_ply
    g, origin, h, _ = analytic_grid("torus", (21, 19, 17))
    v, c, f = mr.extract(g, origin, h)
    data = mesh_to_ply(v, c, f)
    v2, c2, f2 = parse_mesh_ply(data)
    np.testing.assert_array_equal(v2.view(np.uint32), v.view(np.uint32))
    np.testing.assert_array_equal(c2, c)
    np.testing.assert_array_equal(f2, f)
    empty = mesh_to_ply(np.zeros((0, 3), F), np.zeros((0, 3), np.uint8), np.zeros((0, 3), np.int32))
    assert parse_mesh_ply(empty)[0].shape == (0, 3)
    with pytest.raises(ValueError):
        mesh_to_ply(v, c, np.array([[0, 1, len(v)]]))


# ---------------------------------------------------------------------------------------------- C ABI
def _grid_struct(dims=(8, 8, 8), h=0.1, trunc=0.4, ptr=256):
    from brush_b200 import _lib
    g = _lib.BgTsdfGrid()
    for a in range(3):
        g.dims[a] = dims[a]
    g.h, g.trunc = h, trunc
    g.tsdf = g.weight = g.rgb = ptr
    return g


def test_mesh_entry_points_reject_bad_arguments_before_any_cuda_call():
    from brush_b200 import _lib
    lib = _lib.load()
    fake_ctx = ctypes.create_string_buffer(4096)        # never dereferenced: every check here runs before the context is used
    ctx = ctypes.cast(fake_ctx, ctypes.c_void_p)
    cam = _lib.BgCamera()
    g = _grid_struct()
    img, dep = 4096, 8192                               # aligned, never read
    integ = lambda *a: lib.bg_tsdf_integrate(*a)
    assert integ(None, None, ctypes.byref(g), ctypes.byref(cam), 4, 4, img, dep, 0.5) == _lib.BG_ERR_NULL
    assert integ(ctx, None, None, ctypes.byref(cam), 4, 4, img, dep, 0.5) == _lib.BG_ERR_NULL
    assert integ(ctx, None, ctypes.byref(g), None, 4, 4, img, dep, 0.5) == _lib.BG_ERR_NULL
    assert integ(ctx, None, ctypes.byref(g), ctypes.byref(cam), 4, 4, None, dep, 0.5) == _lib.BG_ERR_NULL
    assert integ(ctx, None, ctypes.byref(_grid_struct(ptr=0)), ctypes.byref(cam), 4, 4, img, dep, 0.5) == _lib.BG_ERR_NULL
    for bad in (_grid_struct(dims=(0, 8, 8)), _grid_struct(dims=(2048, 1024, 1024)), _grid_struct(h=0.0),
                _grid_struct(trunc=-1.0), _grid_struct(h=float("nan")), _grid_struct(ptr=258)):
        assert integ(ctx, None, ctypes.byref(bad), ctypes.byref(cam), 4, 4, img, dep, 0.5) == _lib.BG_ERR_INVALID
    assert integ(ctx, None, ctypes.byref(g), ctypes.byref(cam), 0, 4, img, dep, 0.5) == _lib.BG_ERR_INVALID
    for a in (0.0, -1.0, 1.5, float("nan")):
        assert integ(ctx, None, ctypes.byref(g), ctypes.byref(cam), 4, 4, img, dep, a) == _lib.BG_ERR_INVALID
    assert integ(ctx, None, ctypes.byref(g), ctypes.byref(cam), 4, 4, img + 4, dep, 0.5) == _lib.BG_ERR_INVALID
    bad_cam = _lib.BgCamera()
    bad_cam.camera_model = 7
    assert integ(ctx, None, ctypes.byref(g), ctypes.byref(bad_cam), 4, 4, img, dep, 0.5) == _lib.BG_ERR_INVALID

    nv, nt = ctypes.c_uint32(7), ctypes.c_uint32(7)
    need = int(lib.bg_mesh_workspace_bytes(8, 8, 8))
    assert need > 8 * 8 * 8 * 5
    assert lib.bg_mesh_workspace_bytes(513, 512, 512) > 513 * 512 * 512 * 5
    assert lib.bg_mesh_count(None, None, ctypes.byref(g), 256, need, ctypes.byref(nv), ctypes.byref(nt)) == _lib.BG_ERR_NULL
    assert lib.bg_mesh_count(ctx, None, ctypes.byref(g), None, need, ctypes.byref(nv), ctypes.byref(nt)) == _lib.BG_ERR_NULL
    assert lib.bg_mesh_count(ctx, None, ctypes.byref(g), 256, need, None, ctypes.byref(nt)) == _lib.BG_ERR_NULL
    assert lib.bg_mesh_count(ctx, None, ctypes.byref(g), 256 + 4, need, ctypes.byref(nv), ctypes.byref(nt)) == _lib.BG_ERR_INVALID
    assert lib.bg_mesh_count(ctx, None, ctypes.byref(g), 256, need - 1, ctypes.byref(nv), ctypes.byref(nt)) == _lib.BG_ERR_CAPACITY
    assert nv.value == 0 and nt.value == 0
    assert lib.bg_mesh_count(ctx, None, ctypes.byref(_grid_struct(dims=(8, 0, 8))), 256, need, ctypes.byref(nv),
                             ctypes.byref(nt)) == _lib.BG_ERR_INVALID
    assert lib.bg_mesh_emit(None, None, ctypes.byref(g), 256, need, 0, 0, None, None, None) == _lib.BG_ERR_NULL
    assert lib.bg_mesh_emit(ctx, None, ctypes.byref(g), 256, need, 5, 0, None, None, None) == _lib.BG_ERR_NULL
    assert lib.bg_mesh_emit(ctx, None, ctypes.byref(g), 256, need, 0, 5, None, None, None) == _lib.BG_ERR_NULL
    assert lib.bg_mesh_emit(ctx, None, ctypes.byref(g), 256, need, 5, 5, 258, 512, 1024) == _lib.BG_ERR_INVALID
    assert lib.bg_mesh_emit(ctx, None, ctypes.byref(g), 256, need - 1, 0, 0, None, None, None) == _lib.BG_ERR_CAPACITY


def test_tsdf_grid_layout_matches_the_c_header(tmp_path):
    from brush_b200 import _lib
    fields = ["origin", "h", "dims", "trunc", "tsdf", "weight", "rgb"]
    prog = ['#include <stdio.h>', '#include <stddef.h>', '#include "brush_b200.h"', 'int main(void){',
            'printf("%zu", sizeof(BgTsdfGrid));']
    prog += [f'printf(" %zu", offsetof(BgTsdfGrid, {f}));' for f in fields]
    prog += ['printf("\\n"); return 0;}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(prog))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    tok = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert ctypes.sizeof(_lib.BgTsdfGrid) == int(tok[0])
    for f, off in zip(fields, tok[1:]):
        assert getattr(_lib.BgTsdfGrid, f).offset == int(off), f


def test_grid_dims_and_process_config_defaults():
    from brush_b200.loop import ProcessConfig
    from brush_b200.mesh import grid_dims
    h, dims = grid_dims((-1, -1, -0.5), (1, 1, 0.5), 512)
    assert dims[0] == 512 and dims[1] == 512 and 250 <= dims[2] <= 258
    assert (dims[2] - 1) * h >= 1.0 - 1e-6
    h, dims = grid_dims((0, 0, 0), (1, 1e-4, 1), 64)
    assert dims[1] == 2
    with pytest.raises(ValueError):
        grid_dims((0, 0, 0), (1, 0, 1), 64)
    import dataclasses
    names = [f.name for f in dataclasses.fields(ProcessConfig)]
    assert names[-2:] == ["export_mesh", "mesh_resolution"]
    assert ProcessConfig().export_mesh is False and ProcessConfig().mesh_resolution == 512
