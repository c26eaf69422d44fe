"""Mesh export on the device (DESIGN.md section 4.9) against the numpy restatement (tests/mesh_ref.py): integration and
extraction bit for bit, repeatability, the capacity error, fisheye views, splats_to_mesh end to end and the training
loop's mesh export."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

import mesh_ref as mr
from test_mesh_cpu import (SPHERE_R, analytic_grid, fused_sphere_grid, look_at_quat, mesh_topology, parse_mesh_ply,
                           signed_volume, sphere_color, sphere_views, trace_sphere)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
F = np.float32


def _volume_from(ctx, grid, origin, h, trunc):
    """A TsdfVolume holding a copy of a restatement grid."""
    import torch
    from brush_b200.mesh import TsdfVolume
    vol = TsdfVolume.__new__(TsdfVolume)
    vol.ctx = ctx
    vol.dims = grid["tsdf"].shape[::-1]
    vol.h, vol.trunc = float(F(h)), float(F(trunc))
    vol.origin = tuple(float(F(o)) for o in origin)
    vol.tsdf, vol.weight, vol.rgb = (torch.from_numpy(np.ascontiguousarray(grid[k])).to(ctx.device)
                                     for k in ("tsdf", "weight", "rgb"))
    return vol


def _integrate(vol, u, img, depth, alpha_min=0.5):
    import torch
    from brush_b200 import _lib
    from brush_b200.render import _stream_ptr
    dev = vol.ctx.device
    ti = torch.from_numpy(np.ascontiguousarray(img, F)).to(dev)
    td = torch.from_numpy(np.ascontiguousarray(depth, F)).to(dev)
    g, cam = vol.grid_struct(), _lib.camera_struct(u)
    _lib.check(_lib.load().bg_tsdf_integrate(vol.ctx.handle, _stream_ptr(dev), C.byref(g), C.byref(cam), depth.shape[1],
                                             depth.shape[0], ti.data_ptr(), td.data_ptr(), float(alpha_min)), "bg_tsdf_integrate")


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("dims", [(64, 64, 64), (37, 64, 50)])
def test_integration_matches_the_restatement_bit_for_bit(dims):
    import brush_b200.render as R
    ref, origin, h, trunc, maps = fused_sphere_grid(dims, views=12, poison=True)
    ctx = R.RenderContext(16, 128, 128)
    vol = _volume_from(ctx, mr.new_grid(dims), origin, h, trunc)
    for u, img, depth in maps:
        _integrate(vol, u, img, depth)
    for k, t in (("tsdf", vol.tsdf), ("weight", vol.weight), ("rgb", vol.rgb)):
        got = t.cpu().numpy()
        assert (_bits(got) == _bits(ref[k])).all(), (k, int((_bits(got) != _bits(ref[k])).sum()))
    assert ref["weight"].max() >= 5
    ctx.close()


def _grid_case(name):
    if name == "sphere40":
        return analytic_grid("sphere", (40, 40, 40))
    if name == "torus_odd":
        return analytic_grid("torus", (37, 45, 50))
    if name == "two_point_axis":
        return analytic_grid("sphere", (20, 2, 17), lo=-0.9, hi=0.9)
    if name == "fused":
        return fused_sphere_grid((37, 64, 50), views=12, poison=True)[:4]
    g, origin, h, trunc = analytic_grid("torus", (33, 30, 31))
    g["weight"][:, :, :12] = 0.0
    return g, origin, h, trunc


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["sphere40", "torus_odd", "two_point_axis", "fused", "open_rim"])
def test_extraction_matches_the_restatement(name):
    import brush_b200.render as R
    g, origin, h, trunc = _grid_case(name)
    v, c, f = mr.extract(g, origin, h)
    ctx = R.RenderContext(16, 16, 16)
    m = _volume_from(ctx, g, origin, h, trunc).extract()
    assert m.vertices.shape == v.shape and m.faces.shape == f.shape
    assert (_bits(m.vertices) == _bits(v)).all()
    assert (m.colors == c).all()
    assert (m.faces.astype(np.int64) == f).all()
    ctx.close()


@pytest.mark.gpu
def test_extraction_repeats_and_reports_capacity():
    import torch
    import brush_b200.render as R
    from brush_b200 import _lib
    from brush_b200.render import _stream_ptr
    g, origin, h, trunc = analytic_grid("torus", (70, 61, 66))
    ctx = R.RenderContext(16, 16, 16)
    vol = _volume_from(ctx, g, origin, h, trunc)
    a, b = vol.extract(), vol.extract()
    assert a.to_ply() == b.to_ply() and len(a.faces) > 1000
    # the capacity error: nothing is written
    lib, dev = _lib.load(), ctx.device
    grid = vol.grid_struct()
    need = int(lib.bg_mesh_workspace_bytes(*vol.dims))
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    nv, nt = C.c_uint32(), C.c_uint32()
    s = _stream_ptr(dev)
    _lib.check(lib.bg_mesh_count(ctx.handle, s, C.byref(grid), ws.data_ptr(), need, C.byref(nv), C.byref(nt)), "count")
    assert (nv.value, nt.value) == (len(a.vertices), len(a.faces))
    verts = torch.full((nv.value, 3), -7.0, device=dev)
    cols = torch.zeros((nv.value, 3), dtype=torch.uint8, device=dev)
    faces = torch.full((nt.value, 3), -1, dtype=torch.int32, device=dev)
    for mv, mt in ((nv.value - 1, nt.value), (nv.value, nt.value - 1)):
        st = lib.bg_mesh_emit(ctx.handle, s, C.byref(grid), ws.data_ptr(), need, mv, mt, verts.data_ptr(), cols.data_ptr(),
                              faces.data_ptr())
        assert st == _lib.BG_ERR_CAPACITY
    torch.cuda.synchronize()
    assert bool((verts == -7.0).all()) and bool((faces == -1).all())
    # a workspace counted for other dims is refused
    other = analytic_grid("sphere", (70, 61, 65))
    vol2 = _volume_from(ctx, *other)
    g2 = vol2.grid_struct()
    assert lib.bg_mesh_emit(ctx.handle, s, C.byref(g2), ws.data_ptr(), need, 1 << 30, 1 << 30, verts.data_ptr(),
                            cols.data_ptr(), faces.data_ptr()) == _lib.BG_ERR_INVALID
    # empty grids
    e = _volume_from(ctx, mr.new_grid((17, 9, 12)), (0, 0, 0), 0.1, 0.4).extract()
    assert e.vertices.shape == (0, 3) and e.faces.shape == (0, 3)
    ctx.close()


def _fisheye_maps(cam, w, h):
    """Ray-traced maps through the pixel centres of a KB4 or thin-prism fisheye camera: the projection inverted by a
    fixed-point iteration on the prism term around the monotone KB4 radius inversion."""
    from brush_b200.camera import THIN_PRISM_FISHEYE, build_uniforms
    u = build_uniforms(cam, w, h)
    k1, k2, k3, k4 = (float(x) for x in u.model_params[:4])
    xs, ys = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    m = np.stack([(xs - u.cx) / u.fx, (ys - u.cy) / u.fy], -1)

    def inv(rd):                                          # Newton on d(theta) = theta (1 + k1 theta^2 + ...) = rd
        th = rd.copy()
        for _ in range(30):
            t2 = th * th
            d = th * (1 + t2 * (k1 + t2 * (k2 + t2 * (k3 + t2 * k4))))
            dd = 1 + t2 * (3 * k1 + t2 * (5 * k2 + t2 * (7 * k3 + t2 * 9 * k4)))
            th = np.clip(th - (d - rd) / dd, 0.0, math.pi)
        return th

    def kb4_inverse(mm):
        rd = np.linalg.norm(mm, axis=-1)
        th = inv(rd)
        s = np.where(rd > 0, np.sin(th) / np.maximum(rd, 1e-30), 1.0)
        return np.stack([mm[..., 0] * s, mm[..., 1] * s, np.cos(th)], -1)

    d = kb4_inverse(m)
    if u.camera_model == THIN_PRISM_FISHEYE:
        p1, p2, sx1, sy1 = (float(x) for x in u.model_params[4:8])
        for _ in range(20):
            a, b = d[..., 0] / d[..., 2], d[..., 1] / d[..., 2]
            r2 = a * a + b * b
            nu = 2 * p1 * a * b + p2 * (3 * a * a + b * b) + sx1 * r2
            nv = 2 * p2 * a * b + p1 * (a * a + 3 * b * b) + sy1 * r2
            d = kb4_inverse(m - np.stack([nu, nv], -1))
    vm = np.asarray(u.viewmat, np.float64).reshape(4, 3)
    r_w2c = vm[:3].T
    img, depth = trace_sphere(cam.position, d @ r_w2c, r_w2c[2])
    return u, img, depth


@pytest.mark.gpu
def test_fisheye_views_fuse_to_within_a_voxel():
    import brush_b200.render as R
    from brush_b200.camera import KANNALA_BRANDT_4, THIN_PRISM_FISHEYE, Camera
    dims = (64, 64, 64)
    lo, hi = -1.3, 1.3
    h = F((hi - lo) / (dims[0] - 1))
    origin = (F(lo),) * 3
    ctx = R.RenderContext(16, 192, 192)
    vol = _volume_from(ctx, mr.new_grid(dims), origin, h, F(4 * h))
    for i, pos in enumerate(sphere_views(24, radius=1.8)):
        if i % 2 == 0:
            cam = Camera(position=tuple(pos), rotation=look_at_quat(pos), fov_x=2.2, fov_y=2.2, camera_model=KANNALA_BRANDT_4,
                         model_params=(0.05, -0.01, 0.002, -0.0005))
        else:
            cam = Camera(position=tuple(pos), rotation=look_at_quat(pos), fov_x=2.2, fov_y=2.2,
                         camera_model=THIN_PRISM_FISHEYE, model_params=(0.05, -0.01, 0.002, -0.0005, 0.001, -0.001, 0.002, 0.001))
        u, img, depth = _fisheye_maps(cam, 192, 192)
        _integrate(vol, u, img, depth)
    m = vol.extract()
    d = np.abs(np.linalg.norm(m.vertices.astype(np.float64), axis=1) - SPHERE_R)
    assert len(m.faces) > 1000
    assert d.max() < h, (float(d.max()), float(h))
    cnt, directed_unique, chi = mesh_topology(m.vertices, m.faces)
    assert directed_unique and (cnt == 2).all() and chi == 2
    ctx.close()


def _sphere_splats(n, seed=0):
    """n small flat opaque splats on the unit sphere, coloured by position (DC only)."""
    i = np.arange(n) + 0.5
    phi = np.arccos(1 - 2 * i / n)
    th = math.pi * (1 + 5 ** 0.5) * i
    p = np.stack([np.cos(th) * np.sin(phi), np.cos(phi), np.sin(th) * np.sin(phi)], 1)
    t = np.zeros((n, 10), F)
    t[:, :3] = p
    # quaternion (w, x, y, z) turning +z onto the normal p
    ax = np.cross(np.array([0.0, 0.0, 1.0]), p)
    s = np.linalg.norm(ax, axis=1, keepdims=True)
    ang = np.arctan2(s[:, 0], p[:, 2])
    ax = np.where(s > 1e-9, ax / np.maximum(s, 1e-12), np.array([1.0, 0.0, 0.0]))
    t[:, 3] = np.cos(ang / 2)
    t[:, 4:7] = ax * np.sin(ang / 2)[:, None]
    spacing = math.sqrt(4 * math.pi / n)
    t[:, 7:9] = math.log(0.8 * spacing)
    t[:, 9] = math.log(1e-4)
    sh = ((sphere_color(p) - 0.5) / 0.2820947917738781).astype(F)[:, None, :]
    op = np.full(n, 6.0, F)
    return t, sh, op


@pytest.mark.gpu
def test_splats_to_mesh_end_to_end(tmp_path):
    """100k flat opaque splats on the unit sphere, 40 views of 256x256, a 128^3 grid.  Measured on an H100: 168078
    vertices, 336152 faces in one closed component (chi = 2), mean |r - 1| = 0.0075 scene units (about 0.4 voxel; the
    expected depth of the blended splats sits slightly inside the sphere), vertex colour mean error 0.0024."""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    import torch
    from PIL import Image
    import brush_b200.render as R
    import brush_b200.train as T
    from brush_b200.camera import Camera
    from brush_b200.dataset import SceneView
    from brush_b200.mesh import grid_dims, mesh_bounds, splats_to_mesh
    n, size, res = 100_000, 256, 128
    t, sh, op = _sphere_splats(n)
    ctx = R.RenderContext(n, size, size)
    splats = T.Splats(*(torch.from_numpy(x).to(ctx.device) for x in (t, sh, op)))
    path = str(tmp_path / "blank.png")
    Image.fromarray(np.zeros((size, size, 3), np.uint8)).save(path)
    views = [SceneView(Camera(position=tuple(p), rotation=look_at_quat(p), fov_x=0.9, fov_y=0.9), path)
             for p in sphere_views(40)]
    m = splats_to_mesh(ctx, splats, views, resolution=res)
    v = m.vertices.astype(np.float64)
    f = m.faces.astype(np.int64)
    adj = sp.coo_matrix((np.ones(len(f) * 3), (np.repeat(f[:, 0], 3), f.reshape(-1))), shape=(len(v), len(v)))
    _, lab = connected_components(adj, directed=False)
    big = np.bincount(lab[f[:, 0]]).argmax()
    fb = f[lab[f[:, 0]] == big]
    cnt, directed_unique, chi = mesh_topology(v, fb)
    h = grid_dims(*mesh_bounds(ctx, splats.transforms), res)[0]
    used = np.unique(fb)
    err = np.abs(np.linalg.norm(v[used], axis=1) - 1.0)
    cerr = np.abs(m.colors[used].astype(np.float64) / 255.0 - sphere_color(v[used]))
    print(f"end to end: {len(v)} vertices, {len(f)} faces, largest component {len(fb)} faces, chi {chi}, "
          f"mean |r - 1| {err.mean():.5f} ({err.mean() / h:.3f} voxel), max {err.max():.5f}, colour mean err {cerr.mean():.4f}")
    assert directed_unique and (cnt == 2).all() and chi == 2
    assert err.mean() < 0.5 * h
    assert cerr.mean() < 0.01
    assert signed_volume(v, fb) > 0
    ctx.close()


@pytest.mark.gpu
def test_train_loop_writes_a_mesh(tmp_path):
    import torch
    import train_colmap
    import brush_b200.render as R
    import brush_b200.train as T
    from brush_b200 import dataset as ds
    from brush_b200 import splat_init
    from brush_b200.loop import ProcessConfig, train_loop
    w, h, views = 128, 96, 8
    ctx = R.RenderContext(20_000, w, h, 0, device=0)
    train_colmap.make_dataset(str(tmp_path / "set"), ctx, views, w, h, 3_000, 1_500, seed=0xB2000003)
    loaded = ds.load_colmap(str(tmp_path / "set"), eval_split_every=8)
    outs = {}
    for flag in (False, True):
        tr0, sh0, op0 = splat_init.to_init_splats(loaded.init_splat)
        splats = T.Splats(*(torch.from_numpy(np.ascontiguousarray(x)).to(ctx.device) for x in (tr0, sh0, op0)))
        cfg = T.TrainConfig(total_train_iters=30, max_splats=15_000, refine_every=100, seed=1)
        out_dir = tmp_path / f"out_{flag}"
        train_loop(ctx, splats, loaded.train, [], cfg,
                   ProcessConfig(export_every=30, export_path=str(out_dir), seed=7, export_mesh=flag, mesh_resolution=96))
        outs[flag] = {name: open(out_dir / name, "rb").read() for name in sorted(os.listdir(out_dir))}
    assert sorted(outs[False]) == ["export_30.ply"]
    assert sorted(outs[True]) == ["export_30.ply", "export_30_mesh.ply"]
    v, c, f = parse_mesh_ply(outs[True]["export_30_mesh.ply"])
    assert len(v) > 0 and len(f) > 0 and f.max() < len(v) and np.isfinite(v).all()
    ctx.close()


def test_no_spill_in_mesh_kernels():
    path = os.path.join(ROOT, "brush_b200", "csrc", "_obj", "mesh.o.ptxas.txt")
    if not os.path.exists(path):
        from brush_b200 import build
        build.build(force=True)
    txt = open(path).read()
    assert txt.count("Compiling entry function") == 6
    spill = [ln for ln in txt.splitlines() if "spill" in ln]
    assert len(spill) == 6 and all(ln.strip().startswith("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads")
                                   for ln in spill)
