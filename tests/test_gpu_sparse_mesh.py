"""The sparse brick TSDF on the device (DESIGN.md section 4.10): marks and slots against the restatement
(tests/sparse_mesh_ref.py), every allocated point bit-equal to the dense grid, and the extracted mesh bit-equal to the
dense mesh, for fused pinhole and fisheye views, splats_to_mesh, and a lattice of more than 2^31 points."""
import ctypes as C
import os

import numpy as np
import pytest

import mesh_ref as mr
import sparse_mesh_ref as sr
from test_mesh_cpu import fused_sphere_grid, look_at_quat, sphere_views

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint32)


def _call(vol, fn, u, img, depth, alpha_min=0.5):
    """One bg_sparse_tsdf_mark / bg_sparse_tsdf_integrate on numpy maps."""
    import torch
    from brush_b200 import _lib
    from brush_b200.render import _stream_ptr
    dev = vol.ctx.device
    ti = torch.from_numpy(np.ascontiguousarray(img, F)).to(dev)
    td = torch.from_numpy(np.ascontiguousarray(depth, F)).to(dev)
    vol._fit_view(depth.shape[1], depth.shape[0])
    g, cam = vol.grid_struct(), _lib.camera_struct(u)
    return getattr(_lib.load(), fn)(vol.ctx.handle, _stream_ptr(dev), C.byref(g), C.byref(cam), depth.shape[1], depth.shape[0],
                                    ti.data_ptr(), td.data_ptr(), float(alpha_min))


def sparse_from_maps(ctx, dims, origin, h, trunc, maps):
    """A SparseTsdfVolume over the lattice with every view marked, the bricks allocated and every view integrated."""
    from brush_b200 import _lib
    from brush_b200.mesh import SparseTsdfVolume
    vol = SparseTsdfVolume.on_lattice(ctx, origin, h, dims, trunc)
    for u, img, depth in maps:
        _lib.check(_call(vol, "bg_sparse_tsdf_mark", u, img, depth), "mark")
    vol.allocate()
    for u, img, depth in maps:
        _lib.check(_call(vol, "bg_sparse_tsdf_integrate", u, img, depth), "integrate")
    return vol


def _dense_from_maps(ctx, dims, origin, h, trunc, maps):
    from test_gpu_mesh import _integrate, _volume_from
    vol = _volume_from(ctx, mr.new_grid(dims), origin, h, trunc)
    for u, img, depth in maps:
        _integrate(vol, u, img, depth)
    return vol


def _same_mesh(a, b):
    assert a.vertices.shape == b.vertices.shape and a.faces.shape == b.faces.shape
    assert (_bits(a.vertices) == _bits(b.vertices)).all()
    assert (a.colors == b.colors).all()
    assert (a.faces.astype(np.int64) == b.faces.astype(np.int64)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("dims", [(64, 64, 64), (37, 64, 50)])
def test_marks_slots_points_and_mesh_match_the_dense_grid(dims):
    import brush_b200.render as R
    ref, origin, h, trunc, maps = fused_sphere_grid(dims, views=12, poison=True)
    ctx = R.RenderContext(16, 128, 128)
    from brush_b200.mesh import SparseTsdfVolume
    from brush_b200 import _lib
    vol = SparseTsdfVolume.on_lattice(ctx, origin, h, dims, trunc)
    marked = np.zeros(sr.brick_dims(dims)[::-1], bool)
    for u, img, depth in maps:
        _lib.check(_call(vol, "bg_sparse_tsdf_mark", u, img, depth), "mark")
        marked |= sr.bricks_of(sr.near_points(origin, h, trunc, dims, u, img, depth), dims)
    got = vol.mark_bitmap()
    assert (got == marked).all(), int((got != marked).sum())
    n = vol.allocate()
    alloc = sr.dilate(marked)
    assert n == int(alloc.sum()) and n < alloc.size
    assert (vol.slots() == sr.assign_slots(alloc)).all()
    for u, img, depth in maps:
        _lib.check(_call(vol, "bg_sparse_tsdf_integrate", u, img, depth), "integrate")
    # every allocated point holds the dense grid's bits; no point outside the allocation is negative
    bz, by, bx = np.nonzero(alloc)
    pz, py, px = np.meshgrid(np.arange(8), np.arange(8), np.arange(8), indexing="ij")
    i = (bx[:, None] * 8 + px.reshape(-1)[None, :])
    j = (by[:, None] * 8 + py.reshape(-1)[None, :])
    k = (bz[:, None] * 8 + pz.reshape(-1)[None, :])
    inside = (i < dims[0]) & (j < dims[1]) & (k < dims[2])
    for key, t in (("tsdf", vol.tsdf), ("weight", vol.weight), ("rgb", vol.rgb)):
        pool = t.cpu().numpy()
        exp = ref[key][np.minimum(k, dims[2] - 1), np.minimum(j, dims[1] - 1), np.minimum(i, dims[0] - 1)]
        assert (_bits(pool[inside]) == _bits(exp[inside])).all(), key
        assert (_bits(pool[~inside]) == 0).all(), key
    covered = np.zeros(dims[::-1], bool)
    covered[k[inside], j[inside], i[inside]] = True
    assert not ((ref["tsdf"] < 0) & ~covered).any()
    assert ref["weight"][~covered].any()                    # free space outside the allocation was observed by the dense grid
    m = vol.extract()
    _same_mesh(m, _volume_from_ref(ctx, ref, origin, h, trunc).extract())
    v, c, f = mr.extract(ref, origin, h)
    assert (_bits(m.vertices) == _bits(v)).all() and (m.colors == c).all() and (m.faces == f).all() and len(f) > 1000
    ctx.close()


def _volume_from_ref(ctx, ref, origin, h, trunc):
    from test_gpu_mesh import _volume_from
    return _volume_from(ctx, ref, origin, h, trunc)


@pytest.mark.gpu
def test_phases_capacity_and_repeatability():
    import torch
    import brush_b200.render as R
    from brush_b200 import _lib
    from brush_b200.render import _stream_ptr
    from brush_b200.mesh import SparseTsdfVolume
    dims = (40, 33, 47)
    _, origin, h, trunc, maps = fused_sphere_grid(dims, views=6)
    ctx = R.RenderContext(16, 128, 128)
    vol = SparseTsdfVolume.on_lattice(ctx, origin, h, dims, trunc)
    lib, dev, s = _lib.load(), ctx.device, _stream_ptr(ctx.device)
    with pytest.raises(RuntimeError):
        vol.extract()
    with pytest.raises(RuntimeError):
        vol.integrate(None)                                    # the phase is checked before the render
    u, img, depth = maps[0]
    assert _call(vol, "bg_sparse_tsdf_integrate", u, img, depth) == _lib.BG_ERR_INVALID      # before the allocation
    for u, img, depth in maps:
        _lib.check(_call(vol, "bg_sparse_tsdf_mark", u, img, depth), "mark")
    n = vol.allocate()
    assert n > 0
    slots = vol.slots().copy()
    # marking after the allocation changes nothing
    u, img, depth = maps[1]
    assert _call(vol, "bg_sparse_tsdf_mark", u, img, depth) == _lib.BG_OK
    assert (vol.slots() == slots).all()
    with pytest.raises(RuntimeError):
        vol.allocate()
    with pytest.raises(RuntimeError):
        vol.mark(None)
    # a pool smaller than the allocation: the integration refuses and writes nothing
    g = vol.grid_struct()
    g.num_bricks = n - 1
    cam = _lib.camera_struct(u)
    ti = torch.from_numpy(np.ascontiguousarray(img, F)).to(dev)
    td = torch.from_numpy(np.ascontiguousarray(depth, F)).to(dev)
    assert lib.bg_sparse_tsdf_integrate(ctx.handle, s, C.byref(g), C.byref(cam), depth.shape[1], depth.shape[0], ti.data_ptr(),
                                        td.data_ptr(), 0.5) == _lib.BG_ERR_CAPACITY
    need = int(lib.bg_sparse_mesh_workspace_bytes(n - 1))
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    nv, nt = C.c_uint32(), C.c_uint32()
    assert lib.bg_sparse_mesh_count(ctx.handle, s, C.byref(g), ws.data_ptr(), need, C.byref(nv), C.byref(nt)) == _lib.BG_ERR_CAPACITY
    assert float(vol.weight.abs().sum()) == 0.0
    for u, img, depth in maps:
        vol_integrate_numpy(vol, u, img, depth)
    a, b = vol.extract(), vol.extract()
    assert a.to_ply() == b.to_ply() and len(a.faces) > 500
    # the capacity error of the emit writes nothing
    g = vol.grid_struct()
    need = int(lib.bg_sparse_mesh_workspace_bytes(n))
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    _lib.check(lib.bg_sparse_mesh_count(ctx.handle, s, C.byref(g), ws.data_ptr(), need, C.byref(nv), C.byref(nt)), "count")
    assert (nv.value, nt.value) == (len(a.vertices), len(a.faces))
    verts = torch.full((nv.value, 3), -7.0, device=dev)
    cols = torch.zeros((nv.value, 3), dtype=torch.uint8, device=dev)
    faces = torch.full((nt.value, 3), -1, dtype=torch.int32, device=dev)
    for mv, mt in ((nv.value - 1, nt.value), (nv.value, nt.value - 1)):
        assert lib.bg_sparse_mesh_emit(ctx.handle, s, C.byref(g), ws.data_ptr(), need, mv, mt, verts.data_ptr(), cols.data_ptr(),
                                       faces.data_ptr()) == _lib.BG_ERR_CAPACITY
    torch.cuda.synchronize()
    assert bool((verts == -7.0).all()) and bool((faces == -1).all())
    # an empty scene allocates nothing and extracts an empty mesh
    empty = SparseTsdfVolume.on_lattice(ctx, origin, h, dims, trunc)
    assert empty.allocate() == 0
    e = empty.extract()
    assert e.vertices.shape == (0, 3) and e.faces.shape == (0, 3)
    ctx.close()


def vol_integrate_numpy(vol, u, img, depth):
    from brush_b200 import _lib
    _lib.check(_call(vol, "bg_sparse_tsdf_integrate", u, img, depth), "integrate")


@pytest.mark.gpu
def test_fisheye_views_give_the_dense_mesh():
    import brush_b200.render as R
    from brush_b200.camera import KANNALA_BRANDT_4, THIN_PRISM_FISHEYE, Camera
    from test_gpu_mesh import _fisheye_maps
    dims = (64, 64, 64)
    lo, hi = -1.3, 1.3
    h = F((hi - lo) / (dims[0] - 1))
    origin = (F(lo),) * 3
    maps = []
    for i, pos in enumerate(sphere_views(24, radius=1.8)):
        if i % 2 == 0:
            cam = Camera(position=tuple(pos), rotation=look_at_quat(pos), fov_x=2.2, fov_y=2.2, camera_model=KANNALA_BRANDT_4,
                         model_params=(0.05, -0.01, 0.002, -0.0005))
        else:
            cam = Camera(position=tuple(pos), rotation=look_at_quat(pos), fov_x=2.2, fov_y=2.2,
                         camera_model=THIN_PRISM_FISHEYE, model_params=(0.05, -0.01, 0.002, -0.0005, 0.001, -0.001, 0.002, 0.001))
        maps.append(_fisheye_maps(cam, 192, 192))
    ctx = R.RenderContext(16, 192, 192)
    dense = _dense_from_maps(ctx, dims, origin, h, F(4 * h), maps)
    sparse = sparse_from_maps(ctx, dims, origin, h, F(4 * h), maps)
    md, ms = dense.extract(), sparse.extract()
    _same_mesh(ms, md)
    assert len(md.faces) > 1000
    print(f"fisheye: {sparse.num_bricks} of {int(np.prod(sr.brick_dims(dims)))} bricks allocated")
    ctx.close()


@pytest.mark.gpu
def test_splats_to_mesh_through_the_sparse_grid(tmp_path, monkeypatch):
    """test_gpu_mesh's 100k-splat sphere (40 views of 256x256, 128^3): splats_to_mesh on the sparse grid, forced by a
    dense grid that cannot be built, gives the dense path's mesh bit for bit."""
    import torch
    from PIL import Image
    import brush_b200.mesh as M
    import brush_b200.render as R
    import brush_b200.train as T
    from brush_b200.camera import Camera
    from brush_b200.dataset import SceneView
    from test_gpu_mesh import _sphere_splats
    n, size, res = 100_000, 256, 128
    t, sh, op = _sphere_splats(n)
    ctx = R.RenderContext(n, size, size)
    splats = T.Splats(*(torch.from_numpy(x).to(ctx.device) for x in (t, sh, op)))
    path = str(tmp_path / "blank.png")
    Image.fromarray(np.zeros((size, size, 3), np.uint8)).save(path)
    views = [SceneView(Camera(position=tuple(p), rotation=look_at_quat(p), fov_x=0.9, fov_y=0.9), path)
             for p in sphere_views(40)]
    dense = M.splats_to_mesh(ctx, splats, views, resolution=res)
    built = []

    class NoDense:
        def __init__(self, *a, **k):
            raise MemoryError("forced")

    real = M.SparseTsdfVolume

    class Recorded(real):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            built.append(self)

    monkeypatch.setattr(M, "TsdfVolume", NoDense)
    monkeypatch.setattr(M, "SparseTsdfVolume", Recorded)
    sparse = M.splats_to_mesh(ctx, splats, views, resolution=res)
    assert len(built) == 1 and built[0].num_bricks > 0
    _same_mesh(sparse, dense)
    nb = int(np.prod(built[0].brick_dims))
    print(f"splats_to_mesh: {len(dense.vertices)} vertices, {len(dense.faces)} faces; sparse grid {built[0].num_bricks} of "
          f"{nb} bricks")
    ctx.close()


def _trace_ball(cam_pos, rays, cam_z, center, radius, alpha=0.9):
    o = np.asarray(cam_pos, np.float64) - np.asarray(center, np.float64)
    d = rays / np.linalg.norm(rays, axis=-1, keepdims=True)
    b = d @ o
    disc = b * b - (o @ o - radius ** 2)
    hit = disc > 0
    t = -b - np.sqrt(np.where(hit, disc, 0.0))
    hit &= t > 0
    p = d * t[..., None]                                       # hit point relative to the camera
    zc = p @ np.asarray(cam_z, np.float64)
    col = np.clip(0.5 + 0.5 * (p + o) / radius, 0.0, 1.0)
    img = np.zeros(rays.shape[:2] + (4,), F)
    img[..., :3] = np.where(hit[..., None], alpha * col, 0.0)
    img[..., 3] = np.where(hit, alpha, 0.0)
    return img, np.where(hit, alpha * zc, 0.0).astype(F)


@pytest.mark.gpu
def test_lattice_past_the_dense_limit():
    """2048 x 2048 x 600 points (2.5e9 > 2^31) with h = 2^-9 and a dyadic origin, so every lattice coordinate is exact.
    A ball of radius 0.1 inside a brick-aligned 160^3 sub-box: the dense grid on the sub-box (origin shifted by whole
    bricks, hence the same coordinates) gives the expected mesh, and the sparse grid over the whole lattice equals it."""
    import brush_b200.render as R
    from brush_b200.camera import Camera, build_uniforms
    dims = (2048, 2048, 600)
    h = F(2.0 ** -9)
    origin = (F(-2.0), F(-2.0), F(-0.5))
    trunc = F(4 * h)
    sub_b = (150, 40, 30)                                      # first brick of the sub-box
    sub_dims = (160, 160, 160)
    sub_origin = tuple(F(origin[a] + F(sub_b[a] * 8) * h) for a in range(3))
    center = tuple(float(sub_origin[a]) + 80 * float(h) for a in range(3))
    assert int(np.prod(dims, dtype=np.int64)) > 2 ** 31
    size = 160
    maps = []
    for p in sphere_views(16, radius=0.45):
        pos = tuple(np.asarray(center) + p)
        cam = Camera(position=pos, rotation=look_at_quat(pos, center), fov_x=0.7, fov_y=0.7)
        u = build_uniforms(cam, size, size)
        xs, ys = np.meshgrid(np.arange(size) + 0.5, np.arange(size) + 0.5)
        dc = np.stack([(xs - u.cx) / u.fx, (ys - u.cy) / u.fy, np.ones_like(xs)], -1)
        r_w2c = np.asarray(u.viewmat, np.float64).reshape(4, 3)[:3].T
        img, depth = _trace_ball(pos, dc @ r_w2c, r_w2c[2], center, 0.1)
        maps.append((u, img, depth))
    ctx = R.RenderContext(16, size, size)
    dense = _dense_from_maps(ctx, sub_dims, sub_origin, h, trunc, maps).extract()
    sparse_vol = sparse_from_maps(ctx, dims, origin, h, trunc, maps)
    sparse = sparse_vol.extract()
    assert len(dense.faces) > 10_000
    _same_mesh(sparse, dense)
    nb = int(np.prod(sparse_vol.brick_dims))
    print(f"past the dense limit: {sparse_vol.num_bricks} of {nb} bricks allocated, {len(sparse.vertices)} vertices")
    ctx.close()


def test_no_spill_in_sparse_mesh_kernels():
    path = os.path.join(ROOT, "brush_b200", "csrc", "_obj", "mesh_sparse.o.ptxas.txt")
    if not os.path.exists(path):
        from brush_b200 import build
        build.build(force=True)
    txt = open(path).read()
    n = txt.count("Compiling entry function")
    spill = [ln for ln in txt.splitlines() if "spill" in ln]
    assert n == 14 and len(spill) == n
    assert all(ln.strip().startswith("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads") for ln in spill)
