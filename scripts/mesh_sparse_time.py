"""Timing of the sparse brick TSDF (development aid, not the bench), on mesh_time.py's scene: n flat opaque splats on the
unit sphere coloured by position, `views` views around it at w x h.  At `res` (512) the dense and the sparse export run
alternately in the same process (two rounds each, the second reported) and their meshes are compared byte for byte; at
`big_res` (2048), where the dense grid cannot exist, the sparse export runs alone.  CUDA events around every stage:
the marking pass (render + bg_sparse_tsdf_mark per view), bg_sparse_tsdf_allocate (with its readback), the integration
pass (render + integrate per view), bg_*mesh_count and bg_*mesh_emit.  Prints one JSON line with the card and its power
limit.
Usage: mesh_sparse_time.py [n] [views] [w] [h] [res] [big_res]"""
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import brush_b200.render as R
from brush_b200 import _lib
from brush_b200.camera import Camera
from brush_b200.mesh import SparseTsdfVolume, TriangleMesh, TsdfVolume
from brush_b200.render import PASS_BACKWARD, _stream_ptr

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
views = int(sys.argv[2]) if len(sys.argv) > 2 else 200
w = int(sys.argv[3]) if len(sys.argv) > 3 else 1920
h = int(sys.argv[4]) if len(sys.argv) > 4 else 1080
res = int(sys.argv[5]) if len(sys.argv) > 5 else 512
big_res = int(sys.argv[6]) if len(sys.argv) > 6 else 2048
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()


def fib(count, radius):
    i = np.arange(count) + 0.5
    phi = np.arccos(1 - 2 * i / count)
    th = np.pi * (1 + 5 ** 0.5) * i
    return np.stack([np.cos(th) * np.sin(phi), np.cos(phi), np.sin(th) * np.sin(phi)], 1) * radius


def look_at(pos):
    z = -pos / np.linalg.norm(pos)
    a = np.array([0.0, 1.0, 0.0]) if abs(z[1]) < 0.9 else np.array([1.0, 0.0, 0.0])
    x = np.cross(a, z); x /= np.linalg.norm(x)
    y = np.cross(z, x)
    from scipy.spatial.transform import Rotation
    return tuple(Rotation.from_matrix(np.stack([x, y, z], 1)).as_quat())


def sphere_splats(count, dev):
    p = fib(count, 1.0)
    t = np.zeros((count, 10), np.float32)
    t[:, :3] = p
    ax = np.cross([0.0, 0.0, 1.0], p)
    s = np.linalg.norm(ax, axis=1, keepdims=True)
    ang = np.arctan2(s[:, 0], p[:, 2])
    ax = np.where(s > 1e-9, ax / np.maximum(s, 1e-12), [1.0, 0.0, 0.0])
    t[:, 3] = np.cos(ang / 2)
    t[:, 4:7] = ax * np.sin(ang / 2)[:, None]
    t[:, 7:9] = np.log(0.8 * np.sqrt(4 * np.pi / count))
    t[:, 9] = np.log(1e-4)
    sh = ((np.clip(0.5 + 0.5 * p, 0, 1) - 0.5) / 0.2820947917738781).astype(np.float32)[:, None, :]
    op = np.full(count, 6.0, np.float32)
    return [torch.from_numpy(x).to(dev) for x in (t, sh, op)]


ctx = R.RenderContext(n, w, h)
dev = ctx.device
lib = _lib.load()
s = _stream_ptr(dev)
t, sh, op = sphere_splats(n, dev)
cams = [Camera(position=tuple(p), rotation=look_at(p), fov_x=0.9, fov_y=0.9 * h / w) for p in fib(views, 3.0)]
LO, HI = (-1.2, -1.2, -1.2), (1.2, 1.2, 1.2)
ev = lambda: torch.cuda.Event(enable_timing=True)


def render(c):
    return R.render_splats(ctx, c, (w, h), t, sh, op, background=(0.0, 0.0, 0.0), rpass=PASS_BACKWARD, render_depth=True)


def view_pass(step):
    """Renders every view and applies `step`; (render ms, step ms) summed over the views, CUDA events per view."""
    r_ms = s_ms = 0.0
    for c in cams:
        e0, e1, e2 = ev(), ev(), ev()
        e0.record()
        out = render(c)
        e1.record()
        step(out)
        e2.record()
        e2.synchronize()
        r_ms += e0.elapsed_time(e1)
        s_ms += e1.elapsed_time(e2)
    return r_ms, s_ms


def timed_extract(count, emit, g, need):
    ws = torch.empty(need, dtype=torch.uint8, device=dev)
    nv, nt = C.c_uint32(), C.c_uint32()
    torch.cuda.synchronize()
    e0, e1 = ev(), ev()
    e0.record()
    _lib.check(count(ctx.handle, s, C.byref(g), ws.data_ptr(), need, C.byref(nv), C.byref(nt)), "count")
    e1.record()
    e1.synchronize()
    verts = torch.empty((nv.value, 3), dtype=torch.float32, device=dev)
    cols = torch.empty((nv.value, 3), dtype=torch.uint8, device=dev)
    faces = torch.empty((nt.value, 3), dtype=torch.int32, device=dev)
    e2, e3 = ev(), ev()
    e2.record()
    _lib.check(emit(ctx.handle, s, C.byref(g), ws.data_ptr(), need, nv.value, nt.value, verts.data_ptr(), cols.data_ptr(),
                    faces.data_ptr()), "emit")
    e3.record()
    e3.synchronize()
    mesh = TriangleMesh(verts.cpu().numpy(), cols.cpu().numpy(), faces.cpu().numpy())
    return mesh, e0.elapsed_time(e1), e2.elapsed_time(e3)


def dense_export(r):
    vol = TsdfVolume(ctx, LO, HI, r)
    render_ms, integ_ms = view_pass(vol.integrate)
    mesh, count_ms, emit_ms = timed_extract(lib.bg_mesh_count, lib.bg_mesh_emit, vol.grid_struct(),
                                            int(lib.bg_mesh_workspace_bytes(*vol.dims)))
    rec = {"dims": list(vol.dims), "render_ms": render_ms, "integrate_ms": integ_ms, "count_ms": count_ms, "emit_ms": emit_ms,
           "grid_bytes": int(np.prod(vol.dims, dtype=np.int64)) * 20}
    del vol
    return mesh, rec


def sparse_export(r):
    vol = SparseTsdfVolume(ctx, LO, HI, r)
    mark_render_ms, mark_ms = view_pass(vol.mark)
    torch.cuda.synchronize()
    e0, e1 = ev(), ev()
    e0.record()
    nb = vol.allocate()
    e1.record()
    e1.synchronize()
    alloc_ms = e0.elapsed_time(e1)                      # includes the zeroing of the pool
    render_ms, integ_ms = view_pass(vol.integrate)
    mesh, count_ms, emit_ms = timed_extract(lib.bg_sparse_mesh_count, lib.bg_sparse_mesh_emit, vol.grid_struct(),
                                            int(lib.bg_sparse_mesh_workspace_bytes(nb)))
    total_bricks = int(np.prod(vol.brick_dims, dtype=np.int64))
    rec = {"dims": list(vol.dims), "bricks": total_bricks, "allocated_bricks": nb, "allocated_fraction": nb / total_bricks,
           "pool_bytes": nb * 512 * 20, "brick_map_bytes": total_bricks * 4, "workspace_bytes": int(vol.workspace.numel()),
           "mark_render_ms": mark_render_ms, "mark_ms": mark_ms, "allocate_ms": alloc_ms, "render_ms": render_ms,
           "integrate_ms": integ_ms, "count_ms": count_ms, "emit_ms": emit_ms}
    del vol
    return mesh, rec


for c in cams[:3]:                                        # warm-up of the render path
    render(c)
rounds = []
for rep in range(2):
    md, rd = dense_export(res)
    torch.cuda.empty_cache()
    ms, rs = sparse_export(res)
    torch.cuda.empty_cache()
    same = md.to_ply() == ms.to_ply()
    rounds.append({"dense": rd, "sparse": rs, "same_mesh": same, "vertices": len(md.vertices), "triangles": len(md.faces)})
    assert same, "the sparse mesh differs from the dense mesh"
mb, rb = sparse_export(big_res)
rec = {"n": n, "views": views, "w": w, "h": h, "res": res, "at_res": rounds[-1], "all_rounds_equal": all(r["same_mesh"] for r in rounds),
       "big_res": big_res, "at_big_res": dict(rb, vertices=len(mb.vertices), triangles=len(mb.faces)), "card": smi}
print(json.dumps(rec), flush=True)
ctx.close()
