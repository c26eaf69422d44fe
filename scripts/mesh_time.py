"""Timing of the mesh export (development aid, not the bench): n flat opaque splats on the unit sphere coloured by position,
`views` views around it at w x h, a res^3 TSDF grid.  CUDA events around each stage: the depth render and the integration
of every view, then bg_mesh_count and bg_mesh_emit, and the wall time of the PLY write.  Also the updated lattice points
per view (the total weight over the views), the mesh size, and the bytes each stage must move against the H100's
3.35 TB/s data-sheet rate.  Prints one JSON line with the card and its power limit.
Usage: mesh_time.py [n] [views] [w] [h] [res]"""
import ctypes as C
import json
import math
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import brush_b200.render as R
from brush_b200 import _lib
from brush_b200.camera import Camera
from brush_b200.mesh import TsdfVolume, TriangleMesh
from brush_b200.render import PASS_BACKWARD, _stream_ptr

n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
views = int(sys.argv[2]) if len(sys.argv) > 2 else 200
w = int(sys.argv[3]) if len(sys.argv) > 3 else 1920
h = int(sys.argv[4]) if len(sys.argv) > 4 else 1080
res = int(sys.argv[5]) if len(sys.argv) > 5 else 512
HBM = 3.35e12
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()


def fib(count, radius):
    i = np.arange(count) + 0.5
    phi = np.arccos(1 - 2 * i / count)
    th = math.pi * (1 + 5 ** 0.5) * i
    return np.stack([np.cos(th) * np.sin(phi), np.cos(phi), np.sin(th) * np.sin(phi)], 1) * radius


def look_at(pos):
    z = -pos / np.linalg.norm(pos)
    a = np.array([0.0, 1.0, 0.0]) if abs(z[1]) < 0.9 else np.array([1.0, 0.0, 0.0])
    x = np.cross(a, z); x /= np.linalg.norm(x)
    y = np.cross(z, x)
    m = np.stack([x, y, z], 1)
    from scipy.spatial.transform import Rotation
    return tuple(Rotation.from_matrix(m).as_quat())          # x, y, z, w


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
    t[:, 7:9] = math.log(0.8 * math.sqrt(4 * math.pi / count))
    t[:, 9] = math.log(1e-4)
    sh = ((np.clip(0.5 + 0.5 * p, 0, 1) - 0.5) / 0.2820947917738781).astype(np.float32)[:, None, :]
    op = np.full(count, 6.0, np.float32)
    return [torch.from_numpy(x).to(dev) for x in (t, sh, op)]


ctx = R.RenderContext(n, w, h)
dev = ctx.device
t, sh, op = sphere_splats(n, dev)
cams = [Camera(position=tuple(p), rotation=look_at(p), fov_x=0.9, fov_y=0.9 * h / w) for p in fib(views, 3.0)]
vol = TsdfVolume(ctx, (-1.2, -1.2, -1.2), (1.2, 1.2, 1.2), res)
npts = vol.dims[0] * vol.dims[1] * vol.dims[2]
for c in cams[:3]:                                           # warm-up (the grid is re-zeroed below)
    vol.integrate(R.render_splats(ctx, c, (w, h), t, sh, op, background=(0.0, 0.0, 0.0), rpass=PASS_BACKWARD, render_depth=True))
for x in (vol.tsdf, vol.weight, vol.rgb):
    x.zero_()
torch.cuda.synchronize()
ev = lambda: torch.cuda.Event(enable_timing=True)
render_ms, integ_ms = [], []
for c in cams:
    e0, e1, e2 = ev(), ev(), ev()
    e0.record()
    out = R.render_splats(ctx, c, (w, h), t, sh, op, background=(0.0, 0.0, 0.0), rpass=PASS_BACKWARD, render_depth=True)
    e1.record()
    vol.integrate(out)
    e2.record()
    e2.synchronize()
    render_ms.append(e0.elapsed_time(e1))
    integ_ms.append(e1.elapsed_time(e2))
updated = float(vol.weight.double().sum().item()) / views

lib = _lib.load()
g = vol.grid_struct()
need = int(lib.bg_mesh_workspace_bytes(*vol.dims))
ws = torch.empty(need, dtype=torch.uint8, device=dev)
s = _stream_ptr(dev)
nv, nt = C.c_uint32(), C.c_uint32()
count_ms, emit_ms = [], []
for rep in range(4):                                         # the first round warms up
    torch.cuda.synchronize()
    e0, e1 = ev(), ev()
    e0.record()
    _lib.check(lib.bg_mesh_count(ctx.handle, s, C.byref(g), ws.data_ptr(), need, C.byref(nv), C.byref(nt)), "count")
    e1.record()
    e1.synchronize()
    verts = torch.empty((nv.value, 3), dtype=torch.float32, device=dev)
    cols = torch.empty((nv.value, 3), dtype=torch.uint8, device=dev)
    faces = torch.empty((nt.value, 3), dtype=torch.int32, device=dev)
    e2, e3 = ev(), ev()
    e2.record()
    _lib.check(lib.bg_mesh_emit(ctx.handle, s, C.byref(g), ws.data_ptr(), need, nv.value, nt.value, verts.data_ptr(),
                                cols.data_ptr(), faces.data_ptr()), "emit")
    e3.record()
    e3.synchronize()
    if rep:
        count_ms.append(e0.elapsed_time(e1))
        emit_ms.append(e2.elapsed_time(e3))
mesh = TriangleMesh(verts.cpu().numpy(), cols.cpu().numpy(), faces.cpu().numpy())
with tempfile.TemporaryDirectory() as d:
    t0 = time.perf_counter()
    data = mesh.to_ply()
    with open(os.path.join(d, "mesh.ply"), "wb") as f:
        f.write(data)
    ply_s = time.perf_counter() - t0

V, Fc = nv.value, nt.value
# bytes each stage must move: integration reads and writes the 20-byte point and reads its 20 bytes of pixel per update;
# count reads tsdf + weight once; emit reads them twice (vertex and face pass), writes / reads the 5-byte per-point base
# and mask, and writes 15 bytes per vertex and 12 per face
b_int = updated * 60
b_count = npts * 8
b_emit = npts * (16 + 10) + V * 15 + Fc * 12
integ = float(np.median(integ_ms))
rec = {"n": n, "views": views, "w": w, "h": h, "dims": list(vol.dims), "grid_points": npts,
       "render_ms_median": float(np.median(render_ms)), "integrate_ms_median": integ,
       "integrate_ms_total": float(np.sum(integ_ms)), "render_ms_total": float(np.sum(render_ms)),
       "updated_points_per_view": updated, "lattice_points_per_s": npts / integ * 1e3,
       "integrate_GBps": b_int / integ / 1e6, "count_ms": float(np.median(count_ms)), "emit_ms": float(np.median(emit_ms)),
       "count_GBps": b_count / np.median(count_ms) / 1e6, "emit_GBps": b_emit / np.median(emit_ms) / 1e6,
       "vertices": V, "triangles": Fc, "ply_write_s": ply_s, "ply_bytes": len(data),
       "hbm_datasheet_GBps": HBM / 1e9, "card": smi}
print(json.dumps(rec), flush=True)
ctx.close()
