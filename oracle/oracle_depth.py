"""ctypes wrapper around oracle/liborc_depth.so (orc_depth.c) -- TEST INFRASTRUCTURE ONLY.

The CPU oracle of the accumulated depth D = sum_i vis_i z_i (DESIGN.md section 4.6) and its joint colour + depth
adjoint, on top of the renders of oracle.oracle.  Like that module, only tests/ may import it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from . import oracle as orc

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liborc_depth.so")


def build(force: bool = False) -> str:
    """Compile oracle/liborc_depth.so with oracle/depth.mk (gcc, the flags of oracle/Makefile)."""
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".c", ".h")) or f in ("Makefile", "depth.mk")]
    stale = (not os.path.exists(_LIB_PATH)) or any(os.path.getmtime(s) > os.path.getmtime(_LIB_PATH) for s in srcs)
    if force or stale:
        subprocess.run(["make", "-C", _HERE, "-f", "depth.mk", "-B" if force else "-s", "liborc_depth.so"], check=True,
                       capture_output=True)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        L.orc_render_depth.argtypes = [C.POINTER(orc.OrcRender), C.c_void_p]
        L.orc_render_depth.restype = None
        L.orc_rasterize_backward_depth.argtypes = [C.POINTER(orc.OrcRender), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_int, C.c_void_p, C.c_void_p]
        L.orc_rasterize_backward_depth.restype = None
        _lib = L
    return _lib


def render_depth(res: orc.RenderResult):
    """Accumulated depth D = sum_i vis_i z_i [h,w] of a pass != forward render of oracle.render_forward."""
    assert res.rpass != orc.PASS_FORWARD
    out = np.zeros((res.h, res.w), np.float32)
    lib().orc_render_depth(res._handle, orc._ptr(out))
    return out


def rasterize_backward_depth(res: orc.RenderResult, v_output, v_depth, out_depth=None, smooth=None):
    """Joint colour + depth adjoint -> (v_combined [V,10], v_z [V]).  out_depth defaults to render_depth(res)."""
    v_output, v_depth = orc._f32(v_output), orc._f32(v_depth)
    assert v_output.shape == (res.h, res.w, 4) and v_depth.shape == (res.h, res.w)
    out_depth = orc._f32(render_depth(res) if out_depth is None else out_depth)
    if smooth is None:
        smooth = res.rpass == orc.PASS_BACKWARD_SMOOTH
    V = max(res.num_visible, 1)
    v_combined = np.zeros((V, 10), np.float32)
    v_z = np.zeros((V,), np.float32)
    lib().orc_rasterize_backward_depth(res._handle, orc._ptr(res._bg), orc._ptr(v_output), orc._ptr(out_depth),
                                       orc._ptr(v_depth), int(bool(smooth)), orc._ptr(v_combined), orc._ptr(v_z))
    return v_combined[: res.num_visible], v_z[: res.num_visible]


def project_backward_depth(res: orc.RenderResult, v_combined, v_z):
    """oracle.project_backward, then v_transforms[gid, 0:3] += v_z[cgid] * R[2,:] (z = R[2,:] . mean + t_z), in f32 with
    the product and the sum rounded separately; rows with v_z == 0 are left as they are."""
    v_t, v_sh, v_o, v_r = orc.project_backward(res, v_combined)
    row = np.array([res._cam.viewmat[2], res._cam.viewmat[5], res._cam.viewmat[8]], np.float32)
    v_z = orc._f32(v_z)[: res.num_visible]
    nz = np.nonzero(v_z)[0]
    gid = res.gid_from_cgid[nz].astype(np.int64)
    v_t[gid, 0:3] = v_t[gid, 0:3] + v_z[nz, None] * row[None, :]
    return v_t, v_sh, v_o, v_r
