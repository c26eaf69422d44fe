"""numpy f32 restatement of the compressed PLY encoding (DESIGN.md section 4.8) for the tests: the device call must
produce the same chunks, words, SH bytes, order and count, bit for bit.  The sigmoid goes through the oracle's
deterministic exp (orc_expf), so the alpha byte is exact as well."""
from __future__ import annotations

import numpy as np

from brush_b200 import ply
from oracle import oracle as orc

F = np.float32
DROPPED_KEY = 1 << 30
_OTHERS = np.array([[1, 2, 3], [0, 2, 3], [0, 1, 3], [0, 1, 2]])   # the three stored components, by `largest`


def det_sigmoid(x):
    """1 / (1 + orc_expf(-x)) in f32, one oracle call per distinct value."""
    x = np.asarray(x, np.float32).reshape(-1)
    u, inv = np.unique(x, return_inverse=True)
    e = np.array([orc.expf_det(float(-v)) for v in u], np.float32)
    return (F(1.0) / (F(1.0) + e))[inv]


def _quat_norm2(q):
    return ((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]) + q[:, 3] * q[:, 3]


def kept_rows(transforms, sh, raw_opac):
    n = transforms.shape[0]
    with np.errstate(all="ignore"):
        q2 = _quat_norm2(transforms[:, 3:7])
    return (np.isfinite(transforms).all(1) & np.isfinite(sh.reshape(n, -1)).all(1) & np.isfinite(raw_opac) & (q2 != 0))


def _spread3(v):
    v = v.astype(np.uint64) & 0x3FF
    out = np.zeros_like(v)
    for b in range(10):
        out |= ((v >> b) & 1) << (3 * b)
    return out


def _morton_cell(x, lo, hi):
    with np.errstate(all="ignore"):
        v = ((x - lo) / (hi - lo)) * F(1024.0)
        q = np.where(v >= F(1023.0), F(1023.0), np.where(v >= F(1.0), v, F(0.0)))
    return np.where(hi == lo, 0, q.astype(np.uint32))


def morton_keys(transforms, keep):
    """u32 keys: x in bit 3i+2, y in 3i+1, z in 3i over the kept means' bounds; dropped rows DROPPED_KEY."""
    n = transforms.shape[0]
    keys = np.full(n, DROPPED_KEY, np.uint64)
    if keep.any():
        means = transforms[keep, 0:3] + F(0.0)
        lo, hi = means.min(0), means.max(0)
        k = np.zeros(int(keep.sum()), np.uint64)
        for a in range(3):
            k |= _spread3(_morton_cell(means[:, a], lo[a], hi[a])) << (2 - a)
        keys[keep] = k
    return keys.astype(np.uint32)


def _unorm(v, lo, hi, maxq):
    with np.errstate(all="ignore"):
        r = np.rint(((v - lo) / (hi - lo)) * F(maxq))
        r = np.fmin(np.fmax(r, F(0.0)), F(maxq))
    return np.where(hi == lo, 0, r).astype(np.uint32)


def _clamp_rint(x, lo, hi):
    return np.fmin(np.fmax(np.rint(x), F(lo)), F(hi)).astype(np.uint32)


def encode(transforms, sh, raw_opac):
    """dict(m, keys [n], order [m], chunks [ceil(m/256), 18] f32, packed [m, 4] u32, sh [m, 3(K-1)] u8 or None)."""
    t = np.ascontiguousarray(transforms, np.float32)
    shc = np.ascontiguousarray(sh, np.float32)
    op = np.ascontiguousarray(raw_opac, np.float32)
    n, k = shc.shape[0], shc.shape[1]
    keep = kept_rows(t, shc, op)
    keys = morton_keys(t, keep)
    m = int(keep.sum())
    order = np.argsort(keys, kind="stable")[:m]
    t, shc, op = t[order], shc[order], op[order]
    with np.errstate(all="ignore"):
        v = np.concatenate([t[:, 0:3] + F(0.0), t[:, 7:10] + F(0.0), shc[:, 0, :] * F(ply.SH_C0) + F(0.5)], 1)   # [m, 9]
    n_chunks = (m + 255) // 256
    pad = np.full((n_chunks * 256 - m, 9), np.nan, np.float32)
    vp = np.concatenate([v, pad]).reshape(n_chunks, 256, 9)
    lo, hi = np.nanmin(vp, 1) if m else np.zeros((0, 9), F), np.nanmax(vp, 1) if m else np.zeros((0, 9), F)
    chunks = np.stack([lo, hi], 2).reshape(n_chunks, 18)
    c = np.arange(m) // 256
    bits = [2047.0, 1023.0, 2047.0] * 2 + [255.0] * 3
    q = [_unorm(v[:, f], lo[c, f], hi[c, f], bits[f]) for f in range(9)]
    pos = q[0] << 21 | q[1] << 11 | q[2]
    scl = q[3] << 21 | q[4] << 11 | q[5]
    alpha = _clamp_rint(det_sigmoid(op) * F(255.0), 1.0, 254.0)
    col = q[6] << 24 | q[7] << 16 | q[8] << 8 | alpha
    quat = t[:, 3:7]
    with np.errstate(all="ignore"):
        rn = np.maximum(np.sqrt(_quat_norm2(quat)), F(1e-12))
        qn = quat / rn[:, None]
    largest = np.argmax(np.abs(qn), 1)
    qn = np.where((qn[np.arange(m), largest] < 0)[:, None], -qn, qn)
    abc = np.take_along_axis(qn, _OTHERS[largest], 1)
    w = _clamp_rint((abc * (F(0.5) * F(np.sqrt(2.0))) + F(0.5)) * F(1023.0), 0.0, 1023.0)
    rot = largest.astype(np.uint32) << 30 | w[:, 0] << 20 | w[:, 1] << 10 | w[:, 2]
    packed = np.stack([pos, rot, scl, col], 1).astype(np.uint32)
    sh_bytes = None
    if k > 1:
        rest = shc[:, 1:, :].transpose(0, 2, 1).reshape(m, 3 * (k - 1))
        sh_bytes = _clamp_rint((rest * F(0.125) + F(0.5)) * F(254.0), 0.0, 255.0).astype(np.uint8)
    return dict(m=m, keys=keys, order=order, chunks=chunks.astype(np.float32), packed=packed, sh=sh_bytes)


def encode_file(transforms, sh, raw_opac, up_axis=None, render_mip=False) -> bytes:
    e = encode(transforms, sh, raw_opac)
    degree = ply.sh_degree_from_coeffs(np.asarray(sh).shape[1])
    return ply.compressed_ply_bytes(e["chunks"], e["packed"], e["sh"], e["m"], ply.export_comments(degree, up_axis, render_mip))
