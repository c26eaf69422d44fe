"""On-disk Gaussian PLY (the INRIA 3DGS layout the reference reads and writes), host side.

  splat_to_ply      <- brush-serde/src/export.rs:82-206 (field order :50-75, SH permuted [N,K,3] -> channel-major
                       f_rest_*, quaternion normalised on export, min-scale floor baked, comments :188-196)
  load_splat_from_ply <- brush-serde/src/import.rs:176-400 (plain PLY: ascii or binary, optional scale / rot /
                       opacity / f_dc / f_rest / rgb properties, subsampling, up-axis and render-mode comments)
  SplatData.subsample / into_splats <- import.rs:40-103 (defaults for missing fields)

  _load_compressed_ply <- import.rs:408-600, ply_gaussian.rs:23-34,102-122, quant.rs:1-71: the SuperSplat compressed
                       variant (per-256-splat quantisation ranges in a leading `chunk` element, 11/10/11-bit positions and
                       scales, smallest-three quaternions, 8-bit colour + opacity, optional 8-bit higher SH bands)
  compressed_ply_bytes <- no reference writer: the same layout from an encoding made on the device
                       (compress.splat_to_compressed_ply, DESIGN.md section 4.8)

Storage format, not part of the per-step hot path: numpy on the host, one pass.
"""
from __future__ import annotations

import io
import math
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np

SH_C0 = 0.2820947917738781  # shaders::SH_C0

_PLY_DTYPES = {
    "char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2", "uint16": "u2",
    "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4", "double": "f8", "float64": "f8",
}


def sh_coeffs_for_degree(degree: int) -> int:
    return (degree + 1) ** 2


def sh_degree_from_coeffs(k: int) -> int:
    deg = {1: 0, 4: 1, 9: 2, 16: 3, 25: 4}.get(int(k))
    if deg is None:
        raise ValueError(f"Invalid nr. of sh bases {k}")
    return deg


def splat_to_ply(transforms: np.ndarray, sh_coeffs: np.ndarray, raw_opacities: np.ndarray, up_axis=None,
                 render_mip: bool = False) -> bytes:
    """export.rs:176-206.  transforms [N,10] (means, quat wxyz, log scales), sh_coeffs [N,K,3], raw_opacities [N];
    a min-scale floor must already be baked in (Splats.bake_min_scale)."""
    t = np.ascontiguousarray(transforms, np.float32)
    sh = np.ascontiguousarray(sh_coeffs, np.float32)
    op = np.ascontiguousarray(raw_opacities, np.float32)
    n, k = sh.shape[0], sh.shape[1]
    degree = sh_degree_from_coeffs(k)
    rest = k - 1
    names = ["x", "y", "z", "scale_0", "scale_1", "scale_2", "opacity", "rot_0", "rot_1", "rot_2", "rot_3",
             "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(3 * rest)]
    out = np.empty((n, len(names)), np.float32)
    out[:, 0:3] = t[:, 0:3]
    out[:, 3:6] = t[:, 7:10]
    out[:, 6] = op
    q = t[:, 3:7]
    rn = np.maximum(np.sqrt((q * q).sum(1, dtype=np.float32)), np.float32(1e-12))
    out[:, 7:11] = q / rn[:, None]
    chan_major = sh.transpose(0, 2, 1)                      # [N, 3, K] (export.rs:87)
    out[:, 11:14] = chan_major[:, :, 0]
    if rest:
        out[:, 14:] = chan_major[:, :, 1:].reshape(n, 3 * rest)
    comments = export_comments(degree, up_axis, render_mip)
    head = ["ply", "format binary_little_endian 1.0"] + [f"comment {c}" for c in comments] + [f"element vertex {n}"]
    head += [f"property float {nm}" for nm in names] + ["end_header"]
    return ("\n".join(head) + "\n").encode("ascii") + out.astype("<f4").tobytes()


def export_comments(degree: int, up_axis=None, render_mip: bool = False):
    """The header comments of an exported file (export.rs:188-196)."""
    comments = ["Exported from Brush"]
    if up_axis is not None:
        comments.append("Vertical axis: {} {} {}".format(*[_fmt_f32(v) for v in up_axis]))
    else:
        comments.append("Vertical axis: y")
    comments.append(f"SH degree: {degree}")
    comments.append("SplatRenderMode: " + ("mip" if render_mip else "default"))
    return comments


def _fmt_f32(v) -> str:
    f = float(np.float32(v))
    return str(int(f)) if f == int(f) and abs(f) < 1e15 else repr(f)


@dataclass
class ParseMetadata:
    up_axis: Optional[Tuple[float, float, float]]
    render_mip: Optional[bool]
    total_splats: int


@dataclass
class SplatData:
    """import.rs:27-103: only the means are guaranteed."""
    means: np.ndarray                      # [N,3]
    rotations: Optional[np.ndarray] = None   # [N,4] wxyz
    log_scales: Optional[np.ndarray] = None  # [N,3]
    sh_coeffs: Optional[np.ndarray] = None   # [N,K,3]
    raw_opacities: Optional[np.ndarray] = None

    def num_splats(self) -> int:
        return int(self.means.shape[0])

    def subsample(self, max_splats: int) -> "SplatData":
        n = self.num_splats()
        if max_splats == 0 or n <= max_splats:
            return self
        step = -(-n // max_splats)
        pick = lambda a: None if a is None else a[::step].copy()
        return SplatData(pick(self.means), pick(self.rotations), pick(self.log_scales), pick(self.sh_coeffs),
                         pick(self.raw_opacities))

    def into_arrays(self):
        """into_splats (import.rs:80-103): (transforms [N,10], sh [N,K,3], raw_opac [N]) with the reference defaults."""
        n = self.num_splats()
        rot = self.rotations if self.rotations is not None else np.tile(np.array([1, 0, 0, 0], np.float32), (n, 1))
        ls = self.log_scales if self.log_scales is not None else np.full((n, 3), -4.0, np.float32)
        sh = self.sh_coeffs if self.sh_coeffs is not None else np.full((n, 1, 3), 0.5, np.float32)
        op = self.raw_opacities if self.raw_opacities is not None else np.zeros(n, np.float32)  # inverse_sigmoid(0.5)
        t = np.concatenate([self.means, rot, ls], 1).astype(np.float32)
        return np.ascontiguousarray(t), np.ascontiguousarray(sh, np.float32), np.ascontiguousarray(op, np.float32)


def _parse_header(buf: bytes):
    end = buf.find(b"end_header")
    if not buf.startswith(b"ply") or end < 0:
        raise ValueError("missing PLY header")
    nl = buf.index(b"\n", end) + 1
    lines = buf[:nl].decode("ascii", "replace").splitlines()
    fmt, comments, elements = None, [], []
    for ln in lines[1:]:
        p = ln.strip().split()
        if not p:
            continue
        if p[0] == "format":
            fmt = p[1]
        elif p[0] == "comment":
            comments.append(ln.strip()[len("comment"):].strip())
        elif p[0] == "element":
            elements.append((p[1], int(p[2]), []))
        elif p[0] == "property":
            if p[1] == "list":
                raise ValueError("list properties are not supported in a splat PLY")
            elements[-1][2].append((p[2], p[1]))
    return fmt, comments, elements, nl


def _up_axis(comments):
    """import.rs:194-222: last matching comment wins."""
    up = None
    for c in comments:
        s = c.lower()
        if not s.startswith("vertical axis: "):
            continue
        suf = s[len("vertical axis: "):].strip()
        if suf == "x":
            up = (1.0, 0.0, 0.0)
        elif suf == "y":
            up = (0.0, -1.0, 0.0)
        elif suf == "z":
            up = (0.0, 0.0, -1.0)
        else:
            parts = []
            for tok in suf.replace(",", " ").replace("[", " ").replace("]", " ").split():
                try:
                    parts.append(float(tok))
                except ValueError:
                    pass
            if len(parts) == 3:
                up = tuple(parts)
    return up


def _render_mode(comments):
    mode = None
    for c in comments:
        s = c.lower()
        if s.startswith("splatrendermode: "):
            v = s[len("splatrendermode: "):].strip()
            if v == "mip":
                mode = True
            elif v == "default":
                mode = False
    return mode


def load_splat_from_ply(data: bytes, subsample_points: Optional[int] = None):
    """Returns (SplatData, ParseMetadata).  import.rs:176-400."""
    fmt, comments, elements, off = _parse_header(data)
    if not elements or not any(e[0] == "vertex" for e in elements):
        raise ValueError("Unknown format")
    if elements[0][0] == "chunk":                       # PlyFormat::SuperSplatCompressed (import.rs:243-250)
        return _load_compressed_ply(data, fmt, comments, elements, off, max(int(subsample_points or 1), 1))
    cols = None
    for name, count, props in elements:
        if fmt == "ascii":
            if name == "vertex":
                txt = data[off:].decode("ascii").split("\n")
                rows = [ln.split() for ln in txt[:count]]
                cols = {p[0]: np.array([r[i] for r in rows], dtype=np.float64).astype(_PLY_DTYPES[p[1]]) for i, p in enumerate(props)}
                break
            off = _skip_ascii(data, off, count)
        else:
            end = "<" if fmt == "binary_little_endian" else ">"
            dt = np.dtype([(p[0], end + _PLY_DTYPES[p[1]]) for p in props])
            if name == "vertex":
                arr = np.frombuffer(data, dtype=dt, count=count, offset=off)
                cols = {p[0]: arr[p[0]] for p in props}
                break
            off += dt.itemsize * count
    total = len(next(iter(cols.values()))) if cols else 0
    sub = max(int(subsample_points or 1), 1)
    sel = slice(sub - 1, None, sub)                    # row_index is 1-based: keep multiples of `subsample`
    f32 = lambda nm: np.asarray(cols[nm][sel], np.float32) if nm in cols else None
    n = len(cols["x"][sel])
    means = np.stack([f32("x"), f32("y"), f32("z")], 1)

    def colour(nm, alias):
        key = nm if nm in cols else (alias if alias in cols else None)
        if key is None:
            return None
        a = cols[key][sel]
        if a.dtype == np.uint8:
            return a.astype(np.float32) / np.float32(254.0)       # de_quant: value / (u8::MAX - 1)
        if a.dtype == np.uint16:
            return a.astype(np.float32) / np.float32(65534.0)
        return a.astype(np.float32)

    r, g, b = colour("red", "r"), colour("green", "g"), colour("blue", "b")
    rest_names = sorted((nm for nm in cols if nm.startswith("f_rest_")), key=lambda s: int(s[7:]))
    sh_count = len(rest_names) + sum(nm in cols for nm in ("f_dc_0", "f_dc_1", "f_dc_2")) \
        + sum(nm in cols for nm in ("r", "g", "b", "red", "green", "blue"))
    sh = None
    if sh_count > 0:
        zeros = np.zeros(n, np.float32)
        dc = [f32(f"f_dc_{i}") if f"f_dc_{i}" in cols else zeros for i in range(3)]
        if r is not None and g is not None and b is not None:   # prefer rgb if specified (import.rs:353-362)
            dc = [(c - np.float32(0.5)) / np.float32(SH_C0) for c in (r, g, b)]
        n_rest = sh_count - 3
        rest = np.zeros((n, max(n_rest, 0)), np.float32)
        for i, nm in enumerate(rest_names[:max(n_rest, 0)]):
            rest[:, i] = f32(nm)
        per = n_rest // 3 if n_rest > 0 else 0
        sh = np.empty((n, 1 + per, 3), np.float32)
        sh[:, 0, :] = np.stack(dc, 1)
        if per:
            sh[:, 1:, :] = rest[:, :3 * per].reshape(n, 3, per).transpose(0, 2, 1)   # interleave_coeffs
    d = SplatData(
        means=means,
        rotations=np.stack([f32(f"rot_{i}") for i in range(4)], 1) if "rot_0" in cols else None,
        log_scales=np.stack([f32(f"scale_{i}") for i in range(3)], 1) if "scale_0" in cols else None,
        sh_coeffs=sh,
        raw_opacities=f32("opacity") if "opacity" in cols else None,
    )
    return d, ParseMetadata(up_axis=_up_axis(comments), render_mip=_render_mode(comments), total_splats=total // sub)


def _skip_ascii(data: bytes, off: int, lines: int) -> int:
    for _ in range(lines):
        off = data.index(b"\n", off) + 1
    return off


# ---------------------------------------------------------------------------------------------- SuperSplat compressed PLY
_QUANT_META_FIELDS = ("min_x", "max_x", "min_y", "max_y", "min_z", "max_z", "min_scale_x", "max_scale_x", "min_scale_y",
                      "max_scale_y", "min_scale_z", "max_scale_z", "min_r", "max_r", "min_g", "max_g", "min_b", "max_b")


def _read_element(data: bytes, fmt: str, off: int, count: int, props):
    """One PLY element as {property: column}; returns (columns, offset behind the element)."""
    if fmt == "ascii":
        end = _skip_ascii(data, off, count)
        rows = [ln.split() for ln in data[off:end].decode("ascii").split("\n")[:count]]
        cols = {p[0]: np.array([r[i] for r in rows], dtype=np.float64).astype(_PLY_DTYPES[p[1]]) for i, p in enumerate(props)}
        return cols, end
    e = "<" if fmt == "binary_little_endian" else ">"
    dt = np.dtype([(p[0], e + _PLY_DTYPES[p[1]]) for p in props])
    if off + dt.itemsize * count > len(data):
        raise ValueError("unexpected end of PLY data")
    arr = np.frombuffer(data, dtype=dt, count=count, offset=off)
    return {p[0]: arr[p[0]] for p in props}, off + dt.itemsize * count


def _unpack_unorm(packed: np.ndarray, bits: int) -> np.ndarray:
    """quant.rs:4-7."""
    return packed.astype(np.float32) / np.float32((1 << bits) - 1)


def decode_vec_11_10_11(value: np.ndarray) -> np.ndarray:
    """quant.rs:9-18 -> [n,3] in [0,1]."""
    v = np.asarray(value, np.uint32)
    return np.stack([_unpack_unorm((v >> 21) & 0x7FF, 11), _unpack_unorm((v >> 11) & 0x3FF, 10), _unpack_unorm(v & 0x7FF, 11)], -1)


def decode_vec_8_8_8_8(value: np.ndarray) -> np.ndarray:
    """quant.rs:20-35 -> [n,4] in [0,1], most significant byte first."""
    v = np.asarray(value, np.uint32)
    return np.stack([_unpack_unorm((v >> s) & 0xFF, 8) for s in (24, 16, 8, 0)], -1)


def decode_quat(value: np.ndarray) -> np.ndarray:
    """quant.rs:37-71, smallest-three: two bits name the dropped (largest) component of (w, x, y, z), three 10-bit
    values hold the others in order.  Returns [n,4] in the (w, x, y, z) order the splat arrays use."""
    v = np.atleast_1d(np.asarray(value, np.uint32))
    largest = ((v >> 30) & 0x3).astype(np.int64)
    norm = np.float32(0.5) * np.float32(math.sqrt(2.0))
    abc = np.stack([(_unpack_unorm((v >> sft) & 0x3FF, 10) - np.float32(0.5)) / norm for sft in (20, 10, 0)], -1)
    big = np.sqrt(np.float32(1.0) - (abc * abc).sum(-1, dtype=np.float32))
    quat = np.empty((v.shape[0], 4), np.float32)
    rows = np.arange(v.shape[0])
    for comp in range(4):                                # component `comp` of (w, x, y, z)
        idx = comp - (comp > largest)                    # position among the three stored values (skipping the largest)
        quat[:, comp] = np.where(comp == largest, big, abc[rows, np.clip(idx, 0, 2)])
    return quat


def _load_compressed_ply(data: bytes, fmt: str, comments, elements, off: int, sub: int):
    """parse_compressed_ply (import.rs:408-600).  Row i (0-based) uses the quantisation ranges of chunk i // 256 and is
    kept when (i + 1) % subsample == 0; opacity and colour come post-activation and are converted back (inverse sigmoid,
    rgb -> SH DC); the optional third element holds the higher SH bands as u8, channel-major."""
    idx = 0
    metas = {k: [] for k in _QUANT_META_FIELDS}
    while idx < len(elements) and elements[idx][0] == "chunk":
        name, count, props = elements[idx]
        cols, off = _read_element(data, fmt, off, count, props)
        for k in _QUANT_META_FIELDS:
            if k not in cols:
                raise ValueError(f"missing field `{k}`")
            metas[k].append(np.asarray(cols[k], np.float32))
        idx += 1
    meta = {k: np.concatenate(v) for k, v in metas.items()}
    if idx >= len(elements) or elements[idx][0] != "vertex":
        raise ValueError("Unknown format")
    name, total, props = elements[idx]
    cols, off = _read_element(data, fmt, off, total, props)
    for k in ("packed_position", "packed_scale", "packed_rotation", "packed_color"):   # not optional here (import.rs:484)
        if k not in cols:
            raise ValueError(f"missing field `{k}`")
    keep = np.arange(sub - 1, total, sub)
    chunk = keep // 256
    if total and (len(meta["min_x"]) == 0 or chunk.size and chunk.max() >= len(meta["min_x"])):
        raise ValueError("compressed PLY: fewer chunk rows than the vertex count needs")

    def dequant(raw, names):                             # QuantMeta::{mean, scale, color}: raw * (max - min) + min
        lo = np.stack([meta["min_" + nm][chunk] for nm in names], -1)
        hi = np.stack([meta["max_" + nm][chunk] for nm in names], -1)
        return raw * (hi - lo) + lo

    means = dequant(decode_vec_11_10_11(cols["packed_position"][keep]), ("x", "y", "z")).astype(np.float32)
    log_scales = dequant(decode_vec_11_10_11(cols["packed_scale"][keep]), ("scale_x", "scale_y", "scale_z")).astype(np.float32)
    rotations = decode_quat(cols["packed_rotation"][keep]).reshape(-1, 4)
    rgba = decode_vec_8_8_8_8(cols["packed_color"][keep])
    with np.errstate(divide="ignore", invalid="ignore"):
        opacity = np.log(rgba[:, 3] / (np.float32(1.0) - rgba[:, 3])).astype(np.float32)      # inverse_sigmoid
    dc = ((dequant(rgba[:, :3], ("r", "g", "b")) - np.float32(0.5)) / np.float32(SH_C0)).astype(np.float32)   # rgb_to_sh
    n = keep.size
    sh = dc.reshape(n, 1, 3)
    idx += 1
    if idx < len(elements) and len(elements) > 2:        # header.elem_defs.get(2): the higher bands, if present
        name, count, props = elements[idx]
        if name == "sh" and props:
            scols, off = _read_element(data, fmt, off, count, props)
            rest_names = sorted((nm for nm in scols if nm.startswith("f_rest_")), key=lambda t: int(t[7:]))
            sh_count = len(rest_names)
            skeep = np.arange(sub - 1, count, sub)[:n]
            if skeep.size != n:
                raise ValueError("compressed PLY: the sh element is shorter than the vertex element")
            rest = np.stack([(np.asarray(scols[nm][skeep], np.float32) / np.float32(254.0) - np.float32(0.5)) * np.float32(8.0)
                             for nm in rest_names], 1) if sh_count else np.zeros((n, 0), np.float32)     # de_quant_sh
            per = sh_count // 3
            sh = np.empty((n, 1 + per, 3), np.float32)
            sh[:, 0, :] = dc
            if per:
                sh[:, 1:, :] = rest[:, :3 * per].reshape(n, 3, per).transpose(0, 2, 1)                  # interleave_coeffs
    d = SplatData(means=means, rotations=rotations, log_scales=log_scales, sh_coeffs=sh, raw_opacities=opacity)
    return d, ParseMetadata(up_axis=_up_axis(comments), render_mip=_render_mode(comments), total_splats=n)


COMPRESSED_VERTEX_FIELDS = ("packed_position", "packed_rotation", "packed_scale", "packed_color")


def compressed_ply_bytes(chunks: np.ndarray, packed: np.ndarray, sh_bytes: Optional[np.ndarray], m: int, comments) -> bytes:
    """The SuperSplat compressed layout that _load_compressed_ply reads, from an encoding (DESIGN.md section 4.8):
    chunks [ceil(m/256), 18] f32 in _QUANT_META_FIELDS order, packed [m, 4] u32 (COMPRESSED_VERTEX_FIELDS),
    sh_bytes [m, 3(K-1)] u8 channel-major or None for K == 1.  Binary little-endian."""
    m = int(m)
    n_chunks = (m + 255) // 256
    chunks = np.ascontiguousarray(chunks, np.float32).reshape(-1, 18)[:n_chunks]
    packed = np.ascontiguousarray(packed, np.uint32).reshape(-1, 4)[:m]
    rest = 0 if sh_bytes is None else int(sh_bytes.shape[1])
    head = ["ply", "format binary_little_endian 1.0"] + [f"comment {c}" for c in comments]
    head += [f"element chunk {n_chunks}"] + [f"property float {nm}" for nm in _QUANT_META_FIELDS]
    head += [f"element vertex {m}"] + [f"property uint {nm}" for nm in COMPRESSED_VERTEX_FIELDS]
    body = chunks.astype("<f4").tobytes() + packed.astype("<u4").tobytes()
    if rest:
        head += [f"element sh {m}"] + [f"property uchar f_rest_{i}" for i in range(rest)]
        body += np.ascontiguousarray(sh_bytes[:m], np.uint8).tobytes()
    return ("\n".join(head + ["end_header"]) + "\n").encode("ascii") + body


def mesh_to_ply(vertices: np.ndarray, colors: np.ndarray, faces: np.ndarray) -> bytes:
    """A coloured triangle mesh (DESIGN.md section 4.9) as binary little-endian PLY: vertex x, y, z (float) and red, green,
    blue (uchar); face vertex_indices (list uchar int, three per face)."""
    v = np.ascontiguousarray(vertices, np.float32).reshape(-1, 3)
    c = np.ascontiguousarray(colors, np.uint8).reshape(-1, 3)
    f = np.asarray(faces).reshape(-1, 3)
    if len(c) != len(v):
        raise ValueError("mesh_to_ply: one colour per vertex")
    if len(f) and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError("mesh_to_ply: face index out of range")
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}", "property float x", "property float y",
            "property float z", "property uchar red", "property uchar green", "property uchar blue",
            f"element face {len(f)}", "property list uchar int vertex_indices", "end_header"]
    vrow = np.empty(len(v), np.dtype([("p", "<f4", 3), ("c", "u1", 3)]))
    vrow["p"], vrow["c"] = v, c
    frow = np.empty(len(f), np.dtype([("n", "u1"), ("i", "<i4", 3)]))
    frow["n"], frow["i"] = 3, f
    return ("\n".join(head) + "\n").encode("ascii") + vrow.tobytes() + frow.tobytes()
