"""SceneBatch producer and dataset readers (SURVEY 8f N2), host side.

  view_to_packed_data / pack_rgba <- brush-dataset/src/scene.rs:97-136 (u8 RGBA packed little endian into one int32
                                      per pixel, byte-space premultiplication for AlphaMode::Transparent)
  load_dataset                    <- formats/mod.rs:57-110 (COLMAP, then nerfstudio json, then RealityCapture csv; an
                                      init.ply overrides the format's own initial points)
  load_colmap (text or binary)    <- formats/colmap.rs:102-303 (views sorted by image name, subsample / max frames,
                                      w2c -> c2w, fov from focal per camera model, missing images skipped with a warning,
                                      initial points from points3D)
  build_camera_model              <- formats/colmap.rs:305-390 (COLMAP sensor models -> pinhole / RT8 / KB4 / TPF)
  load_nerfstudio                 <- formats/nerfstudio.rs (transforms*.json: per-frame / per-file intrinsics, OPENCV and
                                      OPENCV_FISHEYE models, OpenGL camera-to-world -> brush pose, val / test file)
  load_realitycapture             <- formats/realitycapture.rs (camera csv: 35 mm-film intrinsics, heading / pitch / roll)
  find_image_by_name, find_mask_path, split_eval_every, opengl_c2w_to_pose <- formats/mod.rs:112-189
  SceneView.load_image            <- load_image.rs:59-123 (decode, mask file -> alpha channel, resolution cap)
  SceneView.load_depth, find_depth_path <- per-view depth maps for depth supervision (DESIGN.md section 4.7; nerfstudio's
                                      `depth_file_path`, COLMAP `depths/`); no reference counterpart
  COLMAP text / binary grammar    <- colmap-reader/src/lib.rs (cameras / images / points3D, .txt and .bin)
  SceneLoader                     <- scene_loader.rs:13-170 (loader threads, bounded prefetch queue, packed-batch cache)

The step's only host->device input is the packed [H,W] int32 image of a view.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import camera as cm
from .camera import Camera
from .ply import SH_C0, SplatData

ALPHA_MASKED, ALPHA_TRANSPARENT = "masked", "transparent"


def pack_rgba(rgba: np.ndarray, premultiply: bool) -> np.ndarray:
    """scene.rs:121-136.  rgba: uint8 [H,W,4] -> int32 [H,W] (r | g<<8 | b<<16 | a<<24)."""
    px = np.ascontiguousarray(rgba, np.uint8)
    if premultiply:
        a = px[..., 3:4].astype(np.uint16)
        rgb = ((px[..., :3].astype(np.uint16) * a + 127) // 255).astype(np.uint8)   # byte space, before any float
        px = np.concatenate([rgb, px[..., 3:4]], axis=-1)
    return np.ascontiguousarray(px).view("<u4").reshape(px.shape[0], px.shape[1]).view(np.int32)


def view_to_packed_data(image: np.ndarray, alpha_mode: str = ALPHA_MASKED) -> Tuple[np.ndarray, bool]:
    """scene.rs:97-119.  image: uint8 [H,W,3] or [H,W,4] (other depths: convert to RGBA8 first).
    Returns (packed int32 [H,W], has_alpha)."""
    if image.dtype != np.uint8 or image.ndim != 3 or image.shape[2] not in (3, 4):
        raise ValueError("expected a uint8 [H,W,3|4] image")
    has_alpha = image.shape[2] == 4
    if not has_alpha:
        image = np.concatenate([image, np.full(image.shape[:2] + (1,), 255, np.uint8)], axis=-1)
    return pack_rgba(image, has_alpha and alpha_mode == ALPHA_TRANSPARENT), has_alpha


# ---- COLMAP text model ------------------------------------------------------------------------------------
@dataclass
class ColmapCamera:
    id: int
    model: str
    width: int
    height: int
    params: List[float]

    def focal(self) -> Tuple[float, float]:
        if self.model in ("SIMPLE_PINHOLE", "SIMPLE_RADIAL", "RADIAL", "SIMPLE_RADIAL_FISHEYE", "RADIAL_FISHEYE"):
            return self.params[0], self.params[0]
        return self.params[0], self.params[1]

    def principal_point(self) -> Tuple[float, float]:
        if self.model in ("SIMPLE_PINHOLE", "SIMPLE_RADIAL", "RADIAL", "SIMPLE_RADIAL_FISHEYE", "RADIAL_FISHEYE"):
            return self.params[1], self.params[2]
        return self.params[2], self.params[3]


@dataclass
class ColmapImage:
    id: int
    quat_wxyz: Tuple[float, float, float, float]   # world -> camera
    tvec: Tuple[float, float, float]
    camera_id: int
    name: str


def _data_lines(text: str):
    for ln in text.splitlines():
        s = ln.strip()
        if s and not s.startswith("#"):
            yield s


def read_cameras_text(text: str) -> List[ColmapCamera]:
    out = []
    for s in _data_lines(text):
        p = s.split()
        out.append(ColmapCamera(int(p[0]), p[1], int(p[2]), int(p[3]), [float(v) for v in p[4:]]))
    return out


def read_images_text(text: str) -> List[ColmapImage]:
    """Two lines per image; the second (2D points) may be empty, so blank lines are significant."""
    out = []
    lines = [ln for ln in text.splitlines() if not ln.lstrip().startswith("#")]
    i = 0
    while i < len(lines):
        s = lines[i].strip()
        if not s:
            i += 1
            continue
        p = s.split()
        out.append(ColmapImage(int(p[0]), tuple(float(v) for v in p[1:5]), tuple(float(v) for v in p[5:8]), int(p[8]),
                               " ".join(p[9:])))
        i += 2   # skip the POINTS2D line
    return out


def read_points3d_text(text: str):
    xyz, rgb = [], []
    for s in _data_lines(text):
        p = s.split()
        xyz.append([float(p[1]), float(p[2]), float(p[3])])
        rgb.append([int(p[4]), int(p[5]), int(p[6])])
    return np.array(xyz, np.float32).reshape(-1, 3), np.array(rgb, np.uint8).reshape(-1, 3)


# ---- COLMAP binary model (colmap-reader/src/lib.rs:278-300, 389-470, 546-600) ---------------------------------
_MODEL_BY_ID = {0: ("SIMPLE_PINHOLE", 3), 1: ("PINHOLE", 4), 2: ("SIMPLE_RADIAL", 4), 3: ("RADIAL", 5), 4: ("OPENCV", 8),
                5: ("OPENCV_FISHEYE", 8), 6: ("FULL_OPENCV", 12), 7: ("FOV", 5), 8: ("SIMPLE_RADIAL_FISHEYE", 4),
                9: ("RADIAL_FISHEYE", 5), 10: ("THIN_PRISM_FISHEYE", 12)}


def read_cameras_binary(data: bytes) -> List[ColmapCamera]:
    import struct
    (num,), off, out = struct.unpack_from("<Q", data, 0), 8, []
    for _ in range(num):
        cid, mid, w, h = struct.unpack_from("<iiQQ", data, off)
        off += 24
        if mid not in _MODEL_BY_ID:
            raise ValueError("Invalid camera model")
        name, npar = _MODEL_BY_ID[mid]
        params = list(struct.unpack_from(f"<{npar}d", data, off))
        off += 8 * npar
        out.append(ColmapCamera(cid, name, int(w), int(h), params))
    return out


def read_images_binary(data: bytes) -> List[ColmapImage]:
    import struct
    (num,), off, out = struct.unpack_from("<Q", data, 0), 8, []
    for _ in range(num):
        iid, qw, qx, qy, qz, tx, ty, tz, cid = struct.unpack_from("<i7di", data, off)
        off += 4 + 56 + 4
        end = data.find(b"\0", off)
        if end < 0:
            raise ValueError("image name was not null-terminated (truncated images file?)")
        name = data[off:end].decode("utf-8")
        off = end + 1
        (npts,) = struct.unpack_from("<Q", data, off)
        off += 8 + 24 * npts                                   # (x, y, point3D id) per 2D point: skipped
        if off > len(data):
            raise ValueError("truncated images file")
        f32 = lambda v: float(np.float32(v))                    # the reference narrows pose values to f32 on read
        out.append(ColmapImage(iid, (f32(qw), f32(qx), f32(qy), f32(qz)), (f32(tx), f32(ty), f32(tz)), cid, name))
    return out


def read_points3d_binary(data: bytes):
    import struct
    (num,), off = struct.unpack_from("<Q", data, 0), 8
    xyz, rgb = np.empty((num, 3), np.float32), np.empty((num, 3), np.uint8)
    for i in range(num):
        _, x, y, z, r, g, b, _err, track = struct.unpack_from("<q3d3BdQ", data, off)
        off += 8 + 24 + 3 + 8 + 8 + 8 * track
        xyz[i] = (x, y, z)
        rgb[i] = (r, g, b)
    return xyz, rgb


def build_camera_model(c: ColmapCamera):
    """formats/colmap.rs:305-390 -> (camera_model id, model_params)."""
    p, m = c.params, c.model
    f32 = lambda v: float(np.float32(v))
    if m in ("SIMPLE_PINHOLE", "PINHOLE", "FOV"):          # FOV: no matching polynomial, falls back to pinhole
        return cm.PINHOLE, ()
    if m == "SIMPLE_RADIAL":
        return cm.RADIAL_TANGENTIAL_8, (f32(p[3]), 0, 0, 0, 0, 0, 0, 0)
    if m == "RADIAL":
        return cm.RADIAL_TANGENTIAL_8, (f32(p[3]), f32(p[4]), 0, 0, 0, 0, 0, 0)
    if m == "OPENCV":
        return cm.RADIAL_TANGENTIAL_8, (f32(p[4]), f32(p[5]), 0, 0, 0, 0, f32(p[6]), f32(p[7]))
    if m == "FULL_OPENCV":
        return cm.RADIAL_TANGENTIAL_8, (f32(p[4]), f32(p[5]), f32(p[8]), f32(p[9]), f32(p[10]), f32(p[11]), f32(p[6]), f32(p[7]))
    if m == "SIMPLE_RADIAL_FISHEYE":
        return cm.KANNALA_BRANDT_4, (f32(p[3]), 0, 0, 0)
    if m == "RADIAL_FISHEYE":
        return cm.KANNALA_BRANDT_4, (f32(p[3]), f32(p[4]), 0, 0)
    if m == "OPENCV_FISHEYE":
        return cm.KANNALA_BRANDT_4, (f32(p[4]), f32(p[5]), f32(p[6]), f32(p[7]))
    if m == "THIN_PRISM_FISHEYE":
        return cm.THIN_PRISM_FISHEYE, (f32(p[4]), f32(p[5]), f32(p[8]), f32(p[9]), f32(p[6]), f32(p[7]), f32(p[10]), f32(p[11]))
    raise ValueError(f"unknown COLMAP camera model {m}")


def _quat_to_mat(w, x, y, z):
    n = math.sqrt(w * w + x * x + y * y + z * z)
    w, x, y, z = w / n, x / n, y / n, z / n
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def camera_from_colmap(c: ColmapCamera, img: ColmapImage) -> Camera:
    """colmap.rs:170-202: intrinsics -> fov per model, world-to-camera pose -> camera-to-world."""
    model, params = build_camera_model(c)
    fx, fy = c.focal()
    fov_x = cm.focal_to_fov(fx, c.width, model, params)
    fov_y = cm.focal_to_fov(fy, c.height, model, params)
    cx, cy = c.principal_point()
    qw, qx, qy, qz = img.quat_wxyz
    R = _quat_to_mat(qw, qx, qy, qz)
    pos = -R.T @ np.array(img.tvec, np.float64)
    n = math.sqrt(qw * qw + qx * qx + qy * qy + qz * qz)
    rot_c2w = (-qx / n, -qy / n, -qz / n, qw / n)            # conjugate, glam (x, y, z, w) order
    return Camera(position=tuple(float(v) for v in pos), rotation=rot_c2w, fov_x=fov_x, fov_y=fov_y,
                  center_uv=(float(np.float32(cx) / np.float32(c.width)), float(np.float32(cy) / np.float32(c.height))),
                  camera_model=model, model_params=params)


def split_eval_every(views: Sequence, eval_split_every: Optional[int]):
    """formats/mod.rs:135-148 -> (train, eval)."""
    train, ev = [], []
    for i, v in enumerate(views):
        (ev if (eval_split_every and i % eval_split_every == 0) else train).append(v)
    return train, ev


def find_mask_path(files: Sequence[str], path: str) -> Optional[str]:
    """formats/mod.rs:150-189.  `files`: every file of the dataset (relative or absolute, one convention); `path`: the
    image.  A mask lives under a directory called `masks` (any case), is named img.png.*, img.* or img.mask.* (any case,
    any extension), and the directories below `masks/` must be the tail of the image's own directory:
    masks/foo/bar/img.png matches images/foo/bar/img.jpeg.  First match in `files` order."""
    norm = lambda q: [c for c in q.replace("\\", "/").split("/") if c not in ("", ".")]
    comps = norm(path)
    name = comps[-1].lower()
    stem = name.rsplit(".", 1)[0] if "." in name[1:] else name
    wanted = {name, stem, stem + ".mask"}
    parent = [c for c in comps[:-1]]
    for cand in files:
        cc = norm(cand)
        if not cc:
            continue
        cname = cc[-1].lower()
        cstem = cname.rsplit(".", 1)[0] if "." in cname[1:] else cname
        if cstem not in wanted:
            continue
        idx = next((i for i, c in enumerate(cc) if c.lower() == "masks"), None)
        if idx is None:
            continue
        sub = cc[idx + 1:-1]
        if len(sub) <= len(parent) and (not sub or parent[len(parent) - len(sub):] == sub):
            return cand
    return None


def find_depth_path(files: Sequence[str], path: str) -> Optional[str]:
    """The depth map of a COLMAP image: `<stem>.png` or `<stem>.npy` (any case) under a directory called `depths` (any
    case), whose sub-directories below `depths/` must be the tail of the image's own directory, as find_mask_path requires
    of masks: depths/foo/img.png matches images/foo/img.jpg.  First match in `files` order."""
    norm = lambda q: [c for c in q.replace("\\", "/").split("/") if c not in ("", ".")]
    comps = norm(path)
    name = comps[-1].lower()
    stem = name.rsplit(".", 1)[0] if "." in name[1:] else name
    wanted = {stem + ".png", stem + ".npy"}
    parent = comps[:-1]
    for cand in files:
        cc = norm(cand)
        if not cc or cc[-1].lower() not in wanted:
            continue
        idx = next((i for i, c in enumerate(cc) if c.lower() == "depths"), None)
        if idx is None:
            continue
        sub = cc[idx + 1:-1]
        if len(sub) <= len(parent) and (not sub or parent[len(parent) - len(sub):] == sub):
            return cand
    return None


def decode_depth(path: str) -> np.ndarray:
    """A single-channel depth file -> f32 [H,W] in file units: `.npy` (2-D or [H,W,1]) or a PNG / TIFF in PIL mode
    I;16, I, F or L.  Anything with more than one channel is a ValueError."""
    if path.lower().endswith(".npy"):
        a = np.load(path, allow_pickle=False)
        if a.ndim == 3 and a.shape[2] == 1:
            a = a[..., 0]
        if a.ndim != 2:
            raise ValueError(f"depth map {path}: expected [H,W] or [H,W,1], got shape {a.shape}")
        return np.asarray(a, np.float32)
    from PIL import Image
    with Image.open(path) as im:
        if im.mode not in ("I;16", "I;16B", "I;16L", "I", "F", "L"):
            raise ValueError(f"depth map {path}: expected a single-channel image (I;16, I, F or L), got mode {im.mode}")
        return np.asarray(im).astype(np.float32)


def resize_nearest(a: np.ndarray, w: int, h: int) -> np.ndarray:
    """Nearest-neighbour resize of [H,W] to [h,w] with pixel centres aligned: source index floor((i + 0.5) * src / dst).
    Never blends values, so invalid zeros stay apart from valid depths."""
    sh, sw = a.shape
    if (sh, sw) == (h, w):
        return a
    ys = np.minimum(((np.arange(h) + 0.5) * sh / h).astype(np.int64), sh - 1)
    xs = np.minimum(((np.arange(w) + 0.5) * sw / w).astype(np.int64), sw - 1)
    return a[ys[:, None], xs[None, :]]


def scaled_image_size(w: int, h: int, scale: float, max_resolution: Optional[int] = None) -> Tuple[int, int]:
    """LoadImage::output_scale + load (load_image.rs:115-131), in f32: factor = min(cap * scale, 1) with
    cap = max_res / max(w, h, max_res) (1 without a cap); the size is trunc(max(side * factor, 1)), unchanged when the
    factor is 1."""
    f32 = np.float32
    cap = f32(max_resolution) / f32(max(w, h, max_resolution)) if max_resolution else f32(1.0)
    factor = min(cap * f32(scale), f32(1.0))
    if factor >= f32(1.0):
        return w, h
    return int(max(f32(w) * factor, f32(1.0))), int(max(f32(h) * factor, f32(1.0)))


@dataclass
class SceneView:
    camera: Camera
    image_path: str
    mask_path: Optional[str] = None      # load_image.rs:15: a separate mask image that becomes the alpha channel
    invert_mask: bool = False            # config.rs:46-48: white means "ignore this pixel"
    depth_path: Optional[str] = None     # a per-view depth map (DESIGN.md section 4.7)
    depth_scale: float = 1.0             # file units -> scene units (the dataset's depth_unit_scale_factor)

    def default_alpha_mode(self) -> str:
        """LoadImage::new (load_image.rs:41-47): a view with a mask file is Masked, anything else Transparent, unless the
        load arguments override it."""
        return ALPHA_MASKED if self.mask_path is not None else ALPHA_TRANSPARENT

    def img_name(self) -> str:
        """load_image.rs:174-180: the file name, extension included."""
        return os.path.basename(self.image_path)

    def load_packed(self, alpha_mode: str = ALPHA_MASKED, max_resolution: Optional[int] = None, scale: float = 1.0):
        return view_to_packed_data(self.load_image(max_resolution, scale), alpha_mode)

    def load_image(self, max_resolution: Optional[int] = None, scale: float = 1.0) -> np.ndarray:
        """LoadImage::load (load_image.rs:59-123): decode, put the mask (if any) into the alpha channel, cap the long edge.
        scale < 1 (the LOD levels' downscaled images, LoadImage::with_scale) sizes the output by scaled_image_size.
        Returns uint8 [H,W,3] or [H,W,4]."""
        from PIL import Image
        im = Image.open(self.image_path)
        if im.mode not in ("RGB", "RGBA"):
            im = im.convert("RGBA" if "A" in im.getbands() else "RGB")
        if self.mask_path is not None:      # load_image.rs:69-113: one channel of the mask becomes the alpha channel
            im = im.convert("RGBA")
            mk = Image.open(self.mask_path)
            mk = mk.convert("RGBA").getchannel("A") if "A" in mk.getbands() else mk.convert("L")
            if mk.size != im.size:
                mk = mk.resize(im.size, Image.BILINEAR)          # imageops::FilterType::Triangle; may squash the mask
            alpha = np.asarray(mk, np.uint8)
            if self.invert_mask:
                alpha = np.uint8(255) - alpha
            rgba = np.asarray(im, np.uint8).copy()
            rgba[..., 3] = alpha
            im = Image.fromarray(rgba, "RGBA")
        if scale < 1.0:
            size = scaled_image_size(im.size[0], im.size[1], scale, max_resolution)
            return np.asarray(im.resize(size, Image.LANCZOS) if size != im.size else im, np.uint8)
        if max_resolution and max(im.size) > max_resolution:
            s = max_resolution / max(im.size)
            im = im.resize((max(1, round(im.size[0] * s)), max(1, round(im.size[1] * s))), Image.LANCZOS)
        return np.asarray(im, np.uint8)

    def image_size(self, max_resolution: Optional[int] = None, scale: float = 1.0) -> Tuple[int, int]:
        """(w, h) of load_image(max_resolution, scale), from the image header alone."""
        from PIL import Image
        with Image.open(self.image_path) as im:
            w, h = im.size
        if scale < 1.0:
            return scaled_image_size(w, h, scale, max_resolution)
        if max_resolution and max(w, h) > max_resolution:
            s = max_resolution / max(w, h)
            return max(1, round(w * s)), max(1, round(h * s))
        return w, h

    def load_depth(self, max_resolution: Optional[int] = None, scale: float = 1.0) -> Optional[np.ndarray]:
        """The view's depth target as f32 [H,W] in scene units, at exactly the size load_image(max_resolution, scale)
        returns: decoded (decode_depth), multiplied by depth_scale, nearest-resized; non-finite or <= 0 values become 0
        (no measurement).  None when the view has no depth map."""
        if self.depth_path is None:
            return None
        d = decode_depth(self.depth_path) * np.float32(self.depth_scale)
        w, h = self.image_size(max_resolution, scale)
        d = resize_nearest(d, w, h)
        return np.ascontiguousarray(np.where(np.isfinite(d) & (d > 0), d, np.float32(0.0)), np.float32)


@dataclass
class DatasetLoadResult:
    train: List[SceneView]
    eval: List[SceneView]
    init_splat: Optional[SplatData]
    warnings: List[str] = field(default_factory=list)


def list_files(root: str) -> List[str]:
    """Every file under `root`, relative, '/'-separated, sorted (the role of the reference's vfs listing)."""
    out = []
    for d, _, fs in os.walk(root):
        for f in fs:
            out.append(os.path.relpath(os.path.join(d, f), root).replace(os.sep, "/"))
    return sorted(out)


def find_image_by_name(files: Sequence[str], name: str) -> Optional[str]:
    """formats/mod.rs:112-120: colmap stores a bare (or sub-directory) file name; the image is the lexicographically first
    file whose path ends with it on a component boundary (case-insensitive, like the vfs keys), never one under a
    `masks` directory -- an image must not resolve to its own mask -- nor under a `depths` directory (any case), where its
    depth map may carry the image's own file name (find_depth_path)."""
    key = "/" + name.replace("\\", "/").lower().lstrip("/")
    hits = [f for f in files if ("/" + f.lower()).endswith(key) and "masks" not in f.split("/")[:-1]
            and not any(c.lower() == "depths" for c in f.split("/")[:-1])]
    return min(hits) if hits else None


def _find(root: str, name: str) -> Optional[str]:
    low = name.lower()
    for d, _, files in os.walk(root):
        for f in files:
            if f.lower() == low:
                return os.path.join(d, f)
    return None


def load_colmap(root: str, subsample_frames: Optional[int] = None, max_frames: Optional[int] = None,
                eval_split_every: Optional[int] = None, subsample_points: Optional[int] = None,
                invert_masks: bool = False, depth_unit_scale_factor: float = 1e-3) -> DatasetLoadResult:
    """Text or binary COLMAP model (cameras.{txt,bin} decides; images / points3D are taken from the same directory).
    Views whose image has a counterpart under a `masks/` directory carry it as their alpha channel (colmap.rs:194-218),
    views with a `depths/<stem>.png|.npy` (find_depth_path) a depth map in units of depth_unit_scale_factor."""
    cam_path = _find(root, "cameras.bin") or _find(root, "cameras.txt")
    if cam_path is None:
        raise FileNotFoundError("no cameras.txt / cameras.bin under " + root)
    sparse = os.path.dirname(cam_path)
    is_binary = cam_path.endswith(".bin")
    if is_binary:
        cams = {c.id: c for c in read_cameras_binary(open(cam_path, "rb").read())}
        infos = read_images_binary(open(os.path.join(sparse, "images.bin"), "rb").read())
    else:
        cams = {c.id: c for c in read_cameras_text(open(cam_path).read())}
        infos = read_images_text(open(os.path.join(sparse, "images.txt")).read())
    infos = sorted(infos, key=lambda i: i.name)
    views, warnings = [], []
    files = mask_files = depth_files = None                # the dataset's file list / mask / depth candidates, listed once
    picked = infos[::max(int(subsample_frames or 1), 1)]
    if max_frames is not None:
        picked = picked[:max_frames]
    for info in picked:
        if info.camera_id not in cams:
            raise ValueError(f"Image '{info.name}' references camera ID {info.camera_id} which doesn't exist in camera data")
        if files is None:
            files = list_files(root)
        rel = find_image_by_name(files, info.name)
        if rel is None:
            warnings.append(f"Skipped '{info.name}': image file not found")
            continue
        path = os.path.join(root, rel)
        camera = camera_from_colmap(cams[info.camera_id], info)
        if not camera.is_valid():
            warnings.append(f"Skipped '{info.name}': camera contains nan or inf values")
            continue
        if mask_files is None:                             # mask candidates: paths relative to the root, like the vfs
            mask_files = [f for f in files if any(c.lower() == "masks" for c in f.split("/")[:-1])]
        mask = find_mask_path(mask_files, rel) if mask_files else None
        mask = os.path.join(root, mask) if mask is not None else None
        if depth_files is None:
            depth_files = [f for f in files if any(c.lower() == "depths" for c in f.split("/")[:-1])]
        depth = find_depth_path(depth_files, rel) if depth_files else None
        views.append(SceneView(camera, path, mask, bool(invert_masks) and mask is not None,
                               os.path.join(root, depth) if depth is not None else None, float(depth_unit_scale_factor)))
    train, ev = split_eval_every(views, eval_split_every)
    init = None
    pts_txt, pts_bin = os.path.join(sparse, "points3D.txt"), os.path.join(sparse, "points3D.bin")
    if os.path.exists(pts_txt) or os.path.exists(pts_bin):
        xyz, rgb = read_points3d_text(open(pts_txt).read()) if os.path.exists(pts_txt) else \
            read_points3d_binary(open(pts_bin, "rb").read())
        step = max(int(subsample_points or 1), 1)
        xyz, rgb = xyz[::step], rgb[::step]
        if len(xyz):
            sh = ((rgb.astype(np.float32) / np.float32(255.0)) - np.float32(0.5)) / np.float32(SH_C0)   # rgb_to_sh
            init = SplatData(means=xyz, sh_coeffs=sh.reshape(-1, 1, 3))
    return DatasetLoadResult(train, ev, init, warnings)


load_colmap_text = load_colmap   # earlier name


# ---- nerfstudio transforms.json -----------------------------------------------------------------------------
def _quat_xyzw_from_mat(R: np.ndarray) -> Tuple[float, float, float, float]:
    """Rotation matrix (columns = axes) -> unit quaternion in glam's (x, y, z, w) order (Quat::from_mat3's branches)."""
    m00, m01, m02 = R[0, 0], R[0, 1], R[0, 2]
    m10, m11, m12 = R[1, 0], R[1, 1], R[1, 2]
    m20, m21, m22 = R[2, 0], R[2, 1], R[2, 2]
    tr = m00 + m11 + m22
    if tr > 0:
        s = math.sqrt(tr + 1.0) * 2
        q = ((m21 - m12) / s, (m02 - m20) / s, (m10 - m01) / s, 0.25 * s)
    elif m00 > m11 and m00 > m22:
        s = math.sqrt(1.0 + m00 - m11 - m22) * 2
        q = (0.25 * s, (m01 + m10) / s, (m02 + m20) / s, (m21 - m12) / s)
    elif m11 > m22:
        s = math.sqrt(1.0 + m11 - m00 - m22) * 2
        q = ((m01 + m10) / s, 0.25 * s, (m12 + m21) / s, (m02 - m20) / s)
    else:
        s = math.sqrt(1.0 + m22 - m00 - m11) * 2
        q = ((m02 + m20) / s, (m12 + m21) / s, 0.25 * s, (m10 - m01) / s)
    n = math.sqrt(sum(v * v for v in q))
    return tuple(float(v / n) for v in q)


def opengl_c2w_to_pose(c2w: np.ndarray):
    """formats/mod.rs:122-131: an OpenGL / Blender camera-to-world matrix (+X right, +Y up, +Z back; the nerfstudio
    `transform_matrix`) -> (position, rotation xyzw) in brush's convention (+Y down, +Z forward).  Scale is divided out
    of the axes as glam's to_scale_rotation_translation does."""
    m = np.array(c2w, np.float64).reshape(4, 4).copy()
    m[:, 1] *= -1.0
    m[:, 2] *= -1.0
    A = m[:3, :3]
    scale = np.linalg.norm(A, axis=0)
    if np.linalg.det(A) < 0:
        scale[0] = -scale[0]
    with np.errstate(divide="ignore", invalid="ignore"):
        R = A / scale
    pos = tuple(float(v) for v in m[:3, 3])
    if not np.isfinite(R).all():
        return pos, (float("nan"),) * 4
    return pos, _quat_xyzw_from_mat(R)


def _nerfstudio_camera_model(name, k1, k2, k3, k4, p1, p2):
    """resolve_camera_model (nerfstudio.rs:103-140)."""
    f = lambda o: float(np.float32(0.0 if o is None else o))
    if name is None or name in ("PERSPECTIVE", "perspective"):
        return cm.PINHOLE, ()
    if name in ("OPENCV", "opencv"):
        return cm.RADIAL_TANGENTIAL_8, (f(k1), f(k2), 0.0, 0.0, 0.0, 0.0, f(p1), f(p2))
    if name in ("OPENCV_FISHEYE", "opencv_fisheye"):
        return cm.KANNALA_BRANDT_4, (f(k1), f(k2), f(k3), f(k4))
    raise ValueError(f"Error decoding camera parameters: Unsupported nerfstudio camera_model `{name}`")


def _resolve_frame_file(fp: str, base: str, root: str, lower: dict) -> Optional[str]:
    """A frame's file reference -> the dataset file it names (relative to root), or None."""
    if os.path.isabs(fp):        # absolute references are resolved inside the dataset directory only (brush-vfs lib.rs:313-325)
        fp_rel = os.path.relpath(fp, os.path.abspath(root))
        rel = fp_rel.replace(os.sep, "/") if not fp_rel.startswith("..") else "\0outside"
    else:
        rel = os.path.normpath(os.path.join(base, fp)).replace(os.sep, "/")
    hit = lower.get(rel.lower())
    if hit is None and not os.path.splitext(rel)[1]:
        # "Assume png's by default if no extension is specified" (nerfstudio.rs:183-186; the reference tests existence
        # before adding the extension, which would skip every such frame -- its stated intent is followed here)
        hit = lower.get((rel + ".png").lower())
    return hit


def _read_transforms_file(scene: dict, transforms_rel: str, root: str, files: Sequence[str], subsample_frames, max_frames,
                          invert_masks: bool, warnings: List[str], depth_unit_scale_factor: float = 1e-3) -> List[SceneView]:
    """read_transforms_file (nerfstudio.rs:142-268).  Per-frame values override the file-level ones."""
    lower = {f.lower(): f for f in files}
    mask_files = [f for f in files if any(c.lower() == "masks" for c in f.split("/")[:-1])]
    base = os.path.dirname(transforms_rel)
    frames = scene.get("frames", [])[::max(int(subsample_frames or 1), 1)]
    if max_frames is not None:
        frames = frames[:max_frames]
    views = []
    for fr in frames:
        flat = [float(v) for row in fr["transform_matrix"] for v in row]
        if len(flat) != 16:
            raise ValueError(f"Error when decoding format: frame '{fr['file_path']}' has a {len(flat)}-element transform_matrix, "
                             "expected a 4x4 (16 elements)")
        pos, rot = opengl_c2w_to_pose(np.array(flat, np.float32).reshape(4, 4))
        hit = _resolve_frame_file(fr["file_path"], base, root, lower)
        if hit is None:
            warnings.append(f"Skipped '{fr['file_path']}': image file not found")
            continue
        get = lambda k: fr.get(k) if fr.get(k) is not None else scene.get(k)
        w, h = get("w"), get("h")
        if w is None or h is None:
            from PIL import Image
            with Image.open(os.path.join(root, hit)) as im:          # header only
                w, h = im.size
        w, h = int(w), int(h)
        model, params = _nerfstudio_camera_model(get("camera_model"), *(get(k) for k in ("k1", "k2", "k3", "k4", "p1", "p2")))

        def fov(angle_key, fl_key, px):
            # frame angle, frame focal, scene angle, scene focal -- in that order (nerfstudio.rs:219-229)
            for src in (fr, scene):
                if src.get(angle_key) is not None:
                    return float(src[angle_key])
                if src.get(fl_key) is not None:
                    return cm.focal_to_fov(float(src[fl_key]), px, model, params)
            return None
        fovx, fovy = fov("camera_angle_x", "fl_x", w), fov("camera_angle_y", "fl_y", h)
        if fovx is None and fovy is None:
            raise ValueError("Error decoding camera parameters: Must have some kind of focal length")
        if fovx is None:
            fovx = cm.focal_to_fov(cm.fov_to_focal(fovy, h, model, params), w, model, params)
        if fovy is None:
            fovy = cm.focal_to_fov(cm.fov_to_focal(fovx, w, model, params), h, model, params)
        cx, cy = get("cx"), get("cy")
        cuv = (float(np.float32(0.5 if cx is None else cx / w)), float(np.float32(0.5 if cy is None else cy / h)))
        camera = Camera(position=pos, rotation=rot, fov_x=fovx, fov_y=fovy, center_uv=cuv, camera_model=model, model_params=params)
        if not camera.is_valid():
            warnings.append(f"Skipped '{fr['file_path']}': camera contains nan or inf values")
            continue
        mask = find_mask_path(mask_files, hit) if mask_files else None
        depth = None
        if fr.get("depth_file_path"):                    # resolved exactly like file_path
            depth = _resolve_frame_file(fr["depth_file_path"], base, root, lower)
            if depth is None:
                warnings.append(f"'{fr['file_path']}': depth file '{fr['depth_file_path']}' not found, the view has no depth")
        views.append(SceneView(camera, os.path.join(root, hit), os.path.join(root, mask) if mask else None,
                               bool(invert_masks) and mask is not None, os.path.join(root, depth) if depth else None,
                               float(depth_unit_scale_factor)))
    return views


def load_nerfstudio(root: str, subsample_frames: Optional[int] = None, max_frames: Optional[int] = None,
                    eval_split_every: Optional[int] = None, subsample_points: Optional[int] = None,
                    invert_masks: bool = False, depth_unit_scale_factor: float = 1e-3) -> Optional[DatasetLoadResult]:
    """nerfstudio.rs:270-388.  None when the directory holds no transforms json (the caller tries the next format).
    The training file is the only json, else `transforms.json`, else `transforms_train.json`; `transforms_val.json` (or
    `transforms_test.json`) provides the evaluation views, otherwise every eval_split_every-th training view does.
    A frame's `depth_file_path` (resolved like `file_path`) is its depth map, in units of depth_unit_scale_factor
    (nerfstudio's default: millimetres); a missing depth file is a warning and the view keeps no depth."""
    import json
    files = list_files(root)
    jsons = [f for f in files if f.lower().endswith(".json")]
    if len(jsons) == 1:
        tpath = jsons[0]
    else:
        ending = lambda suffix: next((f for f in files if ("/" + f.lower()).endswith("/" + suffix)), None)
        tpath = ending("transforms.json") or ending("transforms_train.json")
    if tpath is None:
        return None
    warnings: List[str] = []
    scene = json.load(open(os.path.join(root, tpath)))
    train_all = _read_transforms_file(scene, tpath, root, files, subsample_frames, max_frames, invert_masks, warnings,
                                      depth_unit_scale_factor)
    ends = lambda f, name: f.split("/")[-1] == name
    eval_path = next((f for f in jsons if ends(f, "transforms_val.json")), None) or \
        next((f for f in jsons if ends(f, "transforms_test.json")), None)
    val_views = None
    if eval_path is not None:
        val_views = _read_transforms_file(json.load(open(os.path.join(root, eval_path))), eval_path, root, files, subsample_frames,
                                          max_frames, invert_masks, warnings, depth_unit_scale_factor)
    train, ev = [], []
    for i, v in enumerate(train_all):
        if eval_split_every and i % eval_split_every == 0 and val_views is None:   # extra eval images only without a val file
            ev.append(v)
        else:
            train.append(v)
    if val_views is not None:
        ev.extend(val_views)
    init = None
    ply_rel = scene.get("ply_file_path")
    if ply_rel:
        p = os.path.join(root, os.path.dirname(tpath), ply_rel)
        if os.path.exists(p):
            from . import ply as _ply
            init, _ = _ply.load_splat_from_ply(open(p, "rb").read(), subsample_points)
    return DatasetLoadResult(train, ev, init, warnings)


# ---- RealityCapture / RealityScan camera csv ---------------------------------------------------------------------
_RC_REQUIRED = ("name", "x", "y", "alt", "heading", "pitch", "roll", "f")


def rc_parse_header(line: str) -> Optional[dict]:
    """realitycapture.rs:38-51: column name (lower case, leading '#' stripped) -> index; None unless the pose and focal
    columns are all there (the format's detection signature)."""
    cols = {name.strip().lstrip("#").lower(): i for i, name in enumerate(line.split(","))}
    return cols if all(c in cols for c in _RC_REQUIRED) else None


def _rc_f64(fields, header, name) -> float:
    i = header.get(name)
    if i is None or i >= len(fields):
        return 0.0
    try:
        return float(fields[i].strip())
    except ValueError:
        return 0.0


def rc_build_camera_model(k1, k2, k3, t1, t2):
    """realitycapture.rs:205-223: brown3 + tangential -> RadialTangential8 numerator terms; all zero -> pinhole."""
    if all(v == 0.0 for v in (k1, k2, k3, t1, t2)):
        return cm.PINHOLE, ()
    f = lambda v: float(np.float32(v))
    return cm.RADIAL_TANGENTIAL_8, (f(k1), f(k2), f(k3), 0.0, 0.0, 0.0, f(t1), f(t2))


def rc_row_to_camera(fields, header, w: int, h: int) -> Camera:
    """realitycapture.rs:163-203.  f, px, py are in 35 mm film units (36 mm reference) and scale by the larger image
    side; the orientation is yaw(-heading) about Z, pitch about X, roll about Y: a camera-to-world rotation in the OpenGL
    basis."""
    scale = float(max(w, h))
    focal = _rc_f64(fields, header, "f") * scale / 36.0
    cx = _rc_f64(fields, header, "px") * scale + w / 2.0
    cy = _rc_f64(fields, header, "py") * scale + h / 2.0
    model, params = rc_build_camera_model(*(_rc_f64(fields, header, k) for k in ("k1", "k2", "k3", "t1", "t2")))
    fov_x, fov_y = cm.focal_to_fov(focal, w, model, params), cm.focal_to_fov(focal, h, model, params)
    hd, pt, rl = (math.radians(float(np.float32(_rc_f64(fields, header, k)))) for k in ("heading", "pitch", "roll"))

    def rot(axis, a):
        c, s_ = math.cos(a), math.sin(a)
        return {"x": np.array([[1, 0, 0], [0, c, -s_], [0, s_, c]]), "y": np.array([[c, 0, s_], [0, 1, 0], [-s_, 0, c]]),
                "z": np.array([[c, -s_, 0], [s_, c, 0], [0, 0, 1]])}[axis]
    c2w = np.eye(4)
    c2w[:3, :3] = rot("z", -hd) @ rot("x", pt) @ rot("y", rl)
    c2w[:3, 3] = [float(np.float32(_rc_f64(fields, header, k))) for k in ("x", "y", "alt")]
    pos, q = opengl_c2w_to_pose(c2w)
    return Camera(position=pos, rotation=q, fov_x=fov_x, fov_y=fov_y,
                  center_uv=(float(np.float32(cx / w)), float(np.float32(cy / h))), camera_model=model, model_params=params)


def load_realitycapture(root: str, subsample_frames: Optional[int] = None, max_frames: Optional[int] = None,
                        eval_split_every: Optional[int] = None, subsample_points: Optional[int] = None,
                        invert_masks: bool = False) -> Optional[DatasetLoadResult]:
    """realitycapture.rs:65-160: the first .csv whose header carries the pose and focal columns; one image per row, image
    sizes from the file headers, no initial points.  None when no such csv exists."""
    files = list_files(root)
    contents = None
    for f in files:
        if not f.lower().endswith(".csv"):
            continue
        try:
            txt = open(os.path.join(root, f), encoding="utf-8").read()
        except (OSError, UnicodeDecodeError):
            continue
        first = next((ln for ln in txt.splitlines() if ln.strip()), None)
        if first is not None and rc_parse_header(first) is not None:
            contents = txt
            break
    if contents is None:
        return None
    lines = [ln for ln in contents.splitlines() if ln.strip()]
    header = rc_parse_header(lines[0])
    rows = lines[1:][::max(int(subsample_frames or 1), 1)]
    if max_frames is not None:
        rows = rows[:max_frames]
    mask_files = [f for f in files if any(c.lower() == "masks" for c in f.split("/")[:-1])]
    views, warnings, warned = [], [], False
    from PIL import Image
    for ln in rows:
        fields = ln.split(",")
        if header["name"] >= len(fields):
            continue
        name = fields[header["name"]].strip()
        if not warned and _rc_f64(fields, header, "k4") != 0.0:
            warnings.append("RealityCapture brown4 radial term (k4) isn't supported; approximating with brown3")
            warned = True
        rel = find_image_by_name(files, name)
        if rel is None:
            warnings.append(f"Skipped '{name}': image file not found")
            continue
        with Image.open(os.path.join(root, rel)) as im:      # header only
            w, h = im.size
        camera = rc_row_to_camera(fields, header, w, h)
        if not camera.is_valid():
            warnings.append(f"Skipped '{name}': camera contains nan or inf values")
            continue
        mask = find_mask_path(mask_files, rel) if mask_files else None
        views.append(SceneView(camera, os.path.join(root, rel), os.path.join(root, mask) if mask else None,
                               bool(invert_masks) and mask is not None))
    train, ev = split_eval_every(views, eval_split_every)
    return DatasetLoadResult(train, ev, None, warnings)


def load_dataset(root: str, subsample_frames: Optional[int] = None, max_frames: Optional[int] = None,
                 eval_split_every: Optional[int] = None, subsample_points: Optional[int] = None,
                 invert_masks: bool = False, depth_unit_scale_factor: float = 1e-3) -> DatasetLoadResult:
    """formats/mod.rs:57-110: COLMAP first, then nerfstudio json, then a RealityCapture csv; a dataset without a usable training view is an error; an
    `init.ply` (else the last .ply by name) anywhere in the directory overrides the format's own initial points."""
    args = dict(subsample_frames=subsample_frames, max_frames=max_frames, eval_split_every=eval_split_every,
                subsample_points=subsample_points, invert_masks=invert_masks)
    if _find(root, "cameras.bin") or _find(root, "cameras.txt"):
        res = load_colmap(root, **args, depth_unit_scale_factor=depth_unit_scale_factor)
    else:
        res = load_nerfstudio(root, **args, depth_unit_scale_factor=depth_unit_scale_factor)
        if res is None:
            res = load_realitycapture(root, **args)          # RealityCapture exports carry no depth
        if res is None:
            raise ValueError("Format not recognized: only colmap, nerfstudio json and RealityCapture csv are supported")
    if not res.train:
        raise ValueError("Error when decoding format: dataset contains no usable training views (all images missing or filtered out)")
    plys = sorted(f for f in list_files(root) if f.lower().endswith(".ply"))
    if plys:
        main = next((f for f in plys if f.split("/")[-1] == "init.ply"), plys[-1])
        from . import ply as _ply
        res.init_splat, _ = _ply.load_splat_from_ply(open(os.path.join(root, main), "rb").read(), subsample_points)
    return res


class SceneLoader:
    """Threaded prefetch + packed-batch cache (brush-dataset/src/scene_loader.rs:13-170).

    `threads` loader threads, each walking its own shuffled order of the views (seed + task index, like the reference's
    loader tasks), decode -> premultiply -> pack into the [H,W] u32 layout the loss kernel reads and push SceneBatches
    into a bounded queue (4 batches ahead of the trainer, scene_loader.rs:69-72).  A packed batch is cached the first
    time it is produced while the cache stays under `cache_bytes` (BatchCache, :13-58): a hit hands out the same
    immutable pinned tensor again, so nothing a pending host->device copy reads is ever overwritten; batches that do
    not fit the cache are fresh allocations.  `next_batch()` blocks on the queue only."""

    def __init__(self, views: Sequence[SceneView], alpha_mode: str = ALPHA_MASKED, seed: int = 0,
                 cache_bytes: int = 6 << 30, threads: Optional[int] = None, prefetch: int = 4, image_scale: float = 1.0):
        import queue
        import threading
        self.views, self.alpha_mode = list(views), alpha_mode
        self.image_scale = float(image_scale)        # Scene::with_image_scale (scene.rs:61-70): the LOD levels' images
        if not self.views:
            raise ValueError("SceneLoader needs at least one view")
        self._cache = [None] * len(self.views)
        self._cache_used, self._cache_budget = 0, int(cache_bytes)
        self._lock = threading.Lock()
        self._q = queue.Queue(maxsize=max(int(prefetch), 1))
        self._stop = threading.Event()
        n_threads = threads if threads is not None else max(1, min(8, (os.cpu_count() or 2) // 2))
        self._threads = [threading.Thread(target=self._run, args=(seed + i,), daemon=True, name=f"dataloader-{i}")
                         for i in range(n_threads)]
        for t in self._threads:
            t.start()

    def _make_batch(self, index: int):
        import torch
        from .train import SceneBatch
        with self._lock:
            hit = self._cache[index]
        if hit is not None:
            return hit
        v = self.views[index]
        packed, has_alpha = v.load_packed(self.alpha_mode, scale=self.image_scale)
        t = torch.from_numpy(np.ascontiguousarray(packed).view(np.int32))
        nbytes = t.numel() * 4
        depth, depth_count = None, 0
        if v.depth_path is not None:                        # the depth target at the image's size, |valid| counted here
            dm = v.load_depth(scale=self.image_scale)
            depth, depth_count = torch.from_numpy(dm), int(np.count_nonzero(dm))
            nbytes += depth.numel() * 4
        with self._lock:
            if self._cache[index] is not None:              # another loader task produced it meanwhile: one buffer per view
                return self._cache[index]
            admit = self._cache_used + nbytes < self._cache_budget
        if admit and torch.cuda.is_available():
            t = t.pin_memory()      # cached batches are uploaded many times: pin them once
            depth = depth.pin_memory() if depth is not None else None
        batch = SceneBatch(img_packed=t, camera=v.camera, has_alpha=has_alpha,
                           masked_alpha=has_alpha and self.alpha_mode == ALPHA_MASKED, depth=depth, depth_count=depth_count)
        if admit:
            with self._lock:
                if self._cache[index] is not None:
                    return self._cache[index]
                if self._cache_used + nbytes < self._cache_budget:
                    self._cache[index] = batch
                    self._cache_used += nbytes
        return batch

    def _run(self, seed: int):
        import queue
        rng = np.random.default_rng(seed)
        order: List[int] = []
        while not self._stop.is_set():
            if not order:
                order = list(rng.permutation(len(self.views)))
            try:
                batch = self._make_batch(int(order.pop()))
            except Exception as e:   # surface loader failures to the trainer instead of hanging it
                batch = e
            while not self._stop.is_set():
                try:
                    self._q.put(batch, timeout=0.1)
                    break
                except queue.Full:
                    continue

    def next_batch(self):
        b = self._q.get()
        if isinstance(b, Exception):
            raise b
        return b

    def close(self):
        self._stop.set()
        for t in self._threads:
            t.join(timeout=2.0)

    def __del__(self):
        try:
            self._stop.set()
        except Exception:
            pass
