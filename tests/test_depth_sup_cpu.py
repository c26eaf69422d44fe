"""Depth supervision on the host (DESIGN.md section 4.7): the restated term against finite differences, the depth maps of
the nerfstudio and COLMAP loaders, TrainConfig validation and the BgDepthSupervision layout.  No GPU needed."""
import json
import os

import numpy as np
import pytest

from depth_sup_ref import ALPHA_MIN, active_mask, fused_f32, grad_f64, loss_f64

from brush_b200 import dataset as ds
from brush_b200.camera import Camera


# ---------------------------------------------------------------------------------------------- the term
def _case(h=9, w=11, seed=3):
    rng = np.random.default_rng(seed)
    a = rng.uniform(0.05, 1.0, (h, w))
    t = rng.uniform(1.0, 5.0, (h, w))
    D = a * (t + rng.choice([-1.0, 1.0], (h, w)) * rng.uniform(0.2, 1.0, (h, w)))   # |ed - t| >= 0.2: away from the kink
    t[0, 0], t[0, 1], t[0, 2], t[0, 3] = 0.0, np.nan, np.inf, -2.0                   # invalid targets
    a[1, 0], a[1, 1] = 0.5 / 255.0, 0.0                                               # below the coverage threshold
    D[1, 1] = 0.0
    a[2, 0], D[2, 0] = 1.0, t[2, 0]                                                   # ed == t exactly
    return D, a, t


def test_restated_gradient_matches_central_differences():
    D, a, t = _case()
    chain = 0.37
    gD, ga = grad_f64(D, a, t, chain)
    act = active_mask(a, t)
    assert not act[0, :4].any() and not act[1, :2].any() and act[2, 0]
    assert gD[2, 0] == 0.0 and ga[2, 0] == 0.0                                        # sign(0) = 0
    eps = 1e-6
    for arr, g in ((D, gD), (a, ga)):
        for y in range(D.shape[0]):
            for x in range(D.shape[1]):
                p, m = arr.copy(), arr.copy()
                p[y, x] += eps
                m[y, x] -= eps
                args_p = (p, a, t) if arr is D else (D, p, t)
                args_m = (m, a, t) if arr is D else (D, m, t)
                num = (loss_f64(*args_p, chain) - loss_f64(*args_m, chain)) / (2 * eps)
                # at the kink (ed == t) the central difference of |.| in alpha is O(eps) instead of O(eps^2)
                kink = 2 * eps * chain * abs(t[y, x]) / a[y, x] ** 2 if (y, x) == (2, 0) else 0.0
                assert abs(num - g[y, x]) <= 1e-6 + 1e-6 * abs(g[y, x]) + kink, (y, x, num, g[y, x])
    # inactive pixels: no depth gradient and no alpha gradient
    assert (gD[~act] == 0).all() and (ga[~act] == 0).all()


def test_float32_restatement_agrees_with_float64():
    D, a, t = _case(40, 50, 9)
    img = np.zeros((40, 50, 4), np.float32)
    img[..., 3] = a
    v_out = np.random.default_rng(1).uniform(-1, 1, (40, 50, 4)).astype(np.float32)
    chain = 1.0 / 1234.0
    vd, vo, s = fused_f32(img, D.astype(np.float32), t.astype(np.float32), chain, v_out)
    gD, ga = grad_f64(D.astype(np.float32), a.astype(np.float32), t.astype(np.float32), chain)
    np.testing.assert_allclose(vd, gD, rtol=1e-6, atol=0)
    np.testing.assert_allclose(vo[..., 3] - v_out[..., 3], ga, rtol=1e-5, atol=1.2e-7)   # one ulp of |v_out| <= 1
    assert (vo[..., :3] == v_out[..., :3]).all()
    assert abs(s * chain - loss_f64(D.astype(np.float32), a.astype(np.float32), t.astype(np.float32), chain)) < 1e-6 * s * chain
    assert ALPHA_MIN == np.float32(1.0 / 255.0)


# ---------------------------------------------------------------------------------------------- datasets
IMG_W, IMG_H = 16, 12


def _img(path, w=IMG_W, h=IMG_H):
    from PIL import Image
    os.makedirs(os.path.dirname(path), exist_ok=True)
    Image.new("RGB", (w, h), (10, 20, 30)).save(path)


def _png16(path, arr):
    from PIL import Image
    os.makedirs(os.path.dirname(path), exist_ok=True)
    Image.fromarray(arr.astype(np.uint16)).save(path)


def _depth_mm(h, w, seed):
    rng = np.random.default_rng(seed)
    d = rng.integers(500, 5000, (h, w)).astype(np.uint16)
    d[0, 0] = 0                                          # no measurement
    return d


def _write_nerfstudio(root):
    for nm in ("a.png", "b.png", "c.png", "d.png"):
        _img(os.path.join(root, "images", nm))
    da = _depth_mm(IMG_H, IMG_W, 1)
    _png16(os.path.join(root, "depth", "a.png"), da)
    db = _depth_mm(IMG_H, IMG_W, 2).astype(np.float32)
    db[1, 1] = np.nan
    os.makedirs(os.path.join(root, "depth"), exist_ok=True)
    np.save(os.path.join(root, "depth", "b.npy"), db[..., None])          # [H,W,1]
    dd = _depth_mm(IMG_H // 2, IMG_W // 2, 4)                               # half the image's size
    _png16(os.path.join(root, "depth", "d.png"), dd)
    frames = [{"file_path": f"images/{nm}", "transform_matrix": [[1, 0, 0, float(i)], [0, 1, 0, 2.0], [0, 0, 1, 3.0], [0, 0, 0, 1]]}
              for i, nm in enumerate(("a.png", "b.png", "c.png", "d.png"))]
    frames[0]["depth_file_path"] = "depth/a.png"
    frames[1]["depth_file_path"] = "depth/b.npy"
    frames[2]["depth_file_path"] = "depth/missing.png"
    frames[3]["depth_file_path"] = "depth/d.png"
    json.dump({"camera_angle_x": 1.0, "frames": frames}, open(os.path.join(root, "transforms.json"), "w"))
    return da, db, dd


def test_nerfstudio_depth_maps(tmp_path):
    root = str(tmp_path)
    da, db, dd = _write_nerfstudio(root)
    r = ds.load_nerfstudio(root)
    by = {os.path.basename(v.image_path): v for v in r.train + r.eval}
    assert any("missing.png" in w for w in r.warnings)
    assert by["c.png"].depth_path is None and by["c.png"].load_depth() is None
    assert by["a.png"].depth_path == os.path.join(root, "depth", "a.png") and by["a.png"].depth_scale == 1e-3
    # PNG16 in millimetres -> metres; 0 stays "no measurement"
    got = by["a.png"].load_depth()
    assert got.dtype == np.float32 and got.shape == (IMG_H, IMG_W)
    np.testing.assert_array_equal(got, da.astype(np.float32) * np.float32(1e-3))
    assert got[0, 0] == 0.0
    # .npy [H,W,1] with a NaN: the NaN becomes 0
    gb = by["b.png"].load_depth()
    want = db * np.float32(1e-3)
    want[~np.isfinite(want) | (want <= 0)] = 0
    np.testing.assert_array_equal(gb, want)
    # a depth map at half the image's size: nearest upsampling, every source pixel becomes a 2x2 block
    gd = by["d.png"].load_depth()
    assert gd.shape == (IMG_H, IMG_W)
    np.testing.assert_array_equal(gd, np.repeat(np.repeat(dd.astype(np.float32) * np.float32(1e-3), 2, 0), 2, 1))
    # another unit scale
    r2 = ds.load_nerfstudio(root, depth_unit_scale_factor=0.5)
    v = next(v for v in r2.train if v.image_path.endswith("a.png"))
    np.testing.assert_array_equal(v.load_depth(), da.astype(np.float32) * np.float32(0.5))


@pytest.mark.parametrize("max_res,scale", [(None, 1.0), (10, 1.0), (None, 0.5), (None, 0.3), (12, 0.5)])
def test_depth_size_follows_load_image(tmp_path, max_res, scale):
    root = str(tmp_path)
    _write_nerfstudio(root)
    for v in ds.load_nerfstudio(root).train:
        if v.depth_path is None:
            continue
        img = v.load_image(max_res, scale)
        d = v.load_depth(max_res, scale)
        assert d.shape == img.shape[:2], (v.image_path, d.shape, img.shape)
        assert v.image_size(max_res, scale) == (img.shape[1], img.shape[0])


def test_nearest_resize_never_blends():
    src = np.array([[0.0, 2.0], [3.0, 4.0]], np.float32)
    up = ds.resize_nearest(src, 4, 4)
    assert set(np.unique(up)) <= set(np.unique(src))
    np.testing.assert_array_equal(up[:2, :2], 0.0)
    down = ds.resize_nearest(np.arange(36, dtype=np.float32).reshape(6, 6), 3, 3)
    np.testing.assert_array_equal(down, np.arange(36, dtype=np.float32).reshape(6, 6)[1::2, 1::2])


def test_multichannel_depth_is_rejected(tmp_path):
    from PIL import Image
    cam = Camera(position=(0.0, 0.0, 0.0), rotation=(0.0, 0.0, 0.0, 1.0), fov_x=1.0, fov_y=0.8)
    _img(str(tmp_path / "im.png"))
    Image.new("RGB", (IMG_W, IMG_H), (1, 2, 3)).save(tmp_path / "rgb.png")
    np.save(tmp_path / "rgb.npy", np.ones((IMG_H, IMG_W, 3), np.float32))
    for p in ("rgb.png", "rgb.npy"):
        v = ds.SceneView(cam, str(tmp_path / "im.png"), depth_path=str(tmp_path / p))
        with pytest.raises(ValueError):
            v.load_depth()
    # single-channel 8-bit and float TIFF decode
    Image.fromarray(np.full((IMG_H, IMG_W), 7, np.uint8), "L").save(tmp_path / "l.png")
    Image.fromarray(np.full((IMG_H, IMG_W), 2.5, np.float32), "F").save(tmp_path / "f.tif")
    v = ds.SceneView(cam, str(tmp_path / "im.png"), depth_path=str(tmp_path / "l.png"), depth_scale=0.5)
    np.testing.assert_array_equal(v.load_depth(), np.full((IMG_H, IMG_W), 3.5, np.float32))
    v = ds.SceneView(cam, str(tmp_path / "im.png"), depth_path=str(tmp_path / "f.tif"))
    np.testing.assert_array_equal(v.load_depth(), np.full((IMG_H, IMG_W), 2.5, np.float32))


def _write_colmap(root):
    sparse = os.path.join(root, "sparse", "0")
    os.makedirs(sparse)
    open(os.path.join(sparse, "cameras.txt"), "w").write(f"1 PINHOLE {IMG_W} {IMG_H} 20.0 20.0 8.0 6.0\n")
    open(os.path.join(sparse, "images.txt"), "w").write(
        "1 1.0 0.0 0.0 0.0 1.0 2.0 3.0 1 img0.jpg\n\n"
        "2 1.0 0.0 0.0 0.0 0.0 2.0 3.0 1 sub/img1.jpg\n\n"
        "3 1.0 0.0 0.0 0.0 0.0 0.0 3.0 1 img2.jpg\n\n")
    for nm in ("img0.jpg", "sub/img1.jpg", "img2.jpg"):
        _img(os.path.join(root, "images", nm))
    d0 = _depth_mm(IMG_H, IMG_W, 10)
    _png16(os.path.join(root, "Depths", "IMG0.PNG"), d0)                   # any case
    d1 = np.random.default_rng(11).uniform(0.5, 4.0, (IMG_H, IMG_W)).astype(np.float32)
    os.makedirs(os.path.join(root, "Depths", "sub"))
    np.save(os.path.join(root, "Depths", "sub", "img1.npy"), d1)
    _png16(os.path.join(root, "Depths", "other", "img2.png"), d0)         # wrong sub-directory: no match
    return d0, d1


def test_colmap_depth_maps(tmp_path):
    root = str(tmp_path)
    d0, d1 = _write_colmap(root)
    r = ds.load_colmap(root)
    by = {os.path.basename(v.image_path): v for v in r.train + r.eval}
    assert by["img0.jpg"].depth_path == os.path.join(root, "Depths", "IMG0.PNG")
    assert by["img1.jpg"].depth_path == os.path.join(root, "Depths", "sub", "img1.npy")
    assert by["img2.jpg"].depth_path is None
    np.testing.assert_array_equal(by["img0.jpg"].load_depth(), d0.astype(np.float32) * np.float32(1e-3))
    np.testing.assert_array_equal(by["img1.jpg"].load_depth(), d1 * np.float32(1e-3))   # .npy scaled alike
    r2 = ds.load_dataset(root, depth_unit_scale_factor=1.0)
    v = next(v for v in r2.train + r2.eval if v.image_path.endswith("img1.jpg"))
    np.testing.assert_array_equal(v.load_depth(), d1)
    assert by["img0.jpg"].load_depth(None, 0.5).shape == by["img0.jpg"].load_image(None, 0.5).shape[:2]


def test_colmap_image_never_resolves_to_its_depth_map(tmp_path):
    """A depth map may carry its image's file name (depths/view_0000.png next to images/view_0000.png): the image lookup
    must not pick it, although 'depths/...' sorts before 'images/...'."""
    root = str(tmp_path)
    _write_colmap(root)
    with open(os.path.join(root, "Depths", "img2.jpg"), "wb") as f:         # same name as the image itself
        f.write(b"not the image")
    assert ds.find_image_by_name(ds.list_files(root), "img2.jpg") == "images/img2.jpg"
    r = ds.load_colmap(root)
    v = next(v for v in r.train + r.eval if v.image_path.endswith("img2.jpg"))
    assert v.image_path == os.path.join(root, "images", "img2.jpg") and v.load_image().shape == (IMG_H, IMG_W, 3)


def test_find_depth_path_rules():
    files = ["depths/a.png", "depths/x/b.npy", "DEPTHS/c.NPY", "other/d.png", "depths/e.tiff", "depths/y/f.png"]
    assert ds.find_depth_path(files, "images/a.jpg") == "depths/a.png"
    assert ds.find_depth_path(files, "images/x/b.jpg") == "depths/x/b.npy"
    assert ds.find_depth_path(files, "b.jpg") is None                        # depths/x/ needs the image under x/
    assert ds.find_depth_path(files, "c.jpg") == "DEPTHS/c.NPY"
    assert ds.find_depth_path(files, "d.jpg") is None                        # not under depths/
    assert ds.find_depth_path(files, "e.jpg") is None                        # only .png and .npy
    assert ds.find_depth_path(files, "images/z/f.jpg") is None


# ---------------------------------------------------------------------------------------------- config and ABI
def test_train_config_depth_weight_validation():
    pytest.importorskip("torch")
    from brush_b200.train import TrainConfig
    assert TrainConfig().depth_loss_weight == 0.0
    assert TrainConfig(depth_loss_weight=0.5).depth_loss_weight == 0.5
    for bad in (-0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            TrainConfig(depth_loss_weight=bad)


def test_depth_supervision_struct_matches_the_c_header(tmp_path):
    import ctypes
    import subprocess
    from brush_b200 import _lib
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    names = [f for f, _ in _lib.BgDepthSupervision._fields_]
    assert names == ["target", "weight", "valid_count", "depth_loss_out"]
    prog = ['#include <stdio.h>', '#include <stddef.h>', '#include "brush_b200.h"', 'int main(void){',
            'printf("%zu", sizeof(BgDepthSupervision));'] + \
        [f'printf(" %zu", offsetof(BgDepthSupervision, {f}));' for f in names] + ['printf("\\n"); return 0; }']
    src, exe = tmp_path / "s.c", tmp_path / "s"
    src.write_text("\n".join(prog))
    r = subprocess.run(["gcc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    tok = [int(t) for t in subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()]
    assert tok[0] == ctypes.sizeof(_lib.BgDepthSupervision)
    assert tok[1:] == [getattr(_lib.BgDepthSupervision, f).offset for f in names]
    assert "bg_train_step_depth" in _lib.SIGNATURES and "bg_depth_loss_fused" in _lib.SIGNATURES
