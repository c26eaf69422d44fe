"""The bilateral grid of DESIGN.md section 4.11 without a GPU: the two float64 restatements against each other and
against central differences, the TV term, the learning-rate schedule, TrainConfig validation, the ABI struct layout
against the C compiler, and the status codes that come back before any device work."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import bilagrid_ref as ref

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _image(rng, h, w, lo=-0.2, hi=1.3):
    img = rng.uniform(lo, hi, (h, w, 4))
    img[..., 3] = rng.uniform(0.0, 1.0, (h, w))
    return img


@pytest.mark.parametrize("h,w", [(5, 7), (19, 33)])
def test_the_two_restatements_agree(h, w):
    rng = np.random.default_rng(h * 100 + w)
    grid, img, v_out = ref.random_grid(rng), _image(rng, h, w), rng.normal(size=(h, w, 4))
    a = ref.np_slice(grid, img)
    b = ref.torch_slice(torch.tensor(grid), torch.tensor(img)).numpy()
    np.testing.assert_allclose(a, b, rtol=0, atol=1e-12)
    vi_np, vg_np = ref.np_slice_backward(grid, img, v_out)
    vi_t, vg_t = ref.torch_slice_backward(grid, img, v_out)
    np.testing.assert_allclose(vi_np, vi_t, rtol=0, atol=1e-12)
    np.testing.assert_allclose(vg_np, vg_t, rtol=0, atol=1e-12)


def test_identity_grid_is_the_identity():
    rng = np.random.default_rng(3)
    img = _image(rng, 9, 11)
    np.testing.assert_allclose(ref.np_slice(ref.identity()[0], img), img, atol=1e-15)


def _loss(grid, img, v_out):
    return float((ref.np_slice(grid, img) * v_out).sum())


def test_grid_gradient_matches_central_differences():
    rng = np.random.default_rng(11)
    h, w = 6, 9
    grid, img, v_out = ref.random_grid(rng), _image(rng, h, w), rng.normal(size=(h, w, 4))
    _, vg = ref.np_slice_backward(grid, img, v_out)
    touched = np.argwhere(np.abs(vg) > 0)
    eps = 1e-6
    for idx in touched[rng.choice(len(touched), 40, replace=False)]:
        idx = tuple(idx)
        gp, gm = grid.copy(), grid.copy()
        gp[idx] += eps
        gm[idx] -= eps
        fd = (_loss(gp, img, v_out) - _loss(gm, img, v_out)) / (2 * eps)
        assert abs(fd - vg[idx]) < 1e-7 * max(1.0, abs(fd)), (idx, fd, vg[idx])


def test_colour_gradient_matches_central_differences_away_from_kinks():
    """The colour path (M^T v) and the guidance path through gray.  Pixels with gray within 1e-4 of a clamp or of a
    level boundary are excluded (the slice has a kink there); the test lists them and checks some remain on both
    sides of the clamps."""
    rng = np.random.default_rng(12)
    h, w = 7, 8
    grid, img, v_out = ref.random_grid(rng), _image(rng, h, w, -0.6, 1.6), rng.normal(size=(h, w, 4))
    img[0, 0, 0:3] = 0.0                            # gray exactly 0 and exactly 1: at the clamps
    img[0, 1, 0:3] = 1.0
    img[0, 2, 0:3] = 3.0 / 7.0                      # gray exactly on a level boundary
    vi, _ = ref.np_slice_backward(grid, img, v_out)
    excluded = ref.kink_mask(img, 1e-4)
    assert excluded[0, 0] and excluded[0, 1] and excluded[0, 2]
    gray = img[..., 0:3] @ ref.LUMA
    kept = ~excluded
    assert (kept & (gray > 0) & (gray < 1)).sum() > 10 and (kept & ((gray < 0) | (gray > 1))).sum() > 2
    eps = 1e-7
    for y, x in np.argwhere(kept):
        for ch in range(4):
            ip, im = img.copy(), img.copy()
            ip[y, x, ch] += eps
            im[y, x, ch] -= eps
            fd = (_loss(grid, ip, v_out) - _loss(grid, im, v_out)) / (2 * eps)
            assert abs(fd - vi[y, x, ch]) < 1e-6 * max(1.0, abs(fd)), (y, x, ch, fd, vi[y, x, ch])


def test_tv_value_and_gradient():
    rng = np.random.default_rng(13)
    grid = ref.random_grid(rng)
    val, grad = ref.np_tv(grid)
    tval, tgrad = ref.torch_tv(grid)
    assert abs(val - tval) < 1e-12 * max(1.0, tval)
    np.testing.assert_allclose(grad, tgrad, rtol=0, atol=1e-14)
    eps = 1e-6
    for idx in [(0, 0, 0, 0), (7, 15, 15, 11), (3, 8, 0, 5), (4, 0, 9, 2), (1, 2, 3, 4)]:
        gp, gm = grid.copy(), grid.copy()
        gp[idx] += eps
        gm[idx] -= eps
        fd = (ref.np_tv(gp)[0] - ref.np_tv(gm)[0]) / (2 * eps)
        assert abs(fd - grad[idx]) < 1e-8, (idx, fd, grad[idx])
    assert ref.np_tv(ref.identity()[0])[0] == 0.0
    assert ref.tv_counts() == (12 * 7 * 16 * 16, 12 * 8 * 15 * 16, 12 * 8 * 16 * 15)


def test_learning_rate_schedule():
    from brush_b200.bilagrid import bilagrid_lr
    total = 30000
    assert bilagrid_lr(2e-3, 1, total) == pytest.approx(2e-3 * 0.01, rel=1e-15)
    assert bilagrid_lr(2e-3, 1000, total) == pytest.approx(2e-3 * (0.01 + 0.99 * 999 / 1000) * 0.01 ** (999 / total), rel=1e-15)
    assert bilagrid_lr(2e-3, 1001, total) == pytest.approx(2e-3 * 0.01 ** (1000 / total), rel=1e-15)
    assert bilagrid_lr(2e-3, total, total) == pytest.approx(2e-3 * 0.01 ** ((total - 1) / total), rel=1e-15)
    assert bilagrid_lr(2e-3, 5000, total) < bilagrid_lr(2e-3, 1001, total)


def test_train_config_validation():
    from brush_b200.train import TrainConfig
    c = TrainConfig()
    assert (c.bilateral_grid, c.bilateral_grid_lr, c.bilateral_grid_tv_weight) == (False, 2e-3, 10.0)
    TrainConfig(bilateral_grid=True, bilateral_grid_lr=0.0, bilateral_grid_tv_weight=0.0)
    for kw in (dict(bilateral_grid_lr=-1e-3), dict(bilateral_grid_lr=math.nan), dict(bilateral_grid_tv_weight=-1.0),
               dict(bilateral_grid_tv_weight=math.inf), dict(bilateral_grid=1)):
        with pytest.raises(ValueError):
            TrainConfig(**kw)


def test_step_views_refuses_grids():
    from brush_b200.bilagrid import BilateralGrids
    from brush_b200.train import BoundingBox, SplatTrainer, TrainConfig
    grids = BilateralGrids(3, "cpu")
    assert grids.grids.shape == (3, 8, 16, 16, 12)
    np.testing.assert_array_equal(grids.grids.numpy(), ref.identity(3).astype(np.float32))
    tr = SplatTrainer(TrainConfig(bilateral_grid=True), None, BoundingBox(np.zeros(3), np.ones(3)), bilateral_grids=grids)
    for fn in (tr.step_views, tr.step_views_depth):
        with pytest.raises(ValueError, match="bilateral grids"):
            fn([], None)
    # the flag and the grids come together: either alone is refused
    with pytest.raises(ValueError, match="bilateral_grid"):
        SplatTrainer(TrainConfig(bilateral_grid=True), None, BoundingBox(np.zeros(3), np.ones(3)))
    with pytest.raises(ValueError, match="bilateral_grid"):
        SplatTrainer(TrainConfig(), None, BoundingBox(np.zeros(3), np.ones(3)), bilateral_grids=grids)
    with pytest.raises(ValueError):
        grids.check_view(3)
    with pytest.raises(ValueError):
        grids.check_view(-1)


def test_bilagrid_step_struct_matches_the_c_layout(tmp_path):
    from brush_b200 import _lib
    gcc = shutil.which("gcc") or shutil.which("cc")
    if gcc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "off.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "brush_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu %zu %zu %zu %d\\n", sizeof(BgBilagridStep),'
                   ' offsetof(BgBilagridStep, grid), offsetof(BgBilagridStep, m), offsetof(BgBilagridStep, v),'
                   ' offsetof(BgBilagridStep, step), offsetof(BgBilagridStep, lr), offsetof(BgBilagridStep, tv_weight),'
                   ' offsetof(BgBilagridStep, tv_loss_out), BG_BILAGRID_FLOATS); return 0; }\n')
    exe = tmp_path / "off"
    subprocess.run([gcc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    S = _lib.BgBilagridStep
    want = [C.sizeof(S)] + [getattr(S, f).offset for f in ("grid", "m", "v", "step", "lr", "tv_weight", "tv_loss_out")]
    assert got[:8] == want
    assert got[8] == _lib.BILAGRID_FLOATS == 8 * 16 * 16 * 12


def _lib_or_skip():
    from brush_b200 import _lib
    try:
        return _lib, _lib.load()
    except (ImportError, OSError) as e:
        pytest.skip(f"library not built: {e}")


def test_status_codes_come_back_without_a_device():
    _lib, lib = _lib_or_skip()
    fake_ctx = C.c_void_p(0x1000)          # never dereferenced: every call below fails its argument checks first
    p16, p4 = C.c_void_p(0x10000), C.c_void_p(0x10004)
    assert lib.bg_bilagrid_slice(None, None, p16, p16, 4, 4, p16) == _lib.BG_ERR_NULL
    assert lib.bg_bilagrid_slice(fake_ctx, None, None, p16, 4, 4, p16) == _lib.BG_ERR_NULL
    assert lib.bg_bilagrid_slice(fake_ctx, None, p4, p16, 4, 4, p16) == _lib.BG_ERR_INVALID
    assert lib.bg_bilagrid_slice_backward(fake_ctx, None, p16, p16, None, 4, 4, p16, p16) == _lib.BG_ERR_NULL
    assert lib.bg_bilagrid_slice_backward(fake_ctx, None, p16, p16, p16, 4, 4, p16, p4) == _lib.BG_ERR_INVALID
    # overlapping images, checked on their [h,w,4] extent: refused before any device work
    img, near, far = 0x100000, 0x100000 + 4 * 4 * 16 - 16, 0x100000 + 4 * 4 * 16
    assert lib.bg_bilagrid_slice(fake_ctx, None, p16, C.c_void_p(img), 4, 4, C.c_void_p(near)) == _lib.BG_ERR_INVALID
    assert lib.bg_bilagrid_slice_backward(fake_ctx, None, p16, C.c_void_p(img), C.c_void_p(far), 4, 4, C.c_void_p(near),
                                          p16) == _lib.BG_ERR_INVALID
    assert lib.bg_bilagrid_slice_backward(fake_ctx, None, p16, C.c_void_p(far), C.c_void_p(img), 4, 4, C.c_void_p(near),
                                          p16) == _lib.BG_ERR_INVALID

    def step(**kw):
        s = _lib.BgBilagridStep()
        s.grid, s.m, s.v, s.tv_loss_out = 0x10000, 0x20000, 0x30000, 0x40000
        s.step, s.lr, s.tv_weight = 1, 1e-3, 10.0
        for k, v in kw.items():
            setattr(s, k, v)
        return s

    upd = lambda s, vg=p16: lib.bg_bilagrid_update(fake_ctx, None, C.byref(s), vg)
    assert lib.bg_bilagrid_update(fake_ctx, None, None, p16) == _lib.BG_ERR_NULL
    assert upd(step(), None) == _lib.BG_ERR_NULL
    assert upd(step(m=None)) == _lib.BG_ERR_NULL
    assert upd(step(tv_loss_out=None)) == _lib.BG_ERR_NULL
    for bad in (dict(step=0), dict(step=-3), dict(lr=-1e-3), dict(lr=math.nan), dict(lr=math.inf), dict(tv_weight=-1.0),
                dict(tv_weight=math.nan), dict(grid=0x10004), dict(v=0x30008)):
        assert upd(step(**bad)) == _lib.BG_ERR_INVALID, bad
    assert upd(step(), p4) == _lib.BG_ERR_INVALID
    a = _lib.BgTrainStepArgs()
    assert lib.bg_train_step_bilagrid(fake_ctx, None, C.byref(a), None, None) == _lib.BG_ERR_NULL
    assert lib.bg_train_step_bilagrid(fake_ctx, None, C.byref(a), None, C.byref(step(step=0))) == _lib.BG_ERR_INVALID
    assert lib.bg_train_step_bilagrid(fake_ctx, None, C.byref(a), None, C.byref(step())) == _lib.BG_ERR_NULL   # args unset
    base = lib.bg_train_step_depth_workspace_bytes(1000, 16, 64, 48)
    assert lib.bg_train_step_bilagrid_workspace_bytes(1000, 16, 64, 48) >= base + 64 * 48 * 16 + 8 * 16 * 16 * 12 * 4
    # every pointer set (fake, never touched) and a workspace one byte short: capacity, before any launch
    for i, (name, _) in enumerate(_lib.BgTrainStepArgs._fields_):
        if name in ("transforms", "sh", "raw_opac", "m_t", "v_t", "m_sh", "v_sh", "m_o", "v_o", "refine_norm", "vis_weight",
                    "max_screen", "gt_packed", "loss_out"):
            setattr(a, name, 0x100000 * (i + 1))
    a.workspace, a.n, a.k, a.w, a.h, a.step, a.channels = 0x7000000, 1000, 16, 64, 48, 1, 3
    a.workspace_bytes = lib.bg_train_step_bilagrid_workspace_bytes(1000, 16, 64, 48) - 1
    assert lib.bg_train_step_bilagrid(fake_ctx, None, C.byref(a), None, C.byref(step())) == _lib.BG_ERR_CAPACITY
