"""bg_compress_splats on the device against the numpy restatement (tests/compress_ref.py), bit for bit; the file writer;
render quality of a re-imported model at 1080p; the training loop's compressed exports; the capacity check."""
import os
import sys

import numpy as np
import pytest

import compress_ref as cr
from brush_b200 import ply
from test_ply_compress_cpu import _model, _poison, _psnr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def _device(ctx, *arrays):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(x)).to(ctx.device) for x in arrays]


def _check_equal(enc, ref, k):
    m = ref["m"]
    assert int(enc.count.item()) == m
    assert np.array_equal(enc.order[:m].cpu().numpy(), ref["order"].astype(np.int32))
    c = (m + 255) // 256
    assert np.array_equal(enc.chunks[:c].cpu().numpy().view(np.uint32), ref["chunks"].view(np.uint32))
    assert np.array_equal(enc.packed[:m].cpu().numpy().view(np.uint32), ref["packed"])
    if k > 1:
        assert np.array_equal(enc.sh[:m].cpu().numpy(), ref["sh"])
    else:
        assert enc.sh is None


@pytest.mark.gpu
@pytest.mark.parametrize("n,k", [(n, k) for n in (1, 255, 256, 257, 4097) for k in (1, 4, 9, 16)] + [(1 << 20, 1), (1 << 20, 16)])
def test_device_encoding_equals_the_restatement(n, k):
    import brush_b200.render as R
    from brush_b200.compress import compress_splats
    t, sh, op = _model(n, k, seed=n + k, dup=n // 8)
    if n >= 8:
        _poison(t, sh, op, seed=n)
    ctx = R.RenderContext(n, 16, 16)
    enc = compress_splats(ctx, *_device(ctx, t, sh, op))
    _check_equal(enc, cr.encode(t, sh, op), k)
    ctx.close()


@pytest.mark.gpu
def test_same_call_twice_gives_identical_bytes():
    import brush_b200.render as R
    from brush_b200.compress import splat_to_compressed_ply
    t, sh, op = _model(100_000, 16, seed=4, dup=5000)
    _poison(t, sh, op)
    ctx = R.RenderContext(100_000, 16, 16)
    dt = _device(ctx, t, sh, op)
    a = splat_to_compressed_ply(ctx, *dt)
    b = splat_to_compressed_ply(ctx, *dt)
    assert a == b
    assert a == cr.encode_file(t, sh, op)
    assert splat_to_compressed_ply(ctx, *dt, render_mip=True) == cr.encode_file(t, sh, op, render_mip=True)
    ctx.close()


@pytest.mark.gpu
def test_empty_and_all_dropped():
    import torch
    import brush_b200.render as R
    from brush_b200.compress import splat_to_compressed_ply
    ctx = R.RenderContext(1000, 16, 16)
    t, sh, op = _model(300, 4, seed=8)
    t[:, 5] = np.nan
    assert splat_to_compressed_ply(ctx, *_device(ctx, t, sh, op)) == cr.encode_file(t, sh, op)
    z = torch.empty((0, 10), dtype=torch.float32, device=ctx.device)
    data = splat_to_compressed_ply(ctx, z, torch.empty((0, 4, 3), device=ctx.device), torch.empty(0, device=ctx.device))
    assert ply.load_splat_from_ply(data)[0].num_splats() == 0
    ctx.close()


@pytest.mark.gpu
def test_capacity_and_argument_errors():
    import ctypes
    import torch
    import brush_b200.render as R
    from brush_b200 import _lib
    from brush_b200.compress import compress_splats
    n = 5000
    ctx = R.RenderContext(1000, 16, 16, max_intersections=1000)   # sort capacity max(max_splats, max_intersections) < n
    with pytest.raises(_lib.BgError) as err:
        compress_splats(ctx, *_device(ctx, *_model(n, 4)))
    assert err.value.status == _lib.BG_ERR_CAPACITY
    compress_splats(ctx, *_device(ctx, *_model(1000, 4)))
    lib = _lib.load()
    a = _lib.BgCompressArgs()
    a.n, a.k = 10, 4
    out = torch.zeros(64, dtype=torch.int32, device=ctx.device)
    a.count_out = out.data_ptr()
    assert lib.bg_compress_splats(ctx.handle, None, ctypes.byref(a)) == _lib.BG_ERR_NULL   # arrays missing
    a.k = 5
    assert lib.bg_compress_splats(ctx.handle, None, ctypes.byref(a)) == _lib.BG_ERR_INVALID
    a.k, a.n = 4, 0
    assert lib.bg_compress_splats(ctx.handle, None, ctypes.byref(a)) == _lib.BG_OK
    torch.cuda.synchronize()
    ctx.close()


@pytest.mark.gpu
def test_render_of_the_reimported_model_1080p():
    """Measured: 42.92 dB (original against re-imported, rgb) for 1M synthetic splats at K = 16, 1920x1080."""
    import torch
    import brush_b200.render as R
    from brush_b200.compress import splat_to_compressed_ply
    from scenes import synthetic_scene
    n, w, h = 1_000_000, 1920, 1080
    cam, t, sh, op = synthetic_scene(n, w, h, k=16)
    ctx = R.RenderContext(n, w, h)
    dt = _device(ctx, t, sh, op)
    d, _ = ply.load_splat_from_ply(splat_to_compressed_ply(ctx, *dt))
    a = R.render_splats(ctx, cam, (w, h), *dt).out_img.cpu().numpy()
    b = R.render_splats(ctx, cam, (w, h), *_device(ctx, *d.into_arrays())).out_img.cpu().numpy()
    p = _psnr(a, b)
    print(f"psnr {p:.2f} dB")
    assert p > 40.0
    ctx.close()


@pytest.mark.gpu
def test_train_loop_exports_compressed_files(tmp_path):
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
    tr0, sh0, op0 = splat_init.to_init_splats(loaded.init_splat)
    sh0 = splat_init.with_sh_degree(sh0, 3)
    splats = T.Splats(*(torch.from_numpy(np.ascontiguousarray(x)).to(ctx.device) for x in (tr0, sh0, op0)))
    cfg = T.TrainConfig(total_train_iters=40, max_splats=15_000, refine_every=100, seed=1, lod_levels=1,
                        lod_refine_steps=10, lod_decimation_keep=50)
    out_dir = tmp_path / "out"
    counts = []
    train_loop(ctx, splats, loaded.train, [], cfg,
               ProcessConfig(export_every=20, export_path=str(out_dir), seed=7, export_compressed=True),
               on_step=lambda done, st, rf: counts.append(splats.num_splats()))
    files = sorted(os.listdir(out_dir))
    assert files == ["export_10_lod1.ply", "export_20.ply", "export_40.ply"], files
    for name in files:
        data = open(out_dir / name, "rb").read()
        assert data.split(b"\n")[2:4] == [b"comment Exported from Brush", b"comment Vertical axis: y"]
        assert b"element chunk " in data[:2000]
        d, meta = ply.load_splat_from_ply(data)
        assert d.num_splats() > 0 and d.sh_coeffs.shape[1] == 16 and np.all(np.isfinite(d.raw_opacities)), name
    assert ply.load_splat_from_ply(open(out_dir / "export_10_lod1.ply", "rb").read())[0].num_splats() == counts[-1]
    ctx.close()


def test_no_spill_in_compress_kernels():
    path = os.path.join(ROOT, "brush_b200", "csrc", "_obj", "compress.o.ptxas.txt")
    if not os.path.exists(path):
        from brush_b200 import build
        build.build(force=True)
    txt = open(path).read()
    assert txt.count("Compiling entry function") == 3
    assert " 0 bytes spill stores" in txt and all(ln.strip().startswith("0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads")
                                                  for ln in txt.splitlines() if "spill" in ln)
