"""Compressed PLY export without a GPU: the numpy restatement of the encoding (tests/compress_ref.py) against the
importer (ply.load_splat_from_ply, restated from import.rs), hand-computed words, the file layout, the ABI struct and
status codes, and the render quality of a re-imported model through the CPU oracle."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest

import compress_ref as cr
from brush_b200 import ply

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


def _model(n, k, seed=0, dup=0):
    rng = np.random.default_rng(seed)
    t = np.concatenate([rng.normal(0, 3, (n, 3)), rng.normal(size=(n, 4)), rng.uniform(-6, -1, (n, 3))], 1).astype(F)
    sh = np.concatenate([rng.uniform(-1.5, 1.5, (n, 1, 3)), rng.uniform(-0.5, 0.5, (n, k - 1, 3))], 1).astype(F)
    op = rng.uniform(-6, 6, n).astype(F)
    if dup:
        t[rng.integers(0, n, dup), 0:3] = t[0, 0:3]      # duplicate positions: equal Morton keys
    return t, sh, op


def _poison(t, sh, op, seed=1):
    """NaN mean, inf scale, NaN SH and a zero quaternion, each at a seeded row; returns the poisoned rows."""
    rows = np.random.default_rng(seed).choice(t.shape[0], 4, replace=False)
    t[rows[0], 1] = np.nan
    t[rows[1], 8] = np.inf
    sh[rows[2], -1, 2] = np.nan
    t[rows[3], 3:7] = 0.0
    return rows


def _check_roundtrip(t, sh, op, enc, data):
    d, meta = ply.load_splat_from_ply(data)
    m = enc["m"]
    assert d.num_splats() == m and meta.total_splats == m
    src = enc["order"]
    chunk = np.arange(m) // 256
    lo, hi = enc["chunks"][chunk, 0::2], enc["chunks"][chunk, 1::2]
    step = (hi - lo) / np.array([2047, 1023, 2047, 2047, 1023, 2047, 255, 255, 255], F)
    tol = 0.5 * step * (1 + 1e-5) + 1e-6 * np.maximum(np.abs(lo), np.abs(hi))
    rgb = sh[src, 0, :] * F(ply.SH_C0) + F(0.5)
    got_rgb = d.sh_coeffs[:, 0, :] * F(ply.SH_C0) + F(0.5)
    for got, want, sl in ((d.means, t[src, 0:3], slice(0, 3)), (d.log_scales, t[src, 7:10], slice(3, 6)), (got_rgb, rgb, slice(6, 9))):
        assert np.all(np.abs(got - want) <= tol[:, sl] + 1e-5 * (sl.start == 6)), sl
    assert np.all(np.isfinite(d.raw_opacities))
    sig = 1.0 / (1.0 + np.exp(-op[src].astype(np.float64)))
    got_sig = 1.0 / (1.0 + np.exp(-d.raw_opacities.astype(np.float64)))
    assert np.all(np.abs(got_sig - np.clip(sig, 1 / 255, 254 / 255)) <= 0.5 / 255 + 1e-6)
    q = t[src, 3:7].astype(np.float64)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    dq = d.rotations.astype(np.float64)
    sign = np.where(np.abs(dq - q).max(1) <= np.abs(dq + q).max(1), 1.0, -1.0)[:, None]
    err = np.abs(dq - sign * q)
    stored = np.ones_like(err, bool)
    stored[np.arange(m), enc["packed"][:, 1] >> 30] = False
    assert np.all(err[stored] <= 1.0 / 1023 / (0.5 * math.sqrt(2)))   # the 10-bit step of the three stored components
    assert np.all(err[~stored] <= 5e-3)                               # the largest follows from them (>= 1/2)
    k = sh.shape[1]
    if k > 1:
        rest = np.clip(sh[src, 1:, :], -4.0, (255 / 254 - 0.5) * 8)
        assert np.all(np.abs(d.sh_coeffs[:, 1:, :] - rest) <= 0.5 * 8 / 254 + 1e-6)
    return d


@pytest.mark.parametrize("k", [1, 4, 9, 16])
@pytest.mark.parametrize("n", [1, 255, 256, 257, 1000])
def test_restatement_reimports_within_half_a_step(n, k):
    t, sh, op = _model(n, k, seed=n * 31 + k, dup=n // 10)
    enc = cr.encode(t, sh, op)
    data = cr.encode_file(t, sh, op)
    _check_roundtrip(t, sh, op, enc, data)
    assert len(data) - data.index(b"end_header\n") - 11 == 72 * ((n + 255) // 256) + n * (16 + 3 * (k - 1))


def test_morton_keys_are_non_decreasing_in_output_order():
    t, sh, op = _model(5000, 4, seed=3, dup=300)
    enc = cr.encode(t, sh, op)
    keys = enc["keys"][enc["order"]]
    assert np.all(np.diff(keys.astype(np.int64)) >= 0) and keys.max() < cr.DROPPED_KEY
    ties = np.flatnonzero(np.diff(keys.astype(np.int64)) == 0)
    assert ties.size and np.all(enc["order"][ties] < enc["order"][ties + 1])   # ties in index order


@pytest.mark.parametrize("k", [1, 16])
def test_dropped_rows(k):
    t, sh, op = _model(700, k, seed=11)
    rows = _poison(t, sh, op)                            # at k == 1 the NaN coefficient is a DC one
    op[5] = -np.inf
    rows = np.append(rows, 5)
    enc = cr.encode(t, sh, op)
    assert enc["m"] == 700 - len(set(rows.tolist()))
    assert not set(rows.tolist()) & set(enc["order"].tolist())
    assert np.all(np.isfinite(enc["chunks"]))
    _check_roundtrip(t, sh, op, enc, cr.encode_file(t, sh, op))


def test_degenerate_chunk_and_empty_file():
    t, sh, op = _model(300, 4, seed=5)
    t[:] = t[0]
    sh[:] = sh[0]
    enc = cr.encode(t, sh, op)
    assert np.all(enc["chunks"][:, 0::2] == enc["chunks"][:, 1::2])
    assert np.all(enc["packed"][:, 0] == 0) and np.all(enc["packed"][:, 2] == 0)
    assert np.all(enc["packed"][:, 3] >> 8 == 0)
    d = _check_roundtrip(t, sh, op, enc, cr.encode_file(t, sh, op))
    np.testing.assert_array_equal(d.means, np.broadcast_to(t[0, 0:3], (300, 3)))
    t[:, 0] = np.nan                                     # every row dropped: a valid empty file
    data = cr.encode_file(t, sh, op)
    assert b"element chunk 0\n" in data and b"element vertex 0\n" in data and data.endswith(b"end_header\n")
    d, meta = ply.load_splat_from_ply(data)
    assert d.num_splats() == 0 and meta.total_splats == 0


def test_hand_computed_words_one_splat():
    t = np.array([[1.5, -2.0, 3.0, 0.0, 0.0, -2.0, 0.0, -1.0, -2.0, -3.0]], F)
    sh = np.array([[[0.1, 0.2, 0.3]]], F)
    enc = cr.encode(t, sh, np.zeros(1, F))
    # one row: every range is a point, so position, scale and colour quantise to 0; sigmoid(0) * 255 = 127.5 -> 128;
    # (0, 0, -1, 0): y is the largest, negated, the others 0 -> rint(0.5 * 1023) = 512
    assert enc["packed"].tolist() == [[0, 2 << 30 | 512 << 20 | 512 << 10 | 512, 0, 128]]
    np.testing.assert_array_equal(enc["chunks"][0, 0:6], [1.5, 1.5, -2.0, -2.0, 3.0, 3.0])


def test_hand_computed_words_two_splats():
    t = np.array([[1.0, 2.0, 4.0, 1.0, 0.0, 0.0, 0.0, -1.0, -1.0, -1.0],
                  [0.0, 0.0, 0.0, 0.6, 0.8, 0.0, 0.0, -1.0, -2.0, -3.0]], F)
    sh = np.zeros((2, 4, 3), F)
    sh[0, 0] = 1.0
    sh[0, 1:, 0] = (0.0, 1.0, -4.0)
    sh[0, 1:, 1] = (4.0, 5.0, -5.0)
    op = np.array([10.0, -20.0], F)
    enc = cr.encode(t, sh, op)
    assert enc["order"].tolist() == [1, 0]                # the origin has Morton key 0, the far corner 2^30 - 1
    assert enc["keys"].tolist() == [(1 << 30) - 1, 0]
    w_x = 0 << 30 | 512 << 20 | 512 << 10 | 512           # (1, 0, 0, 0)
    a = 946                                               # (0.6, 0.8, 0, 0): x is largest; rint((0.6 N + 0.5) 1023) = 945.5..
    assert enc["packed"].tolist() == [[0, 1 << 30 | a << 20 | 512 << 10 | 512, 0, 1],
                                      [0xFFFFFFFF, w_x, 0 << 21 | 1023 << 11 | 2047, 0xFFFFFF00 | 254]]
    # higher bands, channel-major: 0 -> 127, 1 -> 159 (158.75), -4 -> 0, 4 -> 254, 5 -> 255 (clamped), -5 -> 0
    assert enc["sh"][1].tolist() == [127, 159, 0, 254, 255, 0, 127, 127, 127]
    assert enc["sh"][0].tolist() == [127] * 9


def test_header_matches_the_decoder():
    t, sh, op = _model(600, 9, seed=2)
    data = cr.encode_file(t, sh, op, render_mip=True)
    fmt, comments, elements, off = ply._parse_header(data)
    assert fmt == "binary_little_endian"
    assert comments == ["Exported from Brush", "Vertical axis: y", "SH degree: 2", "SplatRenderMode: mip"]
    assert [(e[0], e[1]) for e in elements] == [("chunk", 3), ("vertex", 600), ("sh", 600)]
    assert [p[0] for p in elements[0][2]] == list(ply._QUANT_META_FIELDS) and {p[1] for p in elements[0][2]} == {"float"}
    assert elements[1][2] == [(nm, "uint") for nm in ("packed_position", "packed_rotation", "packed_scale", "packed_color")]
    assert elements[2][2] == [(f"f_rest_{i}", "uchar") for i in range(24)]
    d, meta = ply.load_splat_from_ply(data)
    assert meta.render_mip is True and meta.up_axis == (0.0, -1.0, 0.0) and d.sh_coeffs.shape == (600, 9, 3)
    assert b"element sh" not in cr.encode_file(*_model(10, 1))


def test_alpha_byte_uses_the_deterministic_exp():
    from oracle import oracle as orc
    x = np.linspace(-8, 8, 4001).astype(F)
    s = cr.det_sigmoid(x)
    ref = np.array([F(1.0) / (F(1.0) + F(orc.expf_det(float(-v)))) for v in x], F)
    np.testing.assert_array_equal(s, ref)
    a = np.clip(np.rint(s * F(255)), 1, 254)
    assert a.min() == 1 and a.max() == 254


def test_ctypes_layout_of_compress_args(tmp_path):
    from brush_b200 import _lib
    fields = ["n", "k", "transforms", "sh", "raw_opac", "chunks_out", "packed_out", "sh_out", "order_out", "count_out",
              "workspace", "workspace_bytes"]
    prog = ['#include <stdio.h>', '#include <stddef.h>', '#include "brush_b200.h"', 'int main(void){',
            'printf("%zu", sizeof(BgCompressArgs));'] + [f'printf(" %zu", offsetof(BgCompressArgs, {f}));' for f in fields]
    prog += ['printf("\\n"); return 0;}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(prog))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    tok = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert ctypes.sizeof(_lib.BgCompressArgs) == int(tok[0])
    for f, off in zip(fields, tok[1:]):
        assert getattr(_lib.BgCompressArgs, f).offset == int(off), f


def test_null_arguments_return_status_codes():
    from brush_b200 import _lib
    lib = _lib.load()
    a = _lib.BgCompressArgs()
    assert lib.bg_compress_splats(None, None, ctypes.byref(a)) == _lib.BG_ERR_NULL
    assert lib.bg_compress_splats(ctypes.c_void_p(8), None, None) == _lib.BG_ERR_NULL   # args checked before the context is used
    assert lib.bg_compress_workspace_bytes(1000) >= 16 * 1000


def _psnr(a, b):
    mse = float(np.mean((a[..., :3].astype(np.float64) - b[..., :3]) ** 2))
    return 10.0 * math.log10(1.0 / mse)


def test_render_of_the_reimported_model_cpu_oracle():
    """Measured: 42.64 dB (original against re-imported, rgb) for 20 000 synthetic splats at K = 16, 320x240."""
    from brush_b200.camera import build_uniforms
    from oracle import oracle as orc
    from scenes import synthetic_scene
    n, w, h = 20_000, 320, 240
    cam, t, sh, op = synthetic_scene(n, w, h, k=16)
    d, _ = ply.load_splat_from_ply(cr.encode_file(t, sh, op))
    t2, sh2, op2 = d.into_arrays()
    u = build_uniforms(cam, w, h)
    a = orc.render_forward(u, w, h, t, sh, op).out_img
    b = orc.render_forward(u, w, h, t2, sh2, op2).out_img
    p = _psnr(a, b)
    print(f"psnr {p:.2f} dB")
    assert p > 38.0
