"""Projection backward with its SH rows staged per warp in shared memory: the rows of 16-byte multiple length come in by
TMA bulk copy only for the splats that have a gradient, and the dense SH-gradient rows leave as one contiguous span per
warp.  The GPU tests pin every edge of that data movement against the CPU oracle (at test_backward_vs_oracle's
tolerances): ragged last warps and blocks, warps with 0, 1, 31 and 32 visible rows and alternating patterns, every SH
degree, Mip on and off, a distorted camera, and exact zeros in every output row of a culled splat, dense and factored.
The static tests read the build's ptxas report (no spill in any instantiation, the K = 16 pinhole kernel still fits 5
blocks per SM) and the shipped library's SASS (the K = 16 pinhole kernel issues UBLKCP)."""
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

torch = pytest.importorskip("torch")

from scenes import random_v_output, synthetic_scene  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
SH_C0 = 0.28209479177387814

# per-warp visibility patterns (True = the splat stays in front of the camera), cycled over the warps of a scene
_PATTERNS = [
    np.zeros(32, bool),                                   # no row read
    np.arange(32) == 7,                                   # one
    np.arange(32) != 13,                                  # 31
    np.ones(32, bool),                                    # all 32
    np.arange(32) % 2 == 0,                               # alternating
    np.arange(32) % 2 == 1,
    np.arange(32) < 16,                                   # one half
    np.arange(32) >= 31,                                  # last lane only
]


def _masked_scene(n, w, h, k, seed):
    """synthetic_scene with the splats a pattern marks off moved behind the camera (culled, zero gradient).  The
    pattern cycle starts at n mod 8, so that small scenes see more than the first patterns."""
    cam, tr, sh, op = synthetic_scene(n, w, h, k=k, seed=seed)
    keep = np.concatenate([_PATTERNS[(i + n) % len(_PATTERNS)] for i in range((n + 31) // 32)])[:n]
    tr = tr.copy()
    tr[~keep, 2] = -5.0
    return cam, tr, sh, op, keep


@pytest.fixture(scope="module")
def rt():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import brush_b200.render as R
    from brush_b200.camera import build_uniforms
    from oracle import oracle as orc

    class RT:
        pass

    r = RT()
    r.R, r.orc, r.build_uniforms = R, orc, build_uniforms
    r.ctx = R.RenderContext(max_splats=1 << 16, max_w=512, max_h=384, max_intersections=1 << 22)
    yield r
    r.ctx.close()


def _grad_close(g, r, rtol=1e-3, name=""):
    g = g.astype(np.float64)
    r = r.astype(np.float64)
    scale = max(np.abs(r).max(), 1e-30)
    err = np.abs(g - r)
    tol = rtol * np.abs(r) + 2e-5 * scale
    bad = err > tol
    assert bad.mean() <= 1e-4, f"{name}: {bad.sum()} of {bad.size} outside tol; max err {err.max():.3e} scale {scale:.3e}"
    l2 = np.linalg.norm(g - r) / max(np.linalg.norm(r), 1e-30)
    assert l2 <= 1e-3, f"{name}: relative L2 {l2:.3e}"


_CASES = [(k, mip, "pinhole", 4045) for k in (1, 4, 9, 16, 25) for mip in (False, True)]
_CASES += [(4, False, "kb4", 4045), (16, True, "kb4", 4045), (16, False, "pinhole", 37), (4, False, "pinhole", 100)]


@pytest.mark.gpu
@pytest.mark.parametrize("k,mip,model,n", _CASES)
def test_project_bwd_staging_vs_oracle(rt, k, mip, model, n):
    w, h = 256, 192
    cam, tr, sh, op, keep = _masked_scene(n, w, h, k, seed=0xB2003000 + 31 * k + n)
    if model == "kb4":
        from brush_b200.camera import KANNALA_BRANDT_4, Camera
        cam = Camera(position=cam.position, rotation=cam.rotation, fov_x=1.2, fov_y=1.0, center_uv=(0.48, 0.53),
                     camera_model=KANNALA_BRANDT_4, model_params=(-0.05, 0.01, -0.001, 5e-5))
    u = rt.build_uniforms(cam, w, h)
    o = rt.orc.render_forward(u, w, h, tr, sh, op, mip=mip)
    v_out = random_v_output(h, w)
    _, ovt, ovsh, ovo, ovr = rt.orc.render_backward(o, v_out)
    d = rt.ctx.device
    ttr, tsh, top = (torch.from_numpy(x).to(d) for x in (tr, sh, op))
    out = rt.R.render_splats(rt.ctx, cam, (w, h), ttr, tsh, top, mip=mip)
    assert out.num_visible == o.num_visible
    vc = rt.R.rasterize_bwd(out, torch.from_numpy(v_out).to(d))
    vt, vsh, vo, vr = (x.cpu().numpy() for x in rt.R.project_bwd(out, ttr, tsh, top, vc))
    ft, fcol, fo, fr = (x.cpu().numpy() for x in rt.R.project_bwd_factored(out, ttr, tsh, top, vc))

    _grad_close(vt[:, 0:3], ovt[:, 0:3], name="v_means")
    _grad_close(vt[:, 3:7], ovt[:, 3:7], name="v_quats")
    _grad_close(vt[:, 7:10], ovt[:, 7:10], name="v_log_scales")
    _grad_close(vsh, ovsh, name="v_sh")
    _grad_close(vo, ovo, name="v_raw_opac")
    _grad_close(vr, ovr, name="v_refine")
    # the factored pass shares the kernel: the same rows bit for bit, and v_color is the DC row of v_sh over Y_0
    np.testing.assert_array_equal(ft.view(np.uint32), vt.view(np.uint32))
    np.testing.assert_array_equal(fo.view(np.uint32), vo.view(np.uint32))
    np.testing.assert_array_equal(fr.view(np.uint32), vr.view(np.uint32))
    _grad_close(fcol * SH_C0, ovsh[:, 0, :], name="factored v_color")

    culled = ~keep
    assert culled.any() and keep.any()
    for name, arr in (("v_transforms", vt), ("v_sh", vsh), ("v_raw_opac", vo), ("v_refine", vr),
                      ("factored v_color", fcol)):
        rows = arr[culled].reshape(int(culled.sum()), -1)
        assert (rows.view(np.uint32) == 0).all(), f"{name}: a culled splat's row is not +0"
    # a splat with a gradient gets a non-zero SH-gradient row in every warp pattern that has one
    live = np.abs(ovsh).reshape(n, -1).max(1) > 0
    assert (np.abs(vsh).reshape(n, -1).max(1)[live] > 0).all()


# ---- static: ptxas report and SASS of the shipped library (no GPU needed)

def _mangled(mip, deg, dist):
    return f"_ZN2bg18project_bwd_kernelILb{int(mip)}ELi{deg}ELb{int(dist)}E"


@pytest.fixture(scope="module")
def ptxas_props():
    from brush_b200 import build
    build.build()
    txt = open(os.path.join(ROOT, "brush_b200", "csrc", "_obj", "project_bwd.o.ptxas.txt")).read()
    props = {}
    for m in re.finditer(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads\s+ptxas info\s+: Used (\d+) registers.*?(\d+) bytes smem", txt):
        if "project_bwd_kernel" in m.group(1):
            props[m.group(1)] = tuple(int(m.group(i)) for i in range(2, 7))
    return props


def test_project_bwd_kernels_do_not_spill(ptxas_props):
    assert len(ptxas_props) == 20, sorted(ptxas_props)
    for name, (stack, spill_st, spill_ld, _, _) in ptxas_props.items():
        assert (stack, spill_st, spill_ld) == (0, 0, 0), name


def test_project_bwd_k16_pinhole_fits_five_blocks_per_sm(ptxas_props):
    for mip in (False, True):
        (_, _, _, regs, smem), = [v for k, v in ptxas_props.items() if k.startswith(_mangled(mip, 3, False))]
        warp_regs = math.ceil(regs * 32 / 256) * 256          # registers are allocated per warp in 256-register units
        by_regs = (65536 // warp_regs) // 4                   # 4 warps per block
        by_smem = (228 * 1024) // (smem + 1024)               # sm_90: 228 KB per SM, 1 KB reserved per block
        assert min(by_regs, by_smem) >= 5, (mip, regs, smem)


def test_project_bwd_k16_pinhole_stages_sh_rows_with_tma(ptxas_props):
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not available")
    from brush_b200 import build
    lib = build.build()
    for mip in (False, True):
        name = [k for k in ptxas_props if k.startswith(_mangled(mip, 3, False))][0]
        sass = subprocess.run([CUOBJDUMP, "-sass", "-fun", name, lib], capture_output=True, text=True, timeout=600).stdout
        assert "Function : " + name in sass, name
        assert re.search(r"\bUBLKCP\b", sass), (name, "no TMA bulk copy")
