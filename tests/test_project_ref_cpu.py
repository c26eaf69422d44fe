"""The float64 projection restatement (tests/project_ref.py) against the CPU oracle, against its own central
differences, and its ambiguity flags on hand-placed splats.  The GPU's projected rows are bit-equal to the oracle's
(test_gpu_parity), so the forward bound model is proven here, without a GPU; test_gpu_project_ref.py then holds the
kernels to it."""
import math

import numpy as np
import pytest

torch = pytest.importorskip("torch")

import project_ref as P  # noqa: E402
from scenes import synthetic_scene  # noqa: E402

MODELS = {"pinhole": P.PINHOLE, "kb4": P.KB4, "rt8": P.RT8, "tpf": P.TPF}
W, H = 256, 192


@pytest.fixture(scope="module")
def orc():
    from oracle import oracle
    return oracle


def _synthetic(model, k, seed, n=1200):
    from brush_b200.camera import Camera
    cam0, tr, sh, op = synthetic_scene(n, W, H, k=k, seed=seed)
    cam = Camera(position=cam0.position, rotation=cam0.rotation, fov_x=1.2, fov_y=1.0, center_uv=(0.42, 0.57),
                 camera_model=model, model_params=P.EDGE_PARAMS[model])
    return cam, tr, sh, op


def _scene(kind, model, k, seed):
    if kind == "edge":
        cam, tr, sh, op, _ = P.edge_scene(model, W, H, k, seed)
    else:
        cam, tr, sh, op = _synthetic(model, k, seed)
    return cam, tr, sh, op


def _rel_l2(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


@pytest.mark.parametrize("kind", ["synthetic", "edge"])
@pytest.mark.parametrize("k", [1, 4, 9, 16, 25])
@pytest.mark.parametrize("mip", [False, True])
@pytest.mark.parametrize("name", list(MODELS))
def test_forward_rows_vs_oracle(orc, name, mip, k, kind):
    from brush_b200.camera import build_uniforms
    model = MODELS[name]
    cam, tr, sh, op = _scene(kind, model, k, 0x9E0000 + 97 * model + k)
    u = build_uniforms(cam, W, H)
    o = orc.render_forward(u, W, H, tr, sh, op, mip=mip)
    ref = P.project_reference(u, W, H, tr, sh, op, mip=mip)
    assert o.num_visible > 0.5 * ref.visible.shape[0] * (0.5 if kind == "edge" else 1.0)
    assert ref.flags.mean() < 0.1
    worst, fails = P.forward_check(ref, o.projected, o.gid_from_cgid, o.max_radius)
    assert not fails, "\n".join(fails)
    # the render's compaction order is ascending depth (the f32 key of world_to_cam's z, ties by index): on the
    # splats whose visibility is not ambiguous, the same set, and float64 depths that never decrease by more than
    # the f32 error of the two keys (splats that close may swap)
    fl = ref.flags
    mine, theirs = ref.gid_from_cgid[~fl[ref.gid_from_cgid]], o.gid_from_cgid[~fl[o.gid_from_cgid]].astype(np.int64)
    assert mine.size > 0
    np.testing.assert_array_equal(np.sort(mine), np.sort(theirs))
    vm = np.asarray(u.viewmat, np.float64)
    Rv = vm[:9].reshape(3, 3).T
    za = (np.abs(tr[:, 0:3].astype(np.float64)) @ np.abs(Rv[2]) + abs(vm[11]))[theirs]
    d = ref.mc[theirs, 2]
    tol = 4 * P.U * (za[1:] + za[:-1])
    assert (d[1:] >= d[:-1] - tol).all(), np.nonzero(d[1:] < d[:-1] - tol)[0][:5]


def _backward_keep(ref, sh):
    """Splats whose backward is compared: not flagged, finite SH rows."""
    return ~ref.flags & np.isfinite(sh).reshape(sh.shape[0], -1).all(1)


@pytest.mark.parametrize("kind", ["synthetic", "edge"])
@pytest.mark.parametrize("k", [1, 4, 9, 16, 25])
@pytest.mark.parametrize("mip", [False, True])
@pytest.mark.parametrize("name", list(MODELS))
def test_vjp_vs_oracle(orc, name, mip, k, kind):
    from brush_b200.camera import build_uniforms
    model = MODELS[name]
    cam, tr, sh, op = _scene(kind, model, k, 0x9F0000 + 97 * model + k)
    u = build_uniforms(cam, W, H)
    o = orc.render_forward(u, W, H, tr, sh, op, mip=mip)
    V = o.num_visible
    rng = np.random.default_rng(model * 100 + k + 7 * mip)
    vc = rng.standard_normal((V, 10)).astype(np.float32)
    vc[:, 9] = np.abs(vc[:, 9])
    vc[rng.random(V) < 0.1] = 0.0                       # rows without a gradient are skipped
    ovt, ovsh, ovo, ovr = orc.project_backward(o, vc)
    ref = P.project_reference(u, W, H, tr, sh, op, mip=mip)
    vt, vsh, vo, vr, _ = P.project_reference_backward(u, W, H, tr, sh, op, o.gid_from_cgid, vc, mip=mip)
    keep = _backward_keep(ref, sh)
    # v_means within 1e-6 of the KB4 / TPF axis follow the kernel's derivative, not the reference's (DESIGN 2,
    # "Deviations"; test_kb4_vjp_on_the_axis below): those rows are compared in every other column
    keep_m = keep & ~ref.near_axis
    if kind == "edge":
        # needles (condition past 1e3), and in v_means the fisheye splats within 1e-5 z of the axis, carry f32
        # cancellation into the oracle's gradient (up to 1e-2 relative, measured); the GPU test holds the kernel to
        # the oracle's own error (needles) and to the stated cancellation bound (axis) on them instead
        r_axis = np.hypot(ref.mc[:, 0], ref.mc[:, 1])
        keep &= ref.m_conic < 1e3
        keep_m &= ref.m_conic < 1e3
        if model in (P.KB4, P.TPF):
            keep_m &= r_axis > 1e-5 * np.abs(ref.mc[:, 2])
    assert keep_m.sum() > 0.4 * V
    for nm, a, b in (("v_means", vt[keep_m, 0:3], ovt[keep_m, 0:3]), ("v_quats", vt[keep, 3:7], ovt[keep, 3:7]),
                     ("v_log_scales", vt[keep, 7:10], ovt[keep, 7:10]), ("v_sh", vsh[keep], ovsh[keep]),
                     ("v_raw_opac", vo[keep], ovo[keep])):
        # measured: 1e-7 .. 5e-7 on the synthetic scenes; the needles and clamped splats of the edge scenes carry
        # their condition number into the f32 oracle
        tol = 2e-6 if kind == "synthetic" else 3e-5   # edge: condition < 1e3 leaves 1e3 2^-24 = 6e-5
        assert _rel_l2(b, a) <= tol, f"{nm}: relative L2 {_rel_l2(b, a):.3e}"
    np.testing.assert_array_equal(vr, ovr)
    culled = np.ones(ref.visible.shape[0], bool)
    culled[o.gid_from_cgid] = False
    assert not vt[culled].any() and not vsh[culled].any() and not vo[culled].any()


@pytest.mark.parametrize("kind", ["synthetic", "edge"])
@pytest.mark.parametrize("k", [1, 4, 9, 16, 25])
@pytest.mark.parametrize("mip", [False, True])
@pytest.mark.parametrize("name", list(MODELS))
def test_autograd_vs_central_differences(name, mip, k, kind):
    """The restatement's backward against float64 central differences of its own forward, on every visible,
    unflagged splat with finite SH where the reference's backward is the derivative of its forward: all but RT8
    splats outside the clamp window (whose backward is the surrogate's, pinned by test_vjp_vs_oracle).  Under Mip the
    compensation is a constant to the geometry (project_backwards.rs:181-183), so the differences hold it fixed; the
    colour is differentiated unclamped.  Splats are independent, so one pair of perturbed forwards per parameter
    gives every splat's difference at once."""
    from brush_b200.camera import build_uniforms
    model = MODELS[name]
    cam, tr, sh, op = _scene(kind, model, k, 0xFD0000 + 97 * model + k)
    u = build_uniforms(cam, W, H)
    ref = P.project_reference(u, W, H, tr, sh, op, mip=mip)
    xr = ref.mc[:, 0] / ref.mc[:, 2]
    yr = ref.mc[:, 1] / ref.mc[:, 2]
    inside = (xr > u.lim_neg_x) & (xr < u.lim_pos_x) & (yr > u.lim_neg_y) & (yr < u.lim_pos_y)
    sel = ref.visible & ~ref.flags & np.isfinite(sh).reshape(sh.shape[0], -1).all(1)
    if model == P.RT8:
        sel &= inside
    gid = np.nonzero(sel)[0][:32]
    assert gid.size >= 24
    tr_s, sh_s, op_s = tr[gid], sh[gid], op[gid]
    m = gid.size
    rng = np.random.default_rng(5 + model + k)
    vc = rng.standard_normal((m, 10)).astype(np.float32)
    vt, vsh, vo, _, _ = P.project_reference_backward(u, W, H, tr_s, sh_s, op_s, np.arange(m), vc, mip=mip)
    vcw = torch.from_numpy(vc[:, :9].astype(np.float64))
    t0, s0, o0 = P._inputs(tr_s, sh_s, op_s)
    comp = P._forward(u, W, H, t0, s0, o0, mip, grad=False).comp.clone()

    def per_splat(t, s, o):
        f = P._forward(u, W, H, t, s, o, mip, grad=False)
        out = torch.stack([f.mean2d[:, 0], f.mean2d[:, 1], f.ca, f.cb, f.cc, f.col[:, 0], f.col[:, 1], f.col[:, 2],
                           f.sig * comp], -1)
        return (out * vcw).sum(1).numpy()

    def central(param, idx):
        base = {"t": t0, "s": s0, "o": o0}[param]
        h = 1e-6 * torch.clamp(base[idx].abs(), min=1.0)
        args = {"t": t0, "s": s0, "o": o0}
        p, q = base.clone(), base.clone()
        p[idx] += h
        q[idx] -= h
        lp = per_splat(**{kk: (p if kk == param else v) for kk, v in args.items()})
        lm = per_splat(**{kk: (q if kk == param else v) for kk, v in args.items()})
        return (lp - lm) / (2 * h.numpy())

    rows = np.arange(m)
    mag = np.maximum(np.abs(vt).max(1), 1.0)
    for j in range(10):
        fd = central("t", (rows, j))
        err = np.abs(fd - vt[:, j])
        assert (err <= 1e-5 * mag).all(), (j, int(gid[np.argmax(err / mag)]), float((err / mag).max()))
    for kk in sorted({0, k - 1}):
        for c in range(3):
            fd = central("s", (rows, kk, c))
            assert np.allclose(fd, vsh[:, kk, c], rtol=1e-6, atol=1e-6), (kk, c)
    fd = central("o", (rows,))
    assert np.allclose(fd, vo, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("name", ["kb4", "tpf"])
def test_kb4_vjp_on_the_axis(orc, name):
    """A splat exactly on the optical axis (DESIGN 2, "Deviations").  The reference's KB4 VJP (kannala_brandt_4.rs:
    154-337, transcribed by the oracle) contracts the fisheye Hessian at r = max(r, 1e-8): inv_r^5 = 1e40 overflows f32,
    0 * inf gives NaN, and the splat's mean gradient is NaN.  The restatement (like the kernel) differentiates the
    pinhole Jacobian the forward switched to for r < 1e-6, which is finite; every other column agrees with the oracle."""
    from brush_b200.camera import build_uniforms
    u = build_uniforms(P.edge_camera(MODELS[name], rotated=False), W, H)
    tr = np.array([[0.0, 0.0, 2.0, 0.9, 0.1, -0.2, 0.3, -2.0, -2.3, -2.6],
                   [0.2, 0.1, 3.0, 1.0, 0.0, 0.0, 0.0, -2.5, -2.5, -2.5]], np.float32)
    sh = np.full((2, 4, 3), 0.2, np.float32)
    op = np.array([2.0, 2.0], np.float32)
    o = orc.render_forward(u, W, H, tr, sh, op)
    assert o.num_visible == 2
    vc = np.random.default_rng(3).standard_normal((2, 10)).astype(np.float32)
    ovt, ovsh, ovo, _ = orc.project_backward(o, vc)
    vt, vsh, vo, _, _ = P.project_reference_backward(u, W, H, tr, sh, op, o.gid_from_cgid, vc)
    assert not np.isfinite(ovt[0, 0:3]).all()
    assert np.isfinite(vt[0]).all()
    np.testing.assert_allclose(vt[:, 3:10], ovt[:, 3:10], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(vt[1, 0:3], ovt[1, 0:3], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(vsh, ovsh, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(vo, ovo, rtol=1e-5, atol=1e-7)


def _one(u, mean_c, ls=(-2.5, -2.5, -2.5), q=(1.0, 0.0, 0.0, 0.0), ro=2.0, mip=False):
    """A single splat placed in camera space (identity camera), padded with a harmless second splat."""
    tr = np.array([[*mean_c, *q, *ls], [0.0, 0.0, 3.0, 1.0, 0.0, 0.0, 0.0, -2.5, -2.5, -2.5]], np.float32)
    sh = np.full((2, 1, 3), 0.3, np.float32)
    op = np.array([ro, 2.0], np.float32)
    return P.project_reference(u, W, H, tr, sh, op, mip=mip)


def _u(model):
    from brush_b200.camera import build_uniforms
    return build_uniforms(P.edge_camera(model, rotated=False), W, H)


@pytest.mark.parametrize("side", [-1.0, 1.0])
def test_flags_fire_on_each_side_of_each_threshold(side):
    e = side * 1e-8
    u0 = _u(P.PINHOLE)
    r = _one(u0, (0.0, 0.0, 0.01 * (1 + e)), ls=(-8, -8, -8))
    assert r.why["z"][0] and r.flags[0]
    assert not _one(u0, (0.0, 0.0, 0.01 * (1 + side * 1e-3)), ls=(-8, -8, -8)).why["z"][0]
    # |q|^2 = 1e-6
    qs = math.sqrt(1e-6 * (1 + e)) / 2
    assert _one(u0, (0.1, 0.1, 2.0), q=(qs, qs, qs, qs)).why["quat"][0]
    qs = math.sqrt(1e-6 * (1 + side * 1e-3)) / 2
    assert not _one(u0, (0.1, 0.1, 2.0), q=(qs, qs, qs, qs)).why["quat"][0]
    # opacity = 1/255: raw = logit(1/255) + a hair
    cut = -math.log(254.0)
    assert _one(u0, (0.1, 0.1, 2.0), ro=cut + side * 1e-7).why["opacity"][0]
    assert not _one(u0, (0.1, 0.1, 2.0), ro=cut + side * 1e-3).why["opacity"][0]
    # the Jacobian clamp limit, at both limits of x and y
    for lim, axis in ((u0.lim_pos_x, 0), (u0.lim_neg_x, 0), (u0.lim_pos_y, 1), (u0.lim_neg_y, 1)):
        p = [0.0, 0.0, 2.0]
        p[axis] = lim * 2.0 * (1 + e)
        assert _one(u0, p, ls=(0.5, 0.5, 0.5)).why["clamp"][0]
        p[axis] = lim * 2.0 * (1 + side * 1e-3)
        assert not _one(u0, p, ls=(0.5, 0.5, 0.5)).why["clamp"][0]
    # a screen edge: the footprint's left edge at x = 0 (placed by a fixed-point iteration on the extent)
    def left_edge(scale):
        x_px = 0.0
        for _ in range(30):
            r = _one(u0, ((x_px - u0.cx) / u0.fx * 2.0, 0.0, 2.0))
            ext = math.sqrt(2 * math.log(255 * r.rows[0, 5]) * r.rows[0, 4] / (r.rows[0, 2] * r.rows[0, 4] - r.rows[0, 3] ** 2))
            x_px = -ext * scale
        return _one(u0, ((x_px - u0.cx) / u0.fx * 2.0, 0.0, 2.0))
    assert left_edge(1 + side * 1e-9).why["screen"][0]
    assert not left_edge(1 + side * 1e-2).why["screen"][0]
    # distorted models: theta = half fov, and r = 1e-6 (KB4's switch to the pinhole form)
    u1 = _u(P.KB4)
    half = float(u1.half_max_render_fov)
    for th, want in ((half * (1 + e), True), (half * (1 + side * 1e-3), False)):
        assert bool(_one(u1, (3 * math.sin(th), 0.0, 3 * math.cos(th))).why["theta"][0]) == want
    for rr, want in ((1e-6 * (1 + e), True), (1e-6 * (1 + side * 1e-3), False)):
        assert bool(_one(u1, (rr, 0.0, 2.0)).why["axis"][0]) == want
    # det = 0: in float64 det(cov + blur I) >= blur^2 > 0, so the threshold is reached only by f32 rounding.  A rank-one
    # footprint of ~1e6 px^2 along the image diagonal (a flat splat turned 45 deg about z) puts blur (a + c) below
    # the f32 error of a c - b^2: flagged.  A round splat is not.
    c8, s8 = math.cos(math.pi / 8), math.sin(math.pi / 8)
    assert _one(u0, (0.0, 0.0, 2.0), ls=(2.3, -30.0, -30.0), q=(c8, 0.0, 0.0, s8)).why["det"][0]
    assert not _one(u0, (0.1, 0.1, 2.0)).why["det"][0]
    # the 1e18 rescale of cov2d: a round splat whose largest cov2d entry lands 3e-7 either side of 1e18 (placed by its
    # depth, whose f32 step moves the entry by ~2.4e-7), and 1e-3 either side
    def rescaled(rel):
        zz = 2.0
        for _ in range(40):
            t, sh_, o_ = P._inputs(np.array([[0.0, 0.0, zz, 1.0, 0.0, 0.0, 0.0, 16.0, 16.0, 16.0]], np.float32),
                                   np.zeros((1, 1, 3), np.float32), np.zeros(1, np.float32))
            with torch.no_grad():
                ma = float(P._forward(u0, W, H, t, sh_, o_, False, grad=False).max_abs[0])
            zz = float(np.float32(zz * math.sqrt(ma / (1e18 * (1 + rel)))))
        return _one(u0, (0.0, 0.0, zz), ls=(16.0, 16.0, 16.0)), ma
    r, ma = rescaled(side * 3e-7)
    assert r.why["rescale"][0], ma
    r, ma = rescaled(side * 1e-3)
    assert not r.why["rescale"][0] and (ma > 1e18) == (side > 0)


def test_sh_basis_is_orthonormal():
    """The restated basis is the real SH basis: orthonormal over the sphere (Lebedev-free check: a dense
    Fibonacci lattice, 1e-4)."""
    m = 20000
    i = np.arange(m) + 0.5
    zz = 1 - 2 * i / m
    ph = math.pi * (1 + 5 ** 0.5) * i
    rr = np.sqrt(1 - zz * zz)
    d = torch.tensor(np.stack([rr * np.cos(ph), rr * np.sin(ph), zz], 1))
    Y = P.sh_basis(d, 25).numpy()
    G = Y.T @ Y * (4 * math.pi / m)
    np.testing.assert_allclose(G, np.eye(25), atol=1e-4)
