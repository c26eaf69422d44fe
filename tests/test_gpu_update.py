"""The fused parameter-update pass (csrc/update.cu) against its exact restatement tests/update_ref.py, and its
per-operator siblings (bg_refine_stats_noise, bg_adam_step, bg_normal_noise) against independent references.

Everything but the mean noise is compared bit for bit: the pass is compiled with -fmad=false and uses only correctly
rounded operations in a fixed order.  The noised means are compared within update_ref.noise_rel_tol of the increment
plus 2 ulp of the mean: the device forms the weight with expf and powf, which are not correctly rounded, and powf(., 150)
multiplies the relative error of 1 - opacity by 150."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import update_ref as U  # noqa: E402

STATE = ("transforms", "sh", "raw_opac", "m_t", "v_t", "m_sh", "v_sh", "m_o", "v_o", "refine_norm", "vis_weight", "max_screen")
GRADS = ("v_transforms", "v_sh_grad", "v_raw_opac", "v_refine", "visible", "max_radius")
LRS = dict(lr_mean=3.1e-5, lr_rotation=2e-3, lr_scale=5e-3, lr_coeffs_dc=2e-3, lr_coeffs_sh_scale=20.0, lr_opac=0.012)
SEED = 0x1234_5678_9ABC_DEF0   # non-zero high word: both key words of the Philox stream matter


@pytest.fixture(scope="module")
def rt():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import brush_b200.render as R
    import brush_b200.train as T
    from brush_b200 import _lib
    from oracle import oracle as orc

    class RT:
        pass

    r = RT()
    r.R, r.T, r._lib, r.orc, r.lib = R, T, _lib, orc, _lib.load()
    r.ctx = R.RenderContext(max_splats=1 << 16, max_w=256, max_h=256)
    r.dev = r.ctx.device
    yield r
    r.ctx.close()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _dev(rt, d):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(rt.dev) for k, v in d.items()}


def _host(d):
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in d.items()}


def _args(rt, st, gr, step, noise_scale=0.0, median_scale=0.0, min_scale=None, seed=SEED, ptr=None):
    a = rt._lib.BgTrainUpdateArgs()
    a.n, a.k = st["transforms"].shape[0], st["sh"].shape[1]
    ptr = ptr or (lambda t: t.data_ptr())
    for key in STATE:
        setattr(a, key, ptr(st[key]))
    for key in GRADS:
        setattr(a, key, ptr(gr[key]))
    for key, v in LRS.items():
        setattr(a, key, v)
    a.noise_scale, a.median_scale, a.seed, a.step = noise_scale, median_scale, seed, step
    a.min_scale = min_scale.data_ptr() if min_scale is not None else None
    return a


def _update(rt, st, gr, step, **kw):
    return rt.lib.bg_train_update(rt.ctx.handle, _stream(), C.byref(_args(rt, st, gr, step, **kw)))


def _noise(rt, seed, offset, count):
    z = torch.empty(max(count, 1), dtype=torch.float32, device=rt.dev)
    rt._lib.check(rt.lib.bg_normal_noise(rt.ctx.handle, _stream(), seed, offset, count, z.data_ptr()), "bg_normal_noise")
    torch.cuda.synchronize()
    return z[:count].cpu().numpy()


def _step_noise(rt, n, step, seed=SEED):
    """The draw of the pass (brush_b200.h): bg_normal_noise(seed, (step-1)*ceil(3n/4), 3n), as [n,3]."""
    return _noise(rt, seed, (step - 1) * ((3 * n + 3) // 4), 3 * n).reshape(n, 3)


def _bitwise(got, want, keys, where):
    for key in keys:
        g, w = np.ascontiguousarray(got[key]).reshape(-1).view(np.uint32), np.ascontiguousarray(want[key]).reshape(-1).view(np.uint32)
        bad = np.nonzero(g != w)[0]
        assert bad.size == 0, (where, key, f"{bad.size} of {g.size} differ; first at {bad[0]}",
                               g[bad[0]:bad[0] + 1].view(np.float32), w[bad[0]:bad[0] + 1].view(np.float32))


NS = [1, 3, 4, 31, 32, 36, 129, 4100, 100_003]


@pytest.mark.parametrize("k", [1, 4, 9, 16, 25])
@pytest.mark.parametrize("n", NS)
def test_train_update_is_bit_exact(rt, n, k):
    """Six consecutive steps on one state, noise off: every output array equals update_ref.update_f32 bit for bit after
    every step, and the parameters stay within the derived float64 bound of AdamScaled.  The N cover the SH load/update
    branches at every degree: full warps; a partial last warp with float4 access when (N mod 32) 3K = 0 mod 4; scalar
    access otherwise (K in {1, 9, 25} with N mod 32 not a multiple of 4)."""
    rng = np.random.default_rng(n * 31 + k)
    st = U.random_state(n, k, rng)
    dst = _dev(rt, st)
    ref64 = U.Adam64(st, U.Consts(1, **LRS))
    for step in range(1, 7):
        gr = U.random_grads(n, k, rng)
        rt._lib.check(_update(rt, dst, _dev(rt, gr), step), "bg_train_update")
        c = U.Consts(step, **LRS)
        st, _ = U.update_f32(st, gr, c)
        got = _host(dst)
        _bitwise(got, st, STATE, (n, k, step))
        ref64.step_and_check(gr, c, got)


@pytest.mark.parametrize("n,k", [(36, 4), (129, 25), (4100, 9), (31, 1)])
def test_first_step_ignores_the_moment_buffers(rt, n, k):
    """step == 1 initialises the moments from the gradient alone: NaN in every m_* / v_* gives the zero-start result."""
    rng = np.random.default_rng(n + k)
    st, gr = U.random_state(n, k, rng), U.random_grads(n, k, rng)
    runs = []
    for fill in (0.0, np.nan):
        s = dict(st)
        for key in ("m_t", "v_t", "m_sh", "v_sh", "m_o", "v_o"):
            s[key] = np.full_like(st[key], fill)
        d = _dev(rt, s)
        rt._lib.check(_update(rt, d, _dev(rt, gr), 1, noise_scale=0.03, median_scale=0.01), "bg_train_update")
        runs.append(_host(d))
    _bitwise(runs[1], runs[0], STATE, (n, k))


def _noise_state(n, k, rng, floor):
    st = U.random_state(n, k, rng)
    st["raw_opac"] = rng.uniform(-9.0, 1.0, n).astype(np.float32)            # weights from ~1 down to 0
    st["transforms"][:, 7:10] = np.log(rng.uniform(1e-4, 0.2, (n, 3)))        # some splats far thinner than the floor
    for key, scale in (("m_t", 1e-3), ("m_sh", 1e-3), ("m_o", 1e-2)):
        st[key] = (rng.normal(size=st[key].shape) * scale).astype(np.float32)
    for key, scale in (("v_t", 1e-6), ("v_sh", 1e-6), ("v_o", 1e-4)):
        st[key] = (rng.uniform(0.1, 1.0, st[key].shape) * scale).astype(np.float32)
    f = rng.uniform(0.002, 0.05, n).astype(np.float32) if floor else None
    return st, f


def _check_noised(got, want, info, visible, where):
    """Bitwise outside the noised means; the noised means within 2 ulp + noise_rel_tol |inc|; the clamp exact."""
    _bitwise(got, want, [x for x in STATE if x != "transforms"], where)
    _bitwise({"t": got["transforms"][:, 3:]}, {"t": want["transforms"][:, 3:]}, ["t"], where)
    noised = info["noised"]
    _bitwise({"m": got["transforms"][~noised, :3]}, {"m": want["transforms"][~noised, :3]}, ["m"], where)
    _bitwise({"m": got["transforms"][visible <= 0, :3]}, {"m": info["mean_adam"][visible <= 0]}, ["m"], where)   # Adam only
    g, w, inc = got["transforms"][noised, :3].astype(np.float64), want["transforms"][noised, :3], info["inc"][noised]
    tol = 2 * np.spacing(np.abs(w)).astype(np.float64) + info["rel_tol"][noised, None] * np.abs(inc) + 2.0 ** -140
    assert (np.abs(g - w) <= tol).all(), (where, float((np.abs(g - w) / tol).max()))
    return noised


@pytest.mark.parametrize("floor", [False, True])
def test_mean_noise_matches_restatement(rt, floor):
    """Noise on, visibilities 0 / 1 / 2, opacities from ~0 to ~0.73, three steps; with a floor the gate is the folded
    opacity.  Some rows reach the clamp (exactly +-median there), invisible rows carry Adam's change only."""
    n, k = 4100, 9
    rng = np.random.default_rng(17 + floor)
    st, f = _noise_state(n, k, rng, floor)
    dst, df = _dev(rt, st), (torch.from_numpy(f).to(rt.dev) if floor else None)
    ns, med = 0.05, 0.01
    clamped_rows = 0
    for step in (1, 2, 3):
        gr = U.random_grads(n, k, rng)
        gr["v_transforms"] *= np.float32(1e-20)      # Adam keeps the means put; the noise is what moves them
        before = _host(dst)
        rt._lib.check(_update(rt, dst, _dev(rt, gr), step, noise_scale=ns, median_scale=med, min_scale=df), "bg_train_update")
        c = U.Consts(step, **LRS, noise_scale=ns, median_scale=med)
        want, info = U.update_f32(before, gr, c, z=_step_noise(rt, n, step), min_scale=f)
        got = _host(dst)
        noised = _check_noised(got, want, info, gr["visible"], (floor, step))
        assert noised.sum() > n // 10 and (gr["visible"][noised] > 0).all() and (gr["visible"][noised] == 2).any()
        rows, cols = np.nonzero(np.abs(info["unclamped"]) > 1.01 * med)   # well past the clamp: exactly +-median
        want_c = info["mean_adam"][rows, cols] + np.sign(info["inc"][rows, cols]).astype(np.float32) * np.float32(med)
        assert np.array_equal(got["transforms"][rows, cols].view(np.uint32), want_c.astype(np.float32).view(np.uint32))
        clamped_rows += rows.size
    assert clamped_rows > 100
    if floor:   # the fold matters: thin splats the plain sigmoid would give (almost) no noise
        w_plain = U.noise_weight64(got["raw_opac"], got["transforms"][:, 7:10], gr["visible"])
        w_fold = U.noise_weight64(got["raw_opac"], got["transforms"][:, 7:10], gr["visible"], f)
        assert ((w_fold > 1e-3) & (w_plain < 1e-6 * w_fold)).sum() > 50


def test_mean_noise_stream_offset_past_2_to_the_32(rt):
    """At N = 100 003 and step 60 000 the draw starts at counter 59 999 * 75 001 > 2^32: the high counter word."""
    n, k, step = 100_003, 1, 60_000
    assert (step - 1) * ((3 * n + 3) // 4) > 2 ** 32
    rng = np.random.default_rng(60)
    st, _ = _noise_state(n, k, rng, False)
    gr = U.random_grads(n, k, rng)
    gr["v_transforms"] *= np.float32(1e-20)
    dst = _dev(rt, st)
    rt._lib.check(_update(rt, dst, _dev(rt, gr), step, noise_scale=0.05, median_scale=0.01), "bg_train_update")
    want, info = U.update_f32(st, gr, U.Consts(step, **LRS, noise_scale=0.05, median_scale=0.01), z=_step_noise(rt, n, step))
    assert _check_noised(_host(dst), want, info, gr["visible"], "offset").sum() > n // 10


def _normal_ref(seed, offset, count):
    """Philox4x32-10 (the numpy restatement pinned by the Random123 known answers in test_refine_cpu.py) on counter
    (offset + q) as (lo, hi, 0, 0) with key (seed lo, seed hi), uniforms ((x >> 8) + 0.5) 2^-24 rounded as in f32, then
    Box-Muller in float64: z = (r0 cos 2pi u1, r0 sin 2pi u1, r1 cos 2pi u3, r1 sin 2pi u3), r = sqrt(-2 log u)."""
    import test_gpu_refine as tgr
    quads = (count + 3) // 4
    ctr = np.uint64(offset) + np.arange(quads, dtype=np.uint64)
    m32 = np.uint64(0xFFFFFFFF)
    r = tgr.philox4x32_10(ctr & m32, ctr >> np.uint64(32), np.zeros(quads, np.uint64), np.zeros(quads, np.uint64),
                          seed & 0xFFFFFFFF, seed >> 32)
    u = [((x >> np.uint64(8)).astype(np.float32) + np.float32(0.5)) * np.float32(1.0 / 16777216.0) for x in r]
    u = [x.astype(np.float64) for x in u]
    r0, r1 = np.sqrt(-2.0 * np.log(u[0])), np.sqrt(-2.0 * np.log(u[2]))
    z = np.stack([r0 * np.cos(2 * np.pi * u[1]), r0 * np.sin(2 * np.pi * u[1]), r1 * np.cos(2 * np.pi * u[3]),
                  r1 * np.sin(2 * np.pi * u[3])], 1).reshape(-1)
    return z[:count]


@pytest.mark.parametrize("offset", [0, 1, 2 ** 32 - 1, 2 ** 32 + 5])
@pytest.mark.parametrize("count", [1, 3, 5, 2_200_003])
def test_normal_noise_known_answers(rt, offset, count):
    """bg_normal_noise against the numpy Philox and a float64 Box-Muller.  logf, sincospif <= 1 ulp, sqrtf and the
    product correctly rounded: <= 4 ulp of z.  2 200 003 draws run the grid-stride loop (more quads than 2112 x 256)."""
    got = _noise(rt, SEED, offset, count).astype(np.float64)
    want = _normal_ref(SEED, offset, count)
    np.testing.assert_allclose(got, want, rtol=2.0 ** -21, atol=1e-37)


def _floor_scene(rt, n, k, seed):
    """synthetic_scene with every 8th splat made mid-opacity (sigmoid 0.5) and 50x thinner than its floor on one axis:
    folded opacity ~0.01, weight (0.99)^150 ~ 0.2 instead of 0.5^150 ~ 7e-46."""
    from scenes import synthetic_scene
    w, h = 192, 128
    cam, tr, sh, op = synthetic_scene(n, w, h, k=k, seed=seed)
    focal = 0.5 * w / np.tan(0.5 * cam.fov_x)
    cams = torch.tensor([[*cam.position, focal]], dtype=torch.float32, device=rt.dev)
    f = rt.T.compute_min_scale(rt.ctx, torch.from_numpy(tr).to(rt.dev), cams, rt.T.MIN_SCALE_FACTOR).cpu().numpy()
    thin = np.arange(0, n, 8)
    tr[thin, 9] = np.log(0.02 * f[thin])
    op[thin] = 0.0
    return cam, tr, sh, op, focal, (w, h)


def test_step_gates_the_noise_on_the_folded_opacity(rt):
    """End to end through SplatTrainer.step with a floor: a refine (N not a multiple of 32, floor recomputed), then
    three steps.  The exact inputs of each update are captured by grad_hook; the result equals the restatement (bitwise
    outside the noise, noise_rel_tol on the noised means) with the floor folded into the gate."""
    T = rt.T
    n, k = 3000, 4
    cam, tr, sh, op, focal, (w, h) = _floor_scene(rt, n, k, 5)
    d = rt.dev
    tgt = rt.R.render_splats(rt.ctx, cam, (w, h), *(torch.from_numpy(x).to(d) for x in (tr, sh, op)), rpass=0)
    batch = T.SceneBatch(img_packed=(tgt.out_img | (255 << 24)).clone(), camera=cam)
    cfg = T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, max_splats=n + 5, growth_grad_threshold=0.0,
                        seed=SEED & 0x7FFFFFFF)
    s = T.Splats(*(torch.from_numpy(x.copy()).to(d) for x in (tr, sh + 0.1, op)))
    cap = {}

    def hook(g):
        a = type("A", (), {})()
        t._fill_schedule(a, t.bounds.median_size())
        cap.update(grads=[x.clone() for x in g], args=a, min_scale=s.min_scale.clone(),
                   state={**{x: v.clone() for x, v in t._state.items()},
                          "transforms": s.transforms.clone(), "sh": s.sh_coeffs.clone(), "raw_opac": s.raw_opacities.clone()})

    t = T.SplatTrainer(cfg, rt.ctx, T.bounds_from_pos(0.8, tr[:, :3]), grad_hook=hook)
    t.set_view_cams([(cam.position, focal)])
    s.min_scale = T.compute_min_scale(rt.ctx, s.transforms, t.view_cams, T.MIN_SCALE_FACTOR)
    t.step(batch, s)
    t.refine(1, s)
    n1 = s.num_splats()
    assert n1 % 32 != 0 and s.min_scale is not None and s.min_scale.shape[0] == n1
    # the refine baked the floor into the parameters: make every 8th splat thin and mid-opacity again
    thin = torch.arange(0, n1, 8, device=d)
    s.transforms[thin, 9] = torch.log(0.02 * s.min_scale[thin])
    s.raw_opacities[thin] = 0.0
    folded = 0
    for _ in range(3):
        t.step(batch, s)
        torch.cuda.synchronize()
        a = cap["args"]
        st = {x: v.cpu().numpy() for x, v in cap["state"].items()}
        st["m_sh"] = st["m_sh"].reshape(n1, k, 3)
        gr = dict(zip(GRADS, (x.cpu().numpy() for x in cap["grads"])))
        gr["v_sh_grad"] = gr["v_sh_grad"].reshape(n1, k, 3)
        f = cap["min_scale"].cpu().numpy()
        c = U.Consts(a.step, a.lr_mean, a.lr_rotation, a.lr_scale, a.lr_coeffs_dc, a.lr_coeffs_sh_scale, a.lr_opac,
                     a.noise_scale, a.median_scale)
        want, info = U.update_f32(st, gr, c, z=_step_noise(rt, n1, a.step, a.seed), min_scale=f)
        got = {"transforms": s.transforms, "sh": s.sh_coeffs, "raw_opac": s.raw_opacities, **t._state}
        got = {x: v.cpu().numpy() for x, v in got.items()}
        _check_noised(got, want, info, gr["visible"], ("step", a.step))
        # rows whose noise is visible at f32 precision only because of the fold
        w_plain = U.noise_weight64(want["raw_opac"], want["transforms"][:, 7:10], gr["visible"])
        moved = np.abs(info["inc"]).max(1) > 8 * np.spacing(np.abs(want["transforms"][:, :3])).max(1)
        folded += int((moved & (w_plain * float(c.noise_scale) * 8 < np.spacing(np.abs(want["transforms"][:, :3])).min(1))).sum())
    assert folded > 20, folded


def test_step_views_gates_the_noise_on_the_folded_opacity(rt):
    """step_views with one rank (the factored update) and a floor, against the sequential definition: per-view dense
    gradients averaged, then the update pass.  The noise of the thin mid-opacity splats is checked row by row against
    the folded-gate increment of the restatement; a whole-array criterion would not see them."""
    import math as m
    from brush_b200.camera import Camera
    T = rt.T
    n, k = 20_000, 9
    cam0, tr, sh, op, focal, (w, h) = _floor_scene(rt, n, k, 21)
    a = m.radians(4.0) / 2.0
    cam1 = Camera(position=(0.1, -0.05, 0.0), rotation=(0.0, m.sin(a), 0.0, m.cos(a)), fov_x=cam0.fov_x, fov_y=cam0.fov_y,
                  center_uv=cam0.center_uv)
    d = rt.dev
    params = [torch.from_numpy(x.copy()).to(d) for x in (tr, sh, op)]
    batches = []
    for cam in (cam0, cam1):
        tgt = rt.R.render_splats(rt.ctx, cam, (w, h), *params, rpass=0)
        batches.append(T.SceneBatch(img_packed=(tgt.out_img | (255 << 24)).clone(), camera=cam))
    bounds = T.bounds_from_pos(0.8, tr[:, :3])
    cams = torch.tensor([[*cam0.position, focal], [*cam1.position, focal]], dtype=torch.float32, device=d)
    floor = T.compute_min_scale(rt.ctx, params[0], cams, T.MIN_SCALE_FACTOR)
    fresh = lambda: T.Splats(params[0].clone(), params[1] + 0.1, params[2].clone(), min_scale=floor.clone())
    cfg = T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, seed=11)
    cfg0 = T.TrainConfig(total_train_iters=1000, background_noise_strength=0.0, seed=11, mean_noise_weight=0.0)
    captured = {}

    class Capture(T.SplatTrainer):
        def _apply_updates(self, splats, v_t, v_sh, v_o, v_r, visible, max_radius, median_scale):
            captured.update(v_t=v_t.clone(), v_sh=v_sh.clone(), v_o=v_o.clone(), v_r=v_r.clone(), vis=visible.clone(),
                            rad=max_radius.clone())
            return 0.0

    multi = fresh()
    T.SplatTrainer(cfg, rt.ctx, bounds).step_views(batches, multi)
    per_view = []
    for b in batches:
        Capture(cfg, rt.ctx, bounds).step(b, fresh())
        per_view.append(dict(captured))
    avg = {x: ((per_view[0][x].double() + per_view[1][x].double()) / 2.0).float() for x in ("v_t", "v_sh", "v_o")}
    vis = per_view[0]["vis"] + per_view[1]["vis"]
    refs = []
    for c in (cfg, cfg0):
        ref = fresh()
        tr_ = T.SplatTrainer(c, rt.ctx, bounds)
        tr_._ensure_state(ref)
        tr_.step_count = 1
        tr_._apply_updates(ref, avg["v_t"], avg["v_sh"], avg["v_o"], torch.maximum(per_view[0]["v_r"], per_view[1]["v_r"]), vis,
                           torch.maximum(per_view[0]["rad"], per_view[1]["rad"]), bounds.median_size())
        refs.append(ref)
    torch.cuda.synchronize()
    noisy, quiet = refs
    lr_mean = float(np.float32(cfg.lr_mean * bounds.median_size()))
    ns, med = np.float32(lr_mean * cfg.mean_noise_weight), np.float32(bounds.median_size())
    z = _step_noise(rt, n, 1, cfg.seed)
    raw, ls, visn = quiet.raw_opacities.cpu().numpy(), quiet.transforms[:, 7:10].cpu().numpy(), vis.cpu().numpy()
    wgt = U.noise_weight64(raw, ls, visn, floor.cpu().numpy())
    inc = np.clip(z * wgt[:, None] * float(ns), -float(med), float(med))
    base = quiet.transforms[:, :3].double().cpu().numpy()
    # the dense route: bg_train_update with the floor, exactly the restatement's increment up to the noise bound
    d_ref = noisy.transforms[:, :3].double().cpu().numpy() - base
    rel = U.noise_rel_tol(raw, ls, floor.cpu().numpy())
    assert (np.abs(d_ref - inc) <= rel[:, None] * np.abs(inc) + 2 * np.spacing(np.abs(base).astype(np.float32))).all()
    # the factored route, row by row on the thin, visible, mid-opacity splats (Adam's step-1 move is +-lr_mean per
    # element; a gradient whose sign flips with the summation order moves it by 2 lr_mean)
    thin = np.zeros(n, bool)
    thin[np.arange(0, n, 8)] = True
    sel = thin & (visn > 0) & (np.abs(inc).max(1) > 20 * lr_mean)
    assert sel.sum() > 200, int(sel.sum())
    d_multi = multi.transforms[:, :3].double().cpu().numpy() - base
    ok = (np.abs(d_multi - inc) <= 0.1 * np.abs(inc) + 2.5 * lr_mean).all(1)
    assert ok[sel].mean() > 0.95, float(ok[sel].mean())


def test_refine_stats_noise_grid_stride(rt):
    """bg_refine_stats_noise at N = 600 001 (more rows than the grid's 2112 x 256 threads): statistics bit for bit; the
    noise, from a caller-supplied z with the reference's weight (1 - sigmoid(raw))^150 * visible, within the bound."""
    n = 600_001
    rng = np.random.default_rng(600)
    tr = U.random_state(n, 1, rng)["transforms"]
    raw = rng.uniform(-9, 1, n).astype(np.float32)
    vr, vis, rad = (rng.uniform(0, 1, n).astype(np.float32), rng.integers(0, 3, n).astype(np.float32),
                    rng.uniform(0, 1, n).astype(np.float32))
    old = [rng.uniform(0, 1, n).astype(np.float32) for _ in range(3)]
    z = rng.normal(size=(n, 3)).astype(np.float32)
    ns, med = np.float32(0.05), np.float32(0.01)
    D = _dev(rt, dict(tr=tr, raw=raw, vr=vr, vis=vis, rad=rad, o0=old[0], o1=old[1], o2=old[2], z=z))
    rt._lib.check(rt.lib.bg_refine_stats_noise(rt.ctx.handle, _stream(), n, D["vr"].data_ptr(), D["vis"].data_ptr(),
                                               D["rad"].data_ptr(), D["o0"].data_ptr(), D["o1"].data_ptr(), D["o2"].data_ptr(),
                                               D["tr"].data_ptr(), D["raw"].data_ptr(), D["z"].data_ptr(), ns, med),
                  "bg_refine_stats_noise")
    got = _host(D)
    _bitwise(got, dict(o0=np.fmax(vr, old[0]), o1=old[1] + vis, o2=np.fmax(rad, old[2])), ["o0", "o1", "o2"], "stats")
    _bitwise({"t": got["tr"][:, 3:]}, {"t": tr[:, 3:]}, ["t"], "untouched")
    w = np.clip((1.0 - 1.0 / (1.0 + np.exp(-raw.astype(np.float64)))) ** 150, 0, 1) * vis
    inc = np.clip(z * (w * float(ns))[:, None], -float(med), float(med))
    want = tr[:, :3].astype(np.float64) + inc
    tol = 2 * np.spacing(np.abs(want).astype(np.float32)) + U.noise_rel_tol(raw, None)[:, None] * np.abs(inc) + 2.0 ** -140
    assert (np.abs(got["tr"][:, :3] - want) <= tol).all()
    assert (np.abs(inc) == float(med)).sum() > 1000 and (got["tr"][vis == 0, :3] == tr[vis == 0, :3]).all()


@pytest.mark.parametrize("rows,cols,reduce_v", [(100_003, 10, False), (20_001, 75, True), (2_000, 201, True)])
def test_adam_step_large(rt, rows, cols, reduce_v):
    """bg_adam_step for t = 1..6 against the oracle at test_adam_vs_oracle's tolerance: the grid-stride loop (10^6
    elements), the row-reduce kernel's scalar tail (75 columns, 33-row last tile) and its opt-in shared memory (201
    columns: 64 x 201 x 4 B > 48 KB)."""
    rng = np.random.default_rng(rows + cols)
    p = rng.normal(0, 1, (rows, cols)).astype(np.float32)
    m = np.zeros_like(p)
    v = np.zeros(rows if reduce_v else (rows, cols), np.float32)
    scale = rng.uniform(0.1, 1.0, cols).astype(np.float32)
    D = _dev(rt, dict(p=p, m=m, v=v, s=scale))
    for t in range(1, 7):
        g = rng.normal(0, 1e-3, (rows, cols)).astype(np.float32)
        rt.orc.adam_step(p, g, m, v, 2e-3, t, lr_scale_per_col=scale, reduce_v=reduce_v)
        tg = torch.from_numpy(g).to(rt.dev)
        rt._lib.check(rt.lib.bg_adam_step(rt.ctx.handle, _stream(), D["p"].data_ptr(), tg.data_ptr(), D["m"].data_ptr(),
                                          D["v"].data_ptr(), rows, cols, D["s"].data_ptr(), 2e-3, 0.9, 0.999, 1e-15, t,
                                          int(reduce_v)), "bg_adam_step")
        got = _host(D)
        np.testing.assert_allclose(got["p"], p, rtol=3e-6, atol=1e-7)
        np.testing.assert_allclose(got["m"], m, rtol=2e-4, atol=1e-9)
        np.testing.assert_allclose(got["v"], v, rtol=2e-4, atol=1e-13)


def test_train_update_argument_checks(rt):
    """Null -> BG_ERR_NULL; bad K or step -> BG_ERR_INVALID; n == 0 -> BG_OK; an array the pass reads as float2
    (transforms, m_t, v_t, v_transforms) off by 4 bytes, or as float4 (sh, m_sh, v_sh_grad) off by 8, is BG_ERR_INVALID
    with every buffer untouched.  The single- and multi-view steps share the checks of their state arrays."""
    L = rt._lib
    n, k = 64, 4
    rng = np.random.default_rng(1)
    st, gr = U.random_state(n, k, rng), U.random_grads(n, k, rng)
    # one spare row in front of every array, so that a pointer can be moved off its alignment inside the buffer
    pad = lambda x: np.concatenate([np.zeros((1,) + x.shape[1:], x.dtype), x])
    dst, dgr = _dev(rt, {x: pad(v) for x, v in st.items()}), _dev(rt, {x: pad(v) for x, v in gr.items()})
    row = lambda t: t.data_ptr() + t[0].numel() * 4
    h = rt.ctx.handle
    call = lambda a: rt.lib.bg_train_update(h, _stream(), C.byref(a))

    def args(**shift):
        a = _args(rt, dst, dgr, 2, ptr=row)
        a.n = n
        for key, by in shift.items():
            setattr(a, key, getattr(a, key) + by)
        return a
    before = _host({**dst, **dgr})
    assert rt.lib.bg_train_update(None, None, C.byref(args())) == L.BG_ERR_NULL
    assert rt.lib.bg_train_update(h, None, None) == L.BG_ERR_NULL
    a = args(); a.m_sh = None
    assert call(a) == L.BG_ERR_NULL
    a = args(); a.k = 5
    assert call(a) == L.BG_ERR_INVALID
    a = args(); a.step = 0
    assert call(a) == L.BG_ERR_INVALID
    for key in ("transforms", "m_t", "v_t", "v_transforms"):
        assert call(args(**{key: 4})) == L.BG_ERR_INVALID, key
    for key in ("sh", "m_sh", "v_sh_grad"):
        assert call(args(**{key: 8})) == L.BG_ERR_INVALID, key
    _bitwise(_host({**dst, **dgr}), before, list(before), "rejected calls write nothing")
    a = args(); a.n = 0
    assert call(a) == L.BG_OK
    assert call(args()) == L.BG_OK
    # the steps: BgTrainStepArgs / BgTrainViewsArgs with a misaligned state array never reach the device
    ws = torch.empty(1 << 16, dtype=torch.uint8, device=rt.dev)
    for cls, fn in ((L.BgTrainStepArgs, "bg_train_step"), (L.BgTrainViewsArgs, "bg_train_step_views")):
        for key, by in (("transforms", 4), ("m_t", 4), ("v_t", 4), ("sh", 8), ("m_sh", 8)):
            s = cls()
            for x in ("transforms", "sh", "raw_opac", "m_t", "v_t", "m_sh", "v_sh", "m_o", "v_o", "refine_norm", "vis_weight",
                      "max_screen"):
                setattr(s, x, row(dst[x]))
            setattr(s, key, getattr(s, key) + by)
            s.n, s.k, s.w, s.h, s.channels, s.step = n, k, 16, 16, 3, 1
            s.loss_out = s.workspace = ws.data_ptr()
            if fn == "bg_train_step":
                s.gt_packed = ws.data_ptr()
                r = rt.lib.bg_train_step(h, _stream(), C.byref(s))
            else:
                cams = (L.BgCamera * 1)()
                gts = (C.c_void_p * 1)(ws.data_ptr())
                s.cams, s.gt_packed, s.local_views = cams, gts, 1
                r = rt.lib.bg_train_step_views(h, None, _stream(), C.byref(s))
            assert r == L.BG_ERR_INVALID, (fn, key)
    assert "aligned" in L.load().bg_last_error_string().decode()
