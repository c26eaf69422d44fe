"""Op-for-op float32 restatement of the fused parameter-update pass (csrc/update.cu, bg_train_update), in numpy.

update.cu is compiled with -fmad=false and uses only IEEE + - * /, correctly rounded sqrt and reciprocal, in the order
written there, so everything but the mean noise is a pure f32 function of the inputs.  Each numpy statement below is one
f32 operation of the kernel (numpy rounds every float32 array operation and never fuses a multiply-add), so
`update_f32` must reproduce the device bit for bit.  The noise weight (expf / powf on the device, neither correctly
rounded) is formed in float64 from the f32 updated values; see `noise_rel_tol` for the bound.

`adam64` is AdamScaled (adam_scaled.rs:75-165) in float64 with the reference's operation order
(m/bc1)/(sqrt(v/bc2)+eps)*lr, the semantic check of both."""
import numpy as np

F = np.float32
EPS32 = 2.0 ** -24          # unit roundoff of f32
BETA1, BETA2, EPS = F(0.9), F(0.999), F(1e-15)


def powi_f32(a, b: int):
    """compiler-rt __powisf2 (what Rust's f32::powi lowers to), as the host forms the bias corrections."""
    a, r, recip = F(a), F(1.0), b < 0
    while True:
        if b & 1:
            r = F(r * a)
        b = int(b / 2)
        if b == 0:
            break
        a = F(a * a)
    return F(F(1.0) / r) if recip else r


class Consts:
    """The host-side constants of one step (api.cu update_params), each rounded to f32 where the host rounds it."""

    def __init__(self, step, lr_mean, lr_rotation, lr_scale, lr_coeffs_dc, lr_coeffs_sh_scale, lr_opac,
                 noise_scale=0.0, median_scale=0.0):
        self.step = int(step)
        self.first = step == 1
        self.f1, self.f2 = F(F(1.0) - BETA1), F(F(1.0) - BETA2)
        self.inv_bc1 = F(F(1.0) / F(F(1.0) - powi_f32(BETA1, step)))
        self.inv_bc2 = F(F(1.0) / F(F(1.0) - powi_f32(BETA2, step)))
        self.lr_t = np.array([lr_mean] * 3 + [lr_rotation] * 4 + [lr_scale] * 3, np.float32)
        self.lr_dc = F(F(1.0) * F(lr_coeffs_dc))
        self.lr_rest = F(F(F(1.0) / F(lr_coeffs_sh_scale)) * F(lr_coeffs_dc))
        self.lr_opac = F(lr_opac)
        self.noise_scale, self.median_scale = F(noise_scale), F(median_scale)


def adam_m(m, g, c):
    return g * c.f1 if c.first else m * BETA1 + g * c.f1


def adam_v(v, gsq, c):
    return gsq * c.f2 if c.first else v * BETA2 + gsq * c.f2


def inv_denom(v, c):
    return F(1.0) / (np.sqrt(v * c.inv_bc2) + EPS)


def adam_p(p, m, inv, lr, c):
    return p - ((m * c.inv_bc1) * inv) * lr


def row_mean_sq(g):
    """Mean of g^2 over the 3K floats of each row, summed sequentially in column order (not numpy's pairwise sum)."""
    s = np.zeros(g.shape[0], np.float32)
    for col in range(g.shape[1]):
        s = s + g[:, col] * g[:, col]
    return s / F(g.shape[1])


def fold_opacity64(raw, log_scales, f):
    """Splats::opacities with the floor folded in (gaussian_splats.rs:215-223), float64:
    clamp(sigmoid(raw) * sqrt(prod s^2 / prod (s^2 + f^2)), 1e-6, 1 - 1e-6)."""
    s2 = np.exp(2.0 * log_scales.astype(np.float64))
    f2 = f.astype(np.float64)[:, None] ** 2
    coef = np.sqrt(np.prod(s2, 1) / np.prod(s2 + f2, 1))
    sig = 1.0 / (1.0 + np.exp(-raw.astype(np.float64)))
    return np.clip(sig * coef, 1e-6, 1.0 - 1e-6)


def noise_weight64(raw, log_scales, visible, min_scale=None):
    """(1 - opacity)^150 where visible > 0, else 0; opacity from the UPDATED raw opacity (and log-scales, with a floor)."""
    with np.errstate(over="ignore"):
        o = (1.0 / (1.0 + np.exp(-raw.astype(np.float64)))) if min_scale is None else fold_opacity64(raw, log_scales, min_scale)
    return np.clip((1.0 - o) ** 150, 0.0, 1.0) * (visible > 0)


def noise_rel_tol(raw, log_scales, min_scale=None):
    """Relative bound on the device's noise increment against noise_weight64 * z * noise_scale, per row.

    The device forms the opacity o in f32 with expf (<= 2 ulp), one add and an IEEE division: |do| <= 8 u o with
    u = 2^-24.  With a floor, coef = sqrtf(prod s^2 / prod s^2f) adds three expf, eight roundings and a sqrt:
    |do| <= 24 u o.  1 - o is rounded once more, so its relative error is <= c u o / (1 - o) + u, which powf(., 150)
    multiplies by 150; powf itself adds <= 2 ulp, the products with noise_scale and z one rounding each.  Hence
    |d inc| / |inc| <= 150 (c u o / (1 - o) + u) + 8 u, about 8e-5 for o <= 0.5 without a floor (c = 8)."""
    c = 8.0 if min_scale is None else 24.0
    with np.errstate(over="ignore"):
        o = (1.0 / (1.0 + np.exp(-raw.astype(np.float64)))) if min_scale is None else fold_opacity64(raw, log_scales, min_scale)
    return 150.0 * (c * EPS32 * o / (1.0 - o) + EPS32) + 8.0 * EPS32


def update_f32(st, gr, c, z=None, min_scale=None):
    """One bg_train_update on host copies.  st: dict of float32 arrays transforms [n,10], sh [n,K,3], raw_opac [n],
    m_t, v_t [n,10], m_sh [n,K,3], v_sh [n], m_o, v_o [n], refine_norm, vis_weight, max_screen [n]; gr: v_transforms,
    v_sh_grad, v_raw_opac, v_refine, visible, max_radius.  Returns the new state and, when noisy, a dict with the
    noise-free means `mean_adam`, the float64 increment `inc` and the rows it applies to `noised`."""
    n = st["transforms"].shape[0]
    o = {}
    # transforms: Adam with per-column learning rates
    g = gr["v_transforms"]
    m = adam_m(st["m_t"], g, c)
    v = adam_v(st["v_t"], g * g, c)
    o["m_t"], o["v_t"] = m, v
    p = adam_p(st["transforms"], m, inv_denom(v, c), c.lr_t[None, :], c)
    # raw opacity
    g = gr["v_raw_opac"]
    mo = adam_m(st["m_o"], g, c)
    vo = adam_v(st["v_o"], g * g, c)
    raw = adam_p(st["raw_opac"], mo, inv_denom(vo, c), c.lr_opac, c)
    o["m_o"], o["v_o"], o["raw_opac"] = mo, vo, raw
    # refine statistics
    o["refine_norm"] = np.fmax(gr["v_refine"], st["refine_norm"])
    o["vis_weight"] = st["vis_weight"] + gr["visible"]
    o["max_screen"] = np.fmax(gr["max_radius"], st["max_screen"])
    # SH: one second moment per row (row mean of g^2), one reciprocal per row, lr_dc on the first three columns
    k3 = st["sh"].shape[1] * 3
    gs = gr["v_sh_grad"].reshape(n, k3)
    vs = adam_v(st["v_sh"], row_mean_sq(gs), c)
    inv = inv_denom(vs, c)
    ms = adam_m(st["m_sh"].reshape(n, k3), gs, c)
    lr = np.full(k3, c.lr_rest, np.float32)
    lr[:3] = c.lr_dc
    o["sh"] = adam_p(st["sh"].reshape(n, k3), ms, inv[:, None], lr[None, :], c).reshape(st["sh"].shape)
    o["m_sh"], o["v_sh"] = ms.reshape(st["sh"].shape), vs
    info = None
    if c.noise_scale != 0.0:
        w = noise_weight64(raw, p[:, 7:10], gr["visible"], min_scale)
        wm = w * np.float64(c.noise_scale)
        unclamped = z.astype(np.float64) * wm[:, None]
        inc = np.clip(unclamped, -np.float64(c.median_scale), np.float64(c.median_scale))
        noised = (wm != 0.0)
        info = dict(mean_adam=p[:, :3].copy(), inc=inc, unclamped=unclamped, noised=noised,
                    rel_tol=noise_rel_tol(raw, p[:, 7:10], min_scale))
        p = p.copy()
        p[:, :3] = np.where(noised[:, None], (p[:, :3].astype(np.float64) + inc).astype(np.float32), p[:, :3])
    o["transforms"] = p
    return o, info


def adam64(p, g, m, v, lr, step, reduce_v=False):
    """AdamScaled::step in float64 with the reference's order: p -= (m/bc1) / (sqrt(v/bc2) + eps) * lr.  The betas are
    the f32 constants the kernel uses (0.9f, 0.999f), widened.  In place on the float64 arrays p, m, v (v: [rows] when
    reduce_v).  Returns the denominator sqrt(v/bc2) + eps and the bias corrections bc1, bc2 of this step (adam64_tol)."""
    b1, b2, eps = float(BETA1), float(BETA2), float(EPS)
    g = g.astype(np.float64)
    first = step == 1
    m[...] = (1 - b1) * g if first else b1 * m + (1 - b1) * g
    gsq = (g * g).mean(1) if reduce_v else g * g
    v[...] = (1 - b2) * gsq if first else b2 * v + (1 - b2) * gsq
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    vv = v[:, None] if reduce_v else v
    den = np.sqrt(vv / bc2) + eps
    p -= (m / bc1) / den * lr
    return den, bc1, bc2


def adam64_tol(abs_m, den, bc1, bc2, lr, step, cols, c):
    """Bound on |p_f32 - p_f64| accumulated up to `step` (one call per step, summed by the caller), per element.

    abs_m: the first moment accumulated from |g| in float64 (the scale of m's rounding error: each step rounds two
    products and a sum, so |dm| <= 3 s u |m|_abs after s steps); v is a sum of squares (no cancellation): |dv| <= 3 s u v,
    plus cols u for the sequential row mean.  The host's 1/bc in f32 differs from the float64 one by the relative amount
    rb = |inv_bc_f32 bc_64 - 1|, measured here (for beta2 it is up to ~500 u: 1 - 0.999^t cancels).  sqrt halves the
    relative error of v, and sqrt, the eps add, the reciprocal and the three products round once each.  The update
    lands on p with one more rounding (1 ulp of p after the step).  Denormal moments lose absolute precision 2^-149 per
    operation; their contribution is bounded by 6 s 2^-149 / bc1 / den * lr."""
    rb1 = abs(float(c.inv_bc1) * bc1 - 1.0)
    rb2 = abs(float(c.inv_bc2) * bc2 - 1.0)
    rel = rb1 + 0.5 * rb2 + (3 * step + 0.5 * (3 * step + cols) + 8) * EPS32
    a = (abs_m / bc1) / den * lr
    return rel * a + 6 * step * 2.0 ** -149 / bc1 / den * lr


class Adam64:
    """Tracks transforms, sh and raw_opac through AdamScaled in float64 alongside update_f32 or the device, with the
    accumulated bound of adam64_tol plus one ulp of the f32 parameter per step."""
    GKEY = dict(transforms="v_transforms", sh="v_sh_grad", raw_opac="v_raw_opac")

    def __init__(self, st, consts):
        n = st["transforms"].shape[0]
        self.n, self.k3 = n, st["sh"].shape[1] * 3
        self.p = {x: st[x].reshape(n, -1).astype(np.float64) for x in self.GKEY}
        self.m = {x: np.zeros_like(self.p[x]) for x in self.p}
        self.a = {x: np.zeros_like(self.p[x]) for x in self.p}
        self.v = dict(transforms=np.zeros((n, 10)), sh=np.zeros(n), raw_opac=np.zeros((n, 1)))
        self.tol = {x: np.zeros_like(self.p[x]) for x in self.p}
        c = consts
        self.lr = dict(transforms=c.lr_t.astype(np.float64), raw_opac=np.float64(c.lr_opac),
                       sh=np.array([c.lr_dc] * 3 + [c.lr_rest] * (self.k3 - 3), np.float64))

    def step_and_check(self, gr, c, st):
        """One step of the float64 reference; asserts that the f32 state st is within the bound."""
        b1 = float(BETA1)
        for x in self.p:
            g = gr[self.GKEY[x]].reshape(self.n, -1)
            ag = np.abs(g.astype(np.float64))
            self.a[x] = (1 - b1) * ag if c.first else b1 * self.a[x] + (1 - b1) * ag
            den, bc1, bc2 = adam64(self.p[x], g, self.m[x], self.v[x], self.lr[x], c.step, reduce_v=x == "sh")
            self.tol[x] += adam64_tol(self.a[x], den, bc1, bc2, self.lr[x], c.step, self.k3 if x == "sh" else 0, c)
            got = st[x].reshape(self.n, -1)
            self.tol[x] += np.spacing(np.abs(got)).astype(np.float64)
            err = np.abs(got.astype(np.float64) - self.p[x])
            assert (err <= self.tol[x]).all(), (c.step, x, float((err / np.maximum(self.tol[x], 1e-300)).max()))


def random_state(n, k, rng):
    """A trainable state with log-scales, opacities and non-zero refine statistics of a real run's spread."""
    tr = np.concatenate([rng.uniform(-2, 2, (n, 3)), rng.normal(size=(n, 4)), np.log(rng.uniform(0.002, 0.2, (n, 3)))], 1)
    z = lambda *s: np.zeros(s, np.float32)
    return dict(transforms=tr.astype(np.float32), sh=(rng.normal(size=(n, k, 3)) * 0.3).astype(np.float32),
                raw_opac=rng.uniform(-6, 4, n).astype(np.float32), m_t=z(n, 10), v_t=z(n, 10), m_sh=z(n, k, 3), v_sh=z(n),
                m_o=z(n), v_o=z(n), refine_norm=rng.uniform(0, 1e-3, n).astype(np.float32),
                vis_weight=rng.integers(0, 4, n).astype(np.float32), max_screen=rng.uniform(0, 0.3, n).astype(np.float32))


def random_grads(n, k, rng):
    """Gradients of both signs spanning 1e-30 .. 1e2, exact-zero transform rows, all-zero SH rows, denormals."""
    def mag(*shape):
        return (np.sign(rng.normal(size=shape)) * 10.0 ** rng.uniform(-30, 2, shape)).astype(np.float32)
    g = dict(v_transforms=mag(n, 10), v_sh_grad=mag(n, k, 3), v_raw_opac=mag(n),
             v_refine=rng.uniform(0, 2e-3, n).astype(np.float32), visible=rng.integers(0, 3, n).astype(np.float32),
             max_radius=rng.uniform(0, 0.5, n).astype(np.float32))
    g["v_transforms"][rng.random(n) < 0.1] = 0.0
    g["v_sh_grad"][rng.random(n) < 0.1] = 0.0
    g["v_raw_opac"][rng.random(n) < 0.1] = 0.0
    den = rng.random((n, 10)) < 0.05
    g["v_transforms"][den] = (np.sign(rng.normal(size=int(den.sum()))) * rng.uniform(1e-45, 1e-38, int(den.sum()))).astype(np.float32)
    g["v_sh_grad"].reshape(n, -1)[rng.random((n, 3 * k)) < 0.05] = np.float32(-3e-42)
    return g
