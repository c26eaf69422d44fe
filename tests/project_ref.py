"""Float64 restatement of the per-splat projection and its backward (TEST INFRASTRUCTURE ONLY).

Restated from the reference's semantics, not from the CUDA or oracle source:
  forward   project_forward.rs (cull), project_visible.rs (row), helpers.rs (world_to_cam, calc_cov2d,
            compensate_cov2d, compute_bbox_extent), camera_model/*.rs (projection and Jacobian), sh.rs (colour)
  backward  project_backwards.rs, by torch autograd through the forward, with the reference's departures from
            its own forward's derivative written out where they occur (see `_forward` below)

The f32 inputs are widened exactly; every operation is float64 on the CPU.  Each camera Jacobian is the derivative
of that model's projection (torch.func.jacfwd), evaluated where the reference evaluates it:
  pinhole  at the clamp surrogate point (clamp(x/z) z, clamp(y/z) z, z): column 3 is -f clamp(x/z) / z (pinhole.rs)
  RT8      at the same surrogate point (radial_tangential_8.rs:66-142)
  KB4/TPF  at the mean itself; the projection switches to the pinhole form for r < 1e-6 (kannala_brandt_4.rs:48),
           so the Jacobian there is the pinhole one.
The SH basis is the real spherical harmonics basis with its normalisations computed in float64 from their closed
forms, in the reference's order and signs (sh.rs), so a wrong f32 constant on either side shows.

Bounds.  `bounds` carries, per projected element, a magnitude companion M (the same formulas on absolute values):
  xy      |f x / z| + |c|  (the terms summed)
  conic   lambda_max(conic)^2 (G + blur), G = max entry of |V| |V|^T with |V| = |J| |R_view| |R_q| diag(s): the f32
          error of cov2d propagated through the inverse (this is the condition factor of the issue)
  opacity opacity; with Mip also the error of comp = sqrt(max(det_raw, 0) / det_blur): the cancellation of det_raw
          is bounded by (|a c| + b^2 + G (|a| + |c| + 2|b|)) and propagated through the sqrt (or sqrt of it, whichever
          is smaller, for det_raw near 0)
  colour  sum_k |c_k| |Y_k| + 0.5
and an element passes when |f32 - ref| <= C_col 2^-24 M.  C_col was calibrated once against the oracle's rows on the
CPU suite (every camera model, Mip on and off, K in {1, 4, 9, 16, 25}, synthetic and edge scenes): the largest
measured ratios |orc - ref| / (2^-24 M) were xy 1.5, conic 9.1, opacity 4.4, colour 1.4 (the colour companion is
scaled by sqrt(K)); C is twice that, rounded up: 3, 20, 9, 3.

Ambiguity.  `flags` marks every splat whose cull or branch decision lies within its f32 error of the threshold:
z = 0.01, theta = half fov, |q|^2 = 1e-6, opacity = 1/255, det = 0, the four screen edges, the four Jacobian clamp
limits, r = 1e-6 and the 1e18 rescale.  Tests exclude flagged splats; there is no flip budget.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np
import torch

F64 = torch.float64
U = 2.0 ** -24
PINHOLE, KB4, RT8, TPF = 0, 1, 2, 3
# calibrated bound constants (see the module docstring)
C_XY, C_CONIC, C_OPAC, C_COLOR = 3.0, 20.0, 9.0, 3.0


# ---- SH basis (sh.rs), normalisations from their closed forms
def _sh_consts():
    pi = math.pi
    s = math.sqrt
    return dict(
        c0=0.5 * s(1 / pi), c1=s(3 / (4 * pi)),
        c2a=0.5 * s(15 / pi), c2b=0.25 * s(5 / pi), c2c=0.25 * s(15 / pi),
        c3a=0.25 * s(35 / (2 * pi)), c3b=0.5 * s(105 / pi), c3c=0.25 * s(21 / (2 * pi)), c3d=0.25 * s(7 / pi),
        c3e=0.25 * s(105 / pi),
        c4a=0.75 * s(35 / pi), c4b=0.75 * s(35 / (2 * pi)), c4c=0.75 * s(5 / pi), c4d=0.75 * s(5 / (2 * pi)),
        c4e=(3 / 16) * s(1 / pi), c4f=0.375 * s(5 / pi), c4g=(3 / 16) * s(35 / pi),
    )


_C = _sh_consts()


def sh_basis(d: torch.Tensor, k: int, terms: bool = False) -> torch.Tensor:
    """Y [n, k] of unit directions d [n, 3], in the reference's coefficient order and signs.  terms=True gives each
    function's magnitude companion instead: the sum of the absolute values of its monomial terms."""
    x, y, z = (d.abs() if terms else d).unbind(-1)
    c = _C
    sg = 1.0 if terms else -1.0                # the sign of every subtracted term and negative constant
    ys = [torch.full_like(x, c["c0"])]
    if k > 1:
        ys += [sg * c["c1"] * y, c["c1"] * z, sg * c["c1"] * x]
    if k > 4:
        ys += [c["c2a"] * x * y, sg * c["c2a"] * y * z, c["c2b"] * (3 * z * z + sg * 1), sg * c["c2a"] * x * z,
               c["c2c"] * (x * x + sg * y * y)]
    if k > 9:
        ys += [sg * c["c3a"] * y * (3 * x * x + sg * y * y), c["c3b"] * x * y * z, sg * c["c3c"] * y * (5 * z * z + sg),
               c["c3d"] * z * (5 * z * z + sg * 3), sg * c["c3c"] * x * (5 * z * z + sg), c["c3e"] * z * (x * x + sg * y * y),
               sg * c["c3a"] * x * (x * x + sg * 3 * y * y)]
    if k > 16:
        z2 = z * z
        ys += [c["c4a"] * x * y * (x * x + sg * y * y), sg * c["c4b"] * y * z * (3 * x * x + sg * y * y),
               c["c4c"] * x * y * (7 * z2 + sg), sg * c["c4d"] * y * z * (7 * z2 + sg * 3),
               c["c4e"] * (35 * z2 * z2 + sg * 30 * z2 + 3), sg * c["c4d"] * x * z * (7 * z2 + sg * 3),
               c["c4f"] * (x * x + sg * y * y) * (7 * z2 + sg), sg * c["c4b"] * x * z * (x * x + sg * 3 * y * y),
               c["c4g"] * (x ** 4 + sg * 6 * x * x * y * y + y ** 4)]
    assert len(ys) == k, "K must be 1, 4, 9, 16 or 25"
    return torch.stack(ys, -1)


# ---- camera models (camera_model/*.rs): project one point p [3] -> [2]
def _project_fn(u):
    fx, fy, cx, cy = u.fx, u.fy, u.cx, u.cy
    k = [float(v) for v in u.model_params]
    model = u.camera_model

    def pinhole(p):
        return torch.stack([fx * p[0] / p[2] + cx, fy * p[1] / p[2] + cy])

    def kb4(p):
        x, y, z = p[0], p[1], p[2]
        r2 = x * x + y * y
        near = r2 < 1e-12                          # r < 1e-6; sqrt is never taken at 0, so no NaN reaches autograd
        rs = torch.sqrt(torch.where(near, torch.ones_like(r2), r2))
        th = torch.atan2(rs, z)
        t2 = th * th
        d = th * (1 + k[0] * t2 + k[1] * t2 ** 2 + k[2] * t2 ** 3 + k[3] * t2 ** 4)
        fish = torch.stack([fx * d * x / rs + cx, fy * d * y / rs + cy])
        return torch.where(near, pinhole(p), fish)

    def rt8(p):
        xn, yn = p[0] / p[2], p[1] / p[2]
        r2 = xn * xn + yn * yn
        rad = (1 + k[0] * r2 + k[1] * r2 ** 2 + k[2] * r2 ** 3) / (1 + k[3] * r2 + k[4] * r2 ** 2 + k[5] * r2 ** 3)
        p1, p2 = k[6], k[7]
        xd = xn * rad + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn * xn)
        yd = yn * rad + p1 * (r2 + 2 * yn * yn) + 2 * p2 * xn * yn
        return torch.stack([fx * xd + cx, fy * yd + cy])

    def tpf(p):
        xn, yn = p[0] / p[2], p[1] / p[2]
        p1, p2, sx1, sy1 = k[4], k[5], k[6], k[7]
        r2 = xn * xn + yn * yn
        du = 2 * p1 * xn * yn + p2 * (3 * xn * xn + yn * yn) + sx1 * r2
        dv = 2 * p2 * xn * yn + p1 * (xn * xn + 3 * yn * yn) + sy1 * r2
        return kb4(p) + torch.stack([fx * du, fy * dv])

    return {PINHOLE: pinhole, KB4: kb4, RT8: rt8, TPF: tpf}[model]


def _clamp_point(u, mc):
    """The Jacobian clamp surrogate (pinhole.rs, radial_tangential_8.rs): (clamp(x/z) z, clamp(y/z) z, z)."""
    x, y, z = mc.unbind(-1)
    xc = torch.clamp(x / z, u.lim_neg_x, u.lim_pos_x) * z
    yc = torch.clamp(y / z, u.lim_neg_y, u.lim_pos_y) * z
    return torch.stack([xc, yc, z], -1)


def _quat_to_mat(q):
    w, x, y, z = q.unbind(-1)
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
        torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
        torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def _view(u):
    vm = torch.tensor(np.asarray(u.viewmat, np.float32).astype(np.float64), dtype=F64)
    return vm[:9].reshape(3, 3).T.contiguous(), vm[9:12].clone()   # column-major 3x3, translation


def _sym2(m):
    return m[..., 0, 0], m[..., 0, 1], m[..., 1, 1]


def _forward(u, w, h, tr, sh, raw, mip, grad):
    """Everything per splat, float64.  With grad=True the returned tensors carry the reference's backward (see the
    stop-gradients and surrogates below); values do not depend on `grad`."""
    n, k = sh.shape[0], sh.shape[1]
    Rv, tv = _view(u)
    mean, qu, ls = tr[:, 0:3], tr[:, 3:7], tr[:, 7:10]
    mc = mean @ Rv.T + tv                                                 # helpers.rs world_to_cam
    scale = torch.exp(ls)
    qn = (qu * qu).sum(-1)
    q = qu / torch.sqrt(torch.where(qn > 0, qn, torch.ones_like(qn)))[:, None]
    Rq = _quat_to_mat(q)
    M = Rq * scale[:, None, :]
    sig_c = Rv @ (M @ M.transpose(-1, -2)) @ Rv.T                          # camera-space covariance
    proj = _project_fn(u)
    model = u.camera_model
    jac = torch.func.vmap(torch.func.jacfwd(proj))
    # keep the points of culled splats finite so that no NaN leaks into autograd
    z_ok = mc[:, 2].abs() > 1e-30
    mcs = torch.where(z_ok[:, None], mc, torch.tensor([0.0, 0.0, 1.0], dtype=F64))
    mean2d = torch.func.vmap(proj)(mcs)
    if model in (PINHOLE, RT8):
        g = _clamp_point(u, mcs)
        J = jac(g)
        if model == RT8 and grad:
            # radial_tangential_8.rs:144-377: the reference's VJP treats the projection as proj(g(mean)) -- the
            # clamped components of the mean gradient go to z -- and forms vJ with J_eff = J(g) dg/dmean.  So the
            # mean2d gradient is that of proj(g(mean)), and cov2d's gradient to the mean is that of J_eff Σ J_eff^T
            # (with Σ held), while its gradient to Σ uses the forward Jacobian J(g).
            S = _dg_dmean(u, mcs).detach()
            Je = J @ S
            m2g = torch.func.vmap(proj)(g)
            mean2d = mean2d.detach() + m2g - m2g.detach()
            cov_mean = Je @ sig_c.detach() @ Je.transpose(-1, -2)
            cov_shape = J.detach() @ sig_c @ J.detach().transpose(-1, -2)
            cov_raw = (J @ sig_c @ J.transpose(-1, -2)).detach() + (cov_mean - cov_mean.detach()) + \
                (cov_shape - cov_shape.detach())
        else:
            cov_raw = J @ sig_c @ J.transpose(-1, -2)
    else:
        J = jac(mcs)
        cov_raw = J @ sig_c @ J.transpose(-1, -2)
    a, b, c = _sym2(cov_raw)
    max_abs = torch.maximum(torch.maximum(a.abs(), c.abs()), b.abs())
    # helpers.rs calc_cov2d: the 1e18 rescale factor is a constant to the backward
    resc = torch.where(max_abs > 1e18, 1e18 / max_abs, torch.ones_like(max_abs)).detach()
    a, b, c = a * resc, b * resc, c * resc
    blur = 0.1 if mip else 0.3
    ab, cb = a + blur, c + blur
    det_b = ab * cb - b * b
    det_raw = a * c - b * b
    if mip:
        # project_backwards.rs:181-183: comp only scales v_raw_opac; no gradient reaches the geometry
        comp = torch.sqrt(torch.clamp(det_raw, min=0.0) / torch.where(det_b > 0, det_b, torch.ones_like(det_b))).detach()
    else:
        comp = torch.ones_like(a)
    sig = torch.sigmoid(raw)
    opac = sig * comp
    det_ok = det_b > 0
    db = torch.where(det_ok, det_b, torch.ones_like(det_b))
    ca, cbo, cc = cb / db, -b / db, ab / db                                # conic = inverse(cov + blur I)
    det_conic = ca * cc - cbo * cbo
    pt = torch.log(torch.clamp(255.0 * opac, min=1e-300))
    dcs = torch.where(det_conic > 0, det_conic, torch.ones_like(det_conic))
    ex = torch.sqrt(torch.clamp(2 * pt * cc / dcs, min=0.0))
    ey = torch.sqrt(torch.clamp(2 * pt * ca / dcs, min=0.0))
    cam_pos = torch.tensor([float(v) for v in u.cam_pos], dtype=F64)
    dvec = mean - cam_pos
    dlen = torch.sqrt((dvec * dvec).sum(-1))
    dirs = dvec / torch.where(dlen > 0, dlen, torch.ones_like(dlen))[:, None]
    Y = sh_basis(dirs, k)
    col = (Y[:, :, None] * sh).sum(1) + 0.5
    return SimpleNamespace(mc=mc, scale=scale, qn=qn, J=J, Rq=Rq, M=M, a=a, b=b, c=c, max_abs=max_abs, det_raw=det_raw,
                           det_b=det_b, comp=comp, opac=opac, sig=sig, ca=ca, cb=cbo, cc=cc, det_conic=det_conic,
                           pt=pt, ex=ex, ey=ey, mean2d=mean2d, dirs=dirs, Y=Y, col=col, blur=blur, det_ok=det_ok)


def _dg_dmean(u, mc):
    """d(clamp point)/d(camera-space mean): identity on a coordinate inside its clamp window; outside, the
    coordinate is the clamp limit times z."""
    x, y, z = mc.unbind(-1)
    xr, yr = x / z, y / z
    in_x = (xr <= u.lim_pos_x) & (xr >= u.lim_neg_x)
    in_y = (yr <= u.lim_pos_y) & (yr >= u.lim_neg_y)
    S = torch.zeros(mc.shape[0], 3, 3, dtype=F64)
    S[:, 0, 0] = in_x.to(F64)
    S[:, 0, 2] = torch.where(in_x, torch.zeros_like(xr), torch.clamp(xr, u.lim_neg_x, u.lim_pos_x))
    S[:, 1, 1] = in_y.to(F64)
    S[:, 1, 2] = torch.where(in_y, torch.zeros_like(yr), torch.clamp(yr, u.lim_neg_y, u.lim_pos_y))
    S[:, 2, 2] = 1.0
    return S


def _inputs(transforms, sh, raw_opac, grad=False):
    t = torch.tensor(np.asarray(transforms, np.float32).astype(np.float64), dtype=F64, requires_grad=grad)
    s = torch.tensor(np.asarray(sh, np.float32).astype(np.float64), dtype=F64, requires_grad=grad)
    o = torch.tensor(np.asarray(raw_opac, np.float32).astype(np.float64), dtype=F64, requires_grad=grad)
    return t, s, o


def _finite(*xs):
    ok = None
    for x in xs:
        f = torch.isfinite(x)
        f = f.all(-1) if f.dim() > 1 else f
        ok = f if ok is None else ok & f
    return ok


def project_reference(u, w, h, transforms, sh, raw_opac, mip=False):
    """Forward restatement.  Returns a namespace with
      visible [n] bool, projected [V, 9] (compact order: ascending f32 depth, ties by index, like the render),
      gid_from_cgid [V], rows [n, 9] (valid where visible), max_radius [n] (0 where culled),
      bound [n, 9] (allowed |f32 - ref| per element), flags [n] bool (ambiguous splats) with the per-threshold
      masks in `why` (a dict of [n] bool)."""
    with torch.no_grad():
        t, s, o = _inputs(transforms, sh, raw_opac)
        f = _forward(u, w, h, t, s, o, mip, grad=False)
    n = t.shape[0]
    model = u.camera_model
    mc, z = f.mc, f.mc[:, 2]
    r = torch.sqrt(mc[:, 0] ** 2 + mc[:, 1] ** 2)
    theta = torch.atan2(r, z)
    half = float(u.half_max_render_fov)
    in_front = (z >= 0.01) if model == PINHOLE else ~(theta > half)
    vis = _finite(mc) & (z <= 1e10) & in_front & _finite(f.scale) & (f.qn >= 1e-6) & torch.isfinite(f.qn)
    vis &= torch.isfinite(o) & f.det_ok & _finite(f.a, f.b, f.c) & (f.opac >= 1.0 / 255.0) & (f.det_conic > 0)
    mx, my = f.mean2d[:, 0], f.mean2d[:, 1]
    on_screen = (mx + f.ex > 0) & (mx - f.ex < w) & (my + f.ey > 0) & (my - f.ey < h)
    vis &= on_screen
    col = f.col
    colf = torch.clamp(torch.where(torch.isfinite(col), col, torch.zeros_like(col)), -100.0, 100.0)
    rows = torch.stack([mx, my, f.ca, f.cb, f.cc, f.opac, colf[:, 0], colf[:, 1], colf[:, 2]], -1)
    max_radius = torch.where(vis, torch.maximum(f.ex / w, f.ey / h), torch.zeros_like(f.ex))

    # ---- magnitude companions and bounds
    Rv, tv = _view(u)
    Vabs = f.J.abs() @ Rv.abs() @ f.Rq.abs() * f.scale[:, None, :]
    G = (Vabs @ Vabs.transpose(-1, -2)).amax((-1, -2))
    lam_conic = 0.5 * (f.ca + f.cc) + torch.sqrt(0.25 * (f.ca - f.cc) ** 2 + f.cb ** 2)
    m_conic = lam_conic ** 2 * (G + f.blur)
    # world_to_cam cancels when the mean is near the camera: carry |R_view| |mean| + |t| through x / z
    mca = t[:, 0:3].abs() @ Rv.abs().T + tv.abs()
    za = z.abs().clamp(min=1e-300)
    m_x = (mx - u.cx).abs() * (1 + mca[:, 0] / mc[:, 0].abs().clamp(min=1e-300) + mca[:, 2] / za)
    m_y = (my - u.cy).abs() * (1 + mca[:, 1] / mc[:, 1].abs().clamp(min=1e-300) + mca[:, 2] / za)
    m_x = torch.minimum(m_x, (mx - u.cx).abs() + u.fx * (mca[:, 0] + mca[:, 2] * (mc[:, 0] / za).abs()) / za)
    m_y = torch.minimum(m_y, (my - u.cy).abs() + u.fy * (mca[:, 1] + mca[:, 2] * (mc[:, 1] / za).abs()) / za)
    b_xy = C_XY * U * (m_x + abs(u.cx)), C_XY * U * (m_y + abs(u.cy))
    b_conic = C_CONIC * U * m_conic
    b_op = C_OPAC * U * f.opac
    if mip:
        s_det = f.a.abs() * f.c.abs() + f.b ** 2 + G * (f.a.abs() + f.c.abs() + 2 * f.b.abs())
        e_det = C_OPAC * U * s_det
        dbp = torch.clamp(f.det_b, min=1e-300)
        lin = e_det / (2 * torch.sqrt(torch.clamp(f.det_raw, min=1e-300) * dbp))
        sq = torch.sqrt(e_det / dbp)
        b_op = b_op + f.sig * torch.minimum(lin, sq)
    colm = (f.Y.abs()[:, :, None] * s.abs()).sum(1) + 0.5
    b_col = C_COLOR * U * colm * max(1.0, math.sqrt(s.shape[1]))
    bound = torch.stack([b_xy[0], b_xy[1], b_conic, b_conic, b_conic, b_op, b_col[:, 0], b_col[:, 1], b_col[:, 2]], -1)

    # ---- ambiguity: decisions within their f32 error of the threshold
    why = {}
    zt = 8 * U * ((Rv.abs() @ t[:, 0:3].abs().T).T + tv.abs())[:, 2]
    why["z"] = ((z - 0.01).abs() <= zt) if model == PINHOLE else torch.zeros(n, dtype=torch.bool)
    why["theta"] = ((theta - half).abs() <= 16 * U * (theta.abs() + half)) if model != PINHOLE \
        else torch.zeros(n, dtype=torch.bool)
    why["quat"] = (f.qn - 1e-6).abs() <= 8 * U * f.qn
    why["opacity"] = (f.opac - 1.0 / 255.0).abs() <= 2 * b_op + 8 * U * f.opac
    det_tol = 16 * U * (f.a.abs() * f.c.abs() + f.b ** 2 + G * (f.a.abs() + f.c.abs() + 2 * f.b.abs()))
    why["det"] = f.det_b.abs() <= det_tol
    # extents: ex ~ sqrt(2 pt cov00); relative error from pt (through the opacity) and from the conic
    rel_pt = (2 * b_op / f.opac.clamp(min=1e-300)) / f.pt.abs().clamp(min=1e-300)
    rel_cov = 2 * b_conic / torch.maximum(f.ca.abs(), f.cc.abs()).clamp(min=1e-300)
    tol_ex = 0.5 * f.ex * (rel_pt + rel_cov) + 8 * U * f.ex
    tol_ey = 0.5 * f.ey * (rel_pt + rel_cov) + 8 * U * f.ey
    tx, ty = 2 * b_xy[0] + tol_ex, 2 * b_xy[1] + tol_ey
    why["screen"] = ((mx + f.ex).abs() <= tx) | ((mx - f.ex - w).abs() <= tx) | \
        ((my + f.ey).abs() <= ty) | ((my - f.ey - h).abs() <= ty)
    if model in (PINHOLE, RT8):
        zs = torch.where(z.abs() > 0, z, torch.ones_like(z))
        xr, yr = mc[:, 0] / zs, mc[:, 1] / zs
        clamp_amb = torch.zeros(n, dtype=torch.bool)
        for v, lim in ((xr, u.lim_neg_x), (xr, u.lim_pos_x), (yr, u.lim_neg_y), (yr, u.lim_pos_y)):
            clamp_amb |= (v - lim).abs() <= 16 * U * (v.abs() + abs(lim)) + 8 * U * zt / zs.abs()
        why["clamp"] = clamp_amb
    else:
        why["clamp"] = torch.zeros(n, dtype=torch.bool)
    why["axis"] = ((r - 1e-6).abs() <= 16 * U * r + 8 * U * zt) if model in (KB4, TPF) \
        else torch.zeros(n, dtype=torch.bool)
    why["rescale"] = (f.max_abs - 1e18).abs() <= 16 * U * G
    flags = torch.zeros(n, dtype=torch.bool)
    for v in why.values():
        flags |= v
    # a splat culled for a non-finite value or a decision far from any threshold is not ambiguous; the flag
    # matters only where the decision could go either way
    vis_np = vis.numpy()
    depth32 = mc[:, 2].numpy().astype(np.float32)
    gids = np.nonzero(vis_np)[0]
    key = depth32[gids].view(np.uint32)
    order = gids[np.argsort(key, kind="stable")]
    rows_np = rows.numpy()
    return SimpleNamespace(
        visible=vis_np, rows=rows_np, projected=rows_np[order], gid_from_cgid=order.astype(np.int64),
        max_radius=max_radius.numpy(), bound=bound.numpy(), flags=flags.numpy(),
        why={k_: v.numpy() for k_, v in why.items()}, dirs=f.dirs.numpy(), mc=mc.numpy(),
        near_axis=(r < 1e-6).numpy(), m_conic=m_conic.numpy())


def project_reference_backward(u, w, h, transforms, sh, raw_opac, gid_from_cgid, v_combined, v_z=None, mip=False):
    """Backward restatement: v_combined [V, 10] (rows in the compact order `gid_from_cgid` of the render being
    checked, columns xy, conic a b c, rgb, opacity, refine) and optionally v_z [V] (gradient w.r.t. the camera-space
    depth of each mean) -> (v_transforms [n, 10], v_sh [n, K, 3], v_raw_opac [n], v_refine [n], v_color [n, 3]).
    Splats not in gid_from_cgid get zero rows."""
    t, s, o = _inputs(transforms, sh, raw_opac, grad=True)
    n, k = s.shape[0], s.shape[1]
    gid = np.asarray(gid_from_cgid, np.int64)
    vc = np.zeros((n, 10), np.float64)
    vc[gid] = np.asarray(v_combined)[: gid.shape[0]].astype(np.float64)   # f32 rows, or a float64 chain's
    vct = torch.tensor(vc, dtype=F64)
    f = _forward(u, w, h, t, s, o, mip, grad=True)
    live = torch.zeros(n, dtype=torch.bool)
    live[torch.from_numpy(gid)] = True
    # project_backwards.rs:189-194 feeds v_conic_b * 0.5 into the symmetric inverse's VJP: that is the derivative
    # with respect to the scalar off-diagonal b of the row, which autograd through the scalar conic gives.
    # The colour's non-finite -> 0 and +-100 clamp do not gate the colour gradient: the loss sees col itself.
    out = torch.stack([f.mean2d[:, 0], f.mean2d[:, 1], f.ca, f.cb, f.cc, f.col[:, 0], f.col[:, 1], f.col[:, 2],
                       f.opac], -1)
    out = torch.where(live[:, None], out, torch.zeros_like(out))
    loss = (out * vct[:, :9]).sum()
    if v_z is not None:
        vz = np.zeros(n, np.float64)
        vz[gid] = np.asarray(v_z)[: gid.shape[0]]
        loss = loss + (torch.where(live, f.mc[:, 2], torch.zeros_like(f.mc[:, 2])) * torch.tensor(vz, dtype=F64)).sum()
    vt, vsh, vo = torch.autograd.grad(loss, (t, s, o), allow_unused=True)
    vt = torch.zeros_like(t) if vt is None else vt
    # v_refine is the reference's pass-through (project_backwards.rs:185-188), in f32
    rin = np.asarray(v_combined, np.float32)[: gid.shape[0], 9]
    vr = np.zeros(n, np.float32)
    vr[gid] = np.clip(np.where(np.isfinite(rin), rin, np.float32(0)), np.float32(0), np.float32(1e32))
    vcol = np.zeros((n, 3))
    vcol[gid] = vc[gid, 5:8]
    return vt.detach().numpy(), vsh.detach().numpy(), vo.detach().numpy(), vr, vcol


def forward_check(ref, rows, gid_from_cgid, max_radius, exclude=None):
    """Rows [V, 9] of an f32 implementation (compact order `gid_from_cgid`) and its max_radius [n] against the
    restatement; returns (worst ratio per column, list of failure strings).  `exclude`: extra [n] mask."""
    gid = np.asarray(gid_from_cgid, np.int64)
    fails = []
    skip = ref.flags.copy()
    if exclude is not None:
        skip |= exclude
    mine = np.zeros(ref.visible.shape[0], bool)
    mine[gid] = True
    diff = (mine != ref.visible) & ~skip
    if diff.any():
        fails.append(f"visible set differs at {np.nonzero(diff)[0][:10]} (of {int(diff.sum())})")
    keep = ~skip[gid] & ref.visible[gid]
    g = gid[keep]
    got = np.asarray(rows, np.float64)[keep]
    want, bnd = ref.rows[g], ref.bound[g]
    err = np.abs(got - want)
    ratio = np.where(bnd > 0, err / np.maximum(bnd, 1e-300), np.where(err > 0, np.inf, 0.0))
    worst = ratio.max(0) if ratio.size else np.zeros(9)
    bad = ratio > 1.0
    names = ["x", "y", "conic_a", "conic_b", "conic_c", "opacity", "r", "g", "b"]
    for j in range(9):
        if bad[:, j].any():
            i = int(np.argmax(ratio[:, j]))
            fails.append(f"{names[j]}: {int(bad[:, j].sum())} of {bad.shape[0]} outside the bound; worst splat "
                         f"{int(g[i])}: got {got[i, j]!r} want {want[i, j]!r} bound {bnd[i, j]:.3e}")
    # max_radius: the extents' error bound, relative
    mr = np.asarray(max_radius, np.float64)
    ok = ~skip & ref.visible
    rel = np.abs(mr[ok] - ref.max_radius[ok]) / np.maximum(ref.max_radius[ok], 1e-300)
    tol = 0.5 * (ref.bound[ok, 5] / np.maximum(ref.rows[ok, 5], 1e-300)) / \
        np.maximum(np.log(255.0 * ref.rows[ok, 5]), 1e-300) + \
        ref.bound[ok, 2:5].max(1) / np.maximum(np.abs(ref.rows[ok, 2:5]).max(1), 1e-300) + 1e-6
    tol = 4 * tol
    if (rel > tol).any():
        fails.append(f"max_radius: {int((rel > tol).sum())} outside; worst rel {rel.max():.3e}")
    culled = ~ref.visible & ~skip
    if (mr[culled] != 0).any():
        fails.append("max_radius of a culled splat is not 0")
    return worst, fails


# ---- edge scenes: where projection kernels go wrong
EDGE_PARAMS = {
    PINHOLE: (),
    KB4: (-0.05, 0.01, -0.004, 1e-3),
    RT8: (-0.2, 0.05, -0.001, 0.01, -0.005, 0.001, 2e-3, -1.5e-3),
    TPF: (-0.05, 0.01, -0.004, 1e-3, 2e-3, -1.5e-3, 1e-3, -8e-4),
}


def edge_camera(model, rotated=True):
    """fov 1.2 x 1.0 rad, an off-centre principal point (so lim_neg != lim_pos), and -- when `rotated` -- a translated
    camera turned so that its forward axis is the world +x axis (the view direction of an on-axis splat is then a
    world axis)."""
    from brush_b200.camera import Camera
    if rotated:   # local +z -> world +x: a rotation of +90 deg about y
        s = math.sqrt(0.5)
        pos, rot = (0.3, -0.2, 0.5), (0.0, s, 0.0, s)
    else:
        pos, rot = (0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0)
    return Camera(position=pos, rotation=rot, fov_x=1.2, fov_y=1.0, center_uv=(0.42, 0.57), camera_model=model,
                  model_params=EDGE_PARAMS[model])


def edge_scene(model, w, h, k, seed, n_fill=256, rotated=True):
    """Splats at the edges of the projection (camera space, then to world), mixed with synthetic_scene rows so that
    every warp of the kernels is partly live.  Returns (camera, transforms, sh, raw_opac, tags) with tags [n] naming
    each splat's edge."""
    from brush_b200.camera import build_uniforms, _mat3_from_quat_xyzw
    from scenes import splitmix64, synthetic_scene
    cam = edge_camera(model, rotated)
    u = build_uniforms(cam, w, h)
    fx, fy = u.fx, u.fy
    rs = splitmix64(seed, 4096)
    ri = iter(rs)
    nxt = lambda: float(next(ri))
    rows, tags = [], []

    def add(tag, p, ls=(-3.5, -3.5, -3.5), q=(1.0, 0.1, -0.2, 0.3), ro=2.0):
        rows.append((list(p), list(q), list(ls), ro))
        tags.append(tag)

    half = float(u.half_max_render_fov)
    # near plane (pinhole) / fov cone (distorted): straddle the threshold at relative offsets 1e-1 .. 1e-7
    for e in range(1, 8):
        for sgn in (-1.0, 1.0):
            if model == PINHOLE:
                z = 0.01 * (1.0 + sgn * 10.0 ** -e)
                add("near", (0.001 * nxt(), -0.001 * nxt(), z), ls=(-7.0, -7.5, -7.2))
            else:
                th = half * (1.0 + sgn * 10.0 ** -e)
                phi = 2 * math.pi * nxt()
                d = 2.0 + nxt()
                add("fov", (d * math.sin(th) * math.cos(phi), d * math.sin(th) * math.sin(phi), d * math.cos(th)),
                    ls=(-1.5, -1.5, -1.5))
    # far outside the Jacobian clamp window, footprint still on screen: x only, y only, both
    for which in ("x", "y", "xy"):
        for side in (-1.0, 1.0):
            for fac in (1.3, 3.0, 10.0):
                z = 2.0 + nxt()
                lx = u.lim_pos_x if side > 0 else u.lim_neg_x
                ly = u.lim_pos_y if side > 0 else u.lim_neg_y
                x = fac * lx * z if "x" in which else 0.1 * z * (nxt() - 0.5)
                y = fac * ly * z if "y" in which else 0.1 * z * (nxt() - 0.5)
                s = math.log(0.7 * fac * z)
                add("clamp_" + which, (x, y, z), ls=(s, s - 0.3, s - 0.1), ro=0.0)
    # exactly on the optical axis (and a hair off it)
    for z in (0.5, 1.0, 3.0, 7.0):
        add("axis", (0.0, 0.0, z), ls=(-3.0, -3.2, -2.8))
        add("axis", (3e-7 * z, -2e-7 * z, z), ls=(-3.0, -3.2, -2.8))
    # needles: scale ratio 1e4
    for i in range(12):
        z = 1.5 + 4 * nxt()
        p = ((nxt() - 0.5) * 0.8 * z, (nxt() - 0.5) * 0.6 * z, z)
        big = math.log(0.3 + nxt())
        add("needle", p, ls=(big, big - math.log(1e4), big - math.log(3e3)),
            q=(nxt() - 0.5, nxt() - 0.5, nxt() - 0.5, nxt() - 0.5))
    # footprints near 1e6 px^2
    for i in range(6):
        z = 1.0 + nxt()
        s = math.log(600.0 * z / fx)
        add("huge", ((nxt() - 0.5) * 0.2 * z, (nxt() - 0.5) * 0.2 * z, z), ls=(s, s - 0.2, s + 0.1), ro=-3.0)
    # sub-pixel: the blur dominates; with Mip det_raw ~ 0 (flat) and det_raw < 0 by rounding (degenerate discs)
    for i in range(12):
        z = 1.0 + 5 * nxt()
        s = math.log(0.02 * z / fx)
        add("subpixel", ((nxt() - 0.5) * 0.8 * z, (nxt() - 0.5) * 0.6 * z, z), ls=(s, s + 0.5, s - 0.5), ro=3.0)
    for i in range(12):
        z = 1.0 + 5 * nxt()
        s = math.log(2.0 * z / fx)
        add("flat", ((nxt() - 0.5) * 0.8 * z, (nxt() - 0.5) * 0.6 * z, z), ls=(s, -25.0, -25.0),
            q=(nxt() - 0.5, nxt() - 0.5, nxt() - 0.5, nxt() - 0.5), ro=4.0)
    # unnormalised quaternions, |q|^2 from 1e-6 (the cut) to 1e6
    for e in (-6.0, -5.0, -3.0, 0.0, 3.0, 6.0):
        qq = np.array([nxt() - 0.5, nxt() - 0.5, nxt() - 0.5, nxt() - 0.5])
        qq *= math.sqrt(10.0 ** e) / np.linalg.norm(qq)
        z = 2.0 + nxt()
        add("quat", ((nxt() - 0.5) * 0.5 * z, (nxt() - 0.5) * 0.5 * z, z), ls=(-2.5, -3.0, -3.5), q=tuple(qq))
    # raw opacity near the 1/255 cut and at +-20
    cut = -math.log(254.0)
    for d in (-1e-2, -1e-4, -1e-6, 1e-6, 1e-4, 1e-2, 2.0):
        z = 2.0 + nxt()
        add("opacity", ((nxt() - 0.5) * 0.5 * z, (nxt() - 0.5) * 0.5 * z, z), ls=(-2.5, -2.5, -2.5), ro=cut + d)
    for ro in (-20.0, 20.0):
        add("opacity", (0.1, 0.1, 2.5), ls=(-2.5, -2.5, -2.5), ro=ro)
    n_edge = len(rows)
    # SH rows whose colour crosses +-100 or is non-finite (assigned below), view directions along each axis
    for tag in ("sh_big", "sh_big", "sh_nan", "sh_inf"):
        z = 2.0 + nxt()
        add(tag, ((nxt() - 0.5) * 0.5 * z, (nxt() - 0.5) * 0.5 * z, z), ls=(-2.5, -2.5, -2.5))

    cam0, ftr, fsh, fop = synthetic_scene(n_fill, w, h, k=k, seed=seed + 1)
    p_loc = np.array([r[0] for r in rows], np.float64)
    p_loc = np.concatenate([p_loc, ftr[:, 0:3].astype(np.float64)])
    # camera space -> world: x_world = R_cam x_local + position (the inverse of the camera's world_to_local)
    Rc = _mat3_from_quat_xyzw(cam.rotation).astype(np.float64).T   # columns -> matrix
    p_w = p_loc @ Rc.T + np.array(cam.position)
    n = p_w.shape[0]
    tr = np.zeros((n, 10), np.float32)
    tr[:, 0:3] = p_w
    tr[: len(rows), 3:7] = [r[1] for r in rows]
    tr[: len(rows), 7:10] = [r[2] for r in rows]
    tr[len(rows):, 3:10] = ftr[:, 3:10]
    op = np.concatenate([np.array([r[3] for r in rows], np.float32), fop])
    sh = np.zeros((n, k, 3), np.float32)
    sr = splitmix64(seed + 2, n * k * 3).reshape(n, k, 3)
    sh[:] = sr * 0.5 - 0.25
    sh[:, 0, :] = sr[:, 0, :] * 2.5 - 1.0
    tags = tags + ["fill"] * n_fill
    tg = np.array(tags)
    big = np.nonzero(tg == "sh_big")[0]
    sh[big[0], 0] = (400.0, -400.0, 354.0)        # colour crosses +100 / -100 / lands near 100.4
    sh[big[1], 0] = (-354.0, 353.0, 0.0)
    sh[np.nonzero(tg == "sh_nan")[0], 0, 1] = np.nan
    sh[np.nonzero(tg == "sh_inf")[0], 0, 2] = np.inf
    # a quarter of the filler splats sit exactly on a world axis through the camera: view direction +-x, +-y, +-z
    ax = np.eye(3)
    pos = np.array(cam.position, np.float32)
    for i in range(6):
        j = len(rows) + 3 * i
        tr[j, 0:3] = pos + (1.0 if i % 2 == 0 else -1.0) * (2.0 + i) * ax[i // 2].astype(np.float32)
        tg[j] = "axis_dir"
    return cam, tr, sh, op, tg
