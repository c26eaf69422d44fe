"""Restatements of the depth-supervision term (DESIGN.md section 4.7) for the tests.

With a = out_img[...,3], ed = D / a, a pixel active when its target t is finite and > 0 and a >= 1/255:
  L_d = c * sum_active |ed - t|,   c = w_d / |valid|
  dL/dD = c * sign(ed - t) / a,    dL/da = -(dL/dD) * ed     (0 on inactive pixels; sign(0) = 0)
"""
import numpy as np

ALPHA_MIN = np.float32(1.0) / np.float32(255.0)


def active_mask(a, t):
    with np.errstate(invalid="ignore"):
        return np.isfinite(t) & (t > 0) & (a >= ALPHA_MIN)


def loss_f64(D, a, t, chain):
    D, a, t = (np.asarray(x, np.float64) for x in (D, a, t))
    act = active_mask(a, t)
    return float(chain) * float(np.abs(D[act] / a[act] - t[act]).sum())


def grad_f64(D, a, t, chain):
    """(dL/dD, dL/da), both [h,w] float64."""
    D, a, t = (np.asarray(x, np.float64) for x in (D, a, t))
    act = active_mask(a, t)
    gD, ga = np.zeros_like(D), np.zeros_like(D)
    ed = D[act] / a[act]
    gD[act] = float(chain) * np.sign(ed - t[act]) / a[act]
    ga[act] = -gD[act] * ed
    return gD, ga


def fused_f32(out_img, D, t, chain, v_output):
    """What bg_depth_loss_fused computes, operation for operation in float32: (v_depth, v_output after the update,
    sum of |ed - t| over the active pixels in float64)."""
    f = np.float32
    a = out_img[..., 3].astype(f)
    D, t = D.astype(f), t.astype(f)
    act = active_mask(a, t)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        ed = (D / a).astype(f)
        diff = (ed - t).astype(f)
        s = np.where(diff > 0, f(1.0), np.where(diff < 0, f(-1.0), f(0.0))).astype(f)
        vd = ((f(chain) * s).astype(f) / a).astype(f)
        va = (-(vd * ed)).astype(f)
    v_depth = np.where(act, vd, f(0.0)).astype(f)
    vo = v_output.astype(f).copy()
    vo[..., 3] = np.where(act, (vo[..., 3] + va).astype(f), vo[..., 3])
    return v_depth, vo, float(np.abs(diff[act].astype(np.float64)).sum())
