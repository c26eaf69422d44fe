"""Float64 back-to-front restatement of the blend stage, and the near-opaque scenes it is checked on.

`blend_reference` renders the projected rows of a render (`oracle.render_forward(...).projected`, [V, 9]: mean x/y,
conic a/b/c, opacity, colour r/g/b) over the tile lists of that render, in float64, with the semantics of the header
comments of brush_b200/csrc/blend_{common.cuh,fwd.cu,bwd.cu}:

  sigma = 0.5 (a dx^2 + c dy^2) + b dx dy  (dx = mean - pixel centre);  g = exp(-sigma);  oa = opacity g
  a pair acts when sigma >= 0 and oa >= 1/255 (the unclamped oa);  alpha = min(0.999, oa);  T' = T (1 - alpha)
  an acting pair with T' <= 1e-4 stops the pixel and is not blended;  colour max(c, 0);  depth: colour z, no clamp,
  no background;  output rgb + T_end bg, a = 1 - T_end.

The thresholds are the f32 constants the kernels compare against (0.999f, 1/255.f, 1e-4f), widened exactly.

The VJP is formed back to front with suffix sums, dC/d alpha_i = T_i c_i - (sum_{j>i} vis_j c_j + T_end bg)/(1 - alpha_i),
not by the kernels' replay that subtracts each blended colour from the f32 final image: behind a near-opaque splat that
subtraction cancels to a few ulp of the front colour and is then multiplied by up to 1/(1 - 0.999), so agreeing with
a reference that does the same would say nothing about its accuracy.

Every decision within the f32 error of its threshold flags its pixel (`ambiguous`): sigma within its rounding of 0,
oa within ~1e-5 relative of 1/255 or of 0.999, and T' within a running first-order bound of its relative error of
1e-4 (each blend adds alpha/(1-alpha) eps_alpha + eps_32; a clamped alpha carries no error).  Tests exclude flagged
pixels and the splats that may act on them (`ambiguous_splats`).
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np

from brush_b200.camera import Camera, focal_to_fov, fov_to_focal
from scenes import splitmix64

TILE = 16
ALPHA_MAX = float(np.float32(0.999))
ALPHA_MIN = float(np.float32(1.0 / 255.0))
T_STOP = float(np.float32(1e-4))
AMB_REL = 1e-5        # relative window around the oa thresholds
EPS_SIGMA = 4e-7      # rounding of the f32 sigma, relative to the sum of its terms' magnitudes
EPS_OA = 3e-7         # ex2.approx / expf and the opacity product, relative
EPS_32 = 2.4e-7       # one (1 - alpha) and one product per blend, relative


def _tile_pixels(tiles_x):
    r = np.arange(TILE * TILE)
    lx, ly = r % TILE, r // TILE
    warp = (lx >= 8).astype(np.int64) + 2 * (ly >= 8).astype(np.int64)
    return lx, ly, warp


def blend_reference(projected, cgid_from_isect, tile_offsets, w, h, bg=(0.0, 0.0, 0.0), z=None, v_output=None,
                    v_depth=None):
    """Forward (and, with v_output, the VJP) of the blend over untrimmed tile lists `tile_offsets` [ty, tx, 2].

    Returns a namespace with
      img [h,w,4], depth [h,w] (z given), t_final [h,w];
      ambiguous [h,w] bool, ambiguous_splats (sorted compact ids that may act on a flagged pixel);
      n_blend, n_stop, n_clamped (blended pairs with oa > 0.999), n_acted_blocks (sum over (tile, 8x8 block) of the
      splats that acted on a live pixel of the block), and the same counts restricted to flagged pixels as the bound
      `flip_bound` (candidate pairs of flagged pixels);
      walked [tiles, 4] batches of 32 each warp walks before its block saturates;  list_len [tiles];
      per-pixel n_blend_px / n_stop_px [h,w];  decisions (int8 code of every evaluated pair, for flip detection);
      with v_output: v_combined [V,10] (v_xy, v_conic a/b/c, v_rgb, v_opac, refine), v_z [V] (z given).
    """
    P = np.asarray(projected, np.float64)
    V = P.shape[0]
    cg = np.asarray(cgid_from_isect, np.int64)
    toff = np.asarray(tile_offsets, np.int64)
    tiles_y, tiles_x = toff.shape[:2]
    toff = toff.reshape(-1, 2)
    lo, hi = toff[:, 0], toff[:, 1]
    lens = np.maximum(hi - lo, 0)
    order = np.argsort(-lens, kind="stable")
    order = order[lens[order] > 0]
    nt = len(order)
    bg = np.asarray(bg, np.float64)
    zz = None if z is None else np.asarray(z, np.float64)
    lx, ly, warp = _tile_pixels(tiles_x)
    tx0 = (order % tiles_x) * TILE
    ty0 = (order // tiles_x) * TILE
    pix_x = tx0[:, None] + lx[None, :]
    pix_y = ty0[:, None] + ly[None, :]
    inside = (pix_x < w) & (pix_y < h)
    pcx, pcy = pix_x + 0.5, pix_y + 0.5
    olens = lens[order]
    olo = lo[order]

    T = np.ones((nt, 256))
    done = ~inside
    rel = np.zeros((nt, 256))
    acc = np.zeros((nt, 256, 3))
    accd = np.zeros((nt, 256))
    amb = np.zeros((nt, 256), bool)
    nbl = np.zeros((nt, 256), np.int64)
    nst = np.zeros((nt, 256), np.int64)
    ncand = np.zeros((nt, 256), np.int64)
    n_clamped = 0
    n_acted_blocks = 0
    done_at = np.full((nt, 4), -1, np.int64)   # list position at which the block's last pixel got done
    for wb in range(4):
        sel = warp == wb
        done_at[done[:, sel].all(1), wb] = -2   # no pixel inside: the warp never walks
    steps, cands, codes = [], [], []
    for j in range(int(olens[0]) if nt else 0):
        k = int(np.searchsorted(-olens, -j, side="left"))   # tiles whose list is longer than j (sorted descending)
        ids = cg[olo[:k] + j]
        r = P[ids]
        dx = r[:, 0:1] - pcx[:k]
        dy = r[:, 1:2] - pcy[:k]
        ta, tc, tb = 0.5 * r[:, 2:3] * dx * dx, 0.5 * r[:, 4:5] * dy * dy, r[:, 3:4] * dx * dy
        sigma = ta + tc + tb
        err_s = EPS_SIGMA * (np.abs(ta) + np.abs(tc) + np.abs(tb))
        oa = r[:, 5:6] * np.exp(-sigma)
        alive = ~done[:k]
        T_k = T[:k]
        act = alive & (sigma >= 0.0) & (oa >= ALPHA_MIN)
        alpha = np.minimum(ALPHA_MAX, oa)
        Tn = T_k * (1.0 - alpha)
        blend = act & (Tn > T_STOP)
        stop = act & ~blend
        clamped = oa > ALPHA_MAX
        # ambiguity
        eps_a = err_s + EPS_OA
        near_sig = np.abs(sigma) < err_s   # (an exact 0 is exact in f32 too)
        cand = (sigma >= -err_s) & (oa >= ALPHA_MIN * (1.0 - AMB_REL - eps_a))
        a_flag = alive & (near_sig & (oa >= ALPHA_MIN * (1.0 - AMB_REL - eps_a)) |
                          cand & (np.abs(oa - ALPHA_MIN) <= ALPHA_MIN * (AMB_REL + eps_a)))
        a_flag |= act & (np.abs(oa - ALPHA_MAX) <= ALPHA_MAX * (AMB_REL + eps_a))
        rel_n = rel[:k] + np.where(clamped, 0.0, alpha / (1.0 - alpha) * eps_a) + EPS_32
        a_flag |= act & (np.abs(Tn - T_STOP) <= Tn * rel_n)
        amb[:k] |= a_flag
        # outputs
        vis = np.where(blend, alpha * T_k, 0.0)
        acc[:k] += vis[..., None] * np.maximum(r[:, None, 6:9], 0.0)
        if zz is not None:
            accd[:k] += vis * zz[ids][:, None]
        nbl[:k] += blend
        nst[:k] += stop
        ncand[:k] += cand
        n_clamped += int((blend & clamped).sum())
        for wb in range(4):
            n_acted_blocks += int(act[:, warp == wb].any(1).sum())
        if blend.any():
            idx = np.flatnonzero(blend)
            steps.append((j, k, ids, idx, T_k.ravel()[idx].copy()))
        cands.append((ids, np.nonzero(cand)))
        codes.append((act + 2 * blend + 4 * (act & clamped)).astype(np.int8).ravel())
        T[:k] = np.where(blend, Tn, T_k)
        rel[:k] = np.where(blend, rel_n, rel[:k])
        done[:k] |= stop
        for wb in range(4):
            newly = (done_at[:k, wb] == -1) & done[:k][:, warp == wb].all(1)
            done_at[:k, wb][newly] = j

    # per (tile, warp) batches walked: up to the batch in which the block saturated, else the whole list
    walked = np.zeros((tiles_x * tiles_y, 4), np.int64)
    nb = (olens + 31) // 32
    wk = np.where(done_at >= 0, done_at // 32 + 1, nb[:, None])
    wk[done_at == -2] = 0
    walked[order] = wk

    def scatter(a, fill=0.0):
        out = np.full((h, w) + a.shape[2:], fill, a.dtype)
        m = inside
        out[pix_y[m], pix_x[m]] = a[m]
        return out

    t_final = scatter(T, 1.0)
    rgb = scatter(acc) + t_final[..., None] * bg
    img = np.concatenate([rgb, (1.0 - t_final)[..., None]], -1)
    ambiguous = scatter(amb, False)
    amb_ids = set()
    for ids, (ti, pj) in cands:
        f = amb[ti, pj]
        amb_ids.update(ids[ti[f]].tolist())
    res = SimpleNamespace(
        img=img, depth=scatter(accd) if zz is not None else None, t_final=t_final, ambiguous=ambiguous,
        ambiguous_splats=np.array(sorted(amb_ids), np.int64), n_blend=int(nbl[inside].sum()),
        n_stop=int(nst[inside].sum()), n_clamped=n_clamped, n_acted_blocks=n_acted_blocks,
        flip_bound=int(ncand[amb].sum()), walked=walked, list_len=lens, n_blend_px=scatter(nbl),
        n_stop_px=scatter(nst), decisions=np.concatenate(codes) if codes else np.zeros(0, np.int8),
        v_combined=None, v_z=None)
    if v_output is None:
        return res

    # ---- VJP, back to front with suffix sums
    vo = np.asarray(v_output, np.float64)
    vo_t = np.zeros((nt, 256, 4))
    vo_t[inside] = vo[pix_y[inside], pix_x[inside]]
    vd_t = np.zeros((nt, 256))
    if zz is not None and v_depth is not None:
        vd_t[inside] = np.asarray(v_depth, np.float64)[pix_y[inside], pix_x[inside]]
    T_end = T.copy()
    inv_fa = 1.0 / np.maximum(1.0 - T_end, 1e-5)
    S = np.zeros((nt, 256, 3))        # colour of the splats behind, sum_{j>i} vis_j c_j
    Sd = np.zeros((nt, 256))
    end_term = (T_end[..., None] * bg[None, None, :] * vo_t[..., :3]).sum(-1) - T_end * vo_t[..., 3]
    vc = np.zeros((V, 10))
    vz = np.zeros(V)
    for j, k, ids, idx, T_i in reversed(steps):
        ti, lane = idx // 256, idx % 256
        gid = ids[ti]
        r = P[gid]
        dx = r[:, 0] - pcx[ti, lane]
        dy = r[:, 1] - pcy[ti, lane]
        sigma = 0.5 * (r[:, 2] * dx * dx + r[:, 4] * dy * dy) + r[:, 3] * dx * dy
        g = np.exp(-sigma)
        oa = r[:, 5] * g
        alpha = np.minimum(ALPHA_MAX, oa)
        c = np.maximum(r[:, 6:9], 0.0)
        v = vo_t[ti, lane]
        vis = alpha * T_i
        ra = 1.0 / (1.0 - alpha)
        v_alpha = (v[:, :3] * (T_i[:, None] * c - S[ti, lane] * ra[:, None])).sum(1) - end_term[ti, lane] * ra
        if zz is not None:
            zi = zz[gid]
            v_alpha += vd_t[ti, lane] * (T_i * zi - Sd[ti, lane] * ra)
            np.add.at(vz, gid, vis * vd_t[ti, lane])
            Sd[ti, lane] += vis * zi
        unsat = oa <= ALPHA_MAX
        v_sigma = np.where(unsat, -alpha * v_alpha, 0.0)
        vx = v_sigma * (r[:, 2] * dx + r[:, 3] * dy)
        vy = v_sigma * (r[:, 3] * dx + r[:, 4] * dy)
        cols = np.stack([
            vx, vy, 0.5 * v_sigma * dx * dx, v_sigma * dx * dy, 0.5 * v_sigma * dy * dy,
            np.where(r[:, 6] >= 0, vis * v[:, 0], 0.0), np.where(r[:, 7] >= 0, vis * v[:, 1], 0.0),
            np.where(r[:, 8] >= 0, vis * v[:, 2], 0.0), np.where(unsat, v_alpha * g, 0.0),
            np.sqrt((vx * w) ** 2 + (vy * h) ** 2) * inv_fa[ti, lane]], 1)
        np.add.at(vc, gid, cols)
        S[ti, lane] += vis[:, None] * c
    res.v_combined = vc
    res.v_z = vz if zz is not None else None
    return res


def reference_for(o, bg, z=False, v_output=None, v_depth=None):
    """blend_reference on the rows, lists and depths of an oracle render `o`."""
    return blend_reference(o.projected, o.cgid_from_isect, o.tile_offsets_untrimmed, o.w, o.h, bg=bg,
                           z=o.depths_sorted if z else None, v_output=v_output, v_depth=v_depth)


def opaque_scene(seed: int, n: int, w: int, h: int, k: int = 1, n_front: int = 60, n_specks: int = None,
                 n_mid: int = None, cluster: float = 0.2):
    """A near-opaque scene in the regime of a converged model, camera as in scenes.synthetic_scene (pinhole at the
    origin looking +z, fov_x 60 deg).  Layers, front to back:
      * front: n_front large splats, log-scales of synthetic_scene shifted by +2.5, depth U(2, 3), raw opacity
        U(7, 12): clamped cores, unclamped skirts, edges through tiles;
      * specks: sub-pixel splats (sigma 0.1 px before the 0.3 px^2 screen-space blur) at depth U(2, 6) whose means project onto pixel centres and raw
        opacity U(7, 12): their one acting pixel is clamped.  A Gaussian only clamps where oa > 0.999, i.e. within
        sigma < ln(opacity / 0.999) <= 1e-3 of its centre, so a footprint wider than a pixel has at most ~2e-4 of its
        pairs clamped; sub-pixel splats are what makes clamped pairs a sizeable share of the blend;
      * middle: n_mid splats, log-scales +1, depth U(3, 6), raw opacity U(6.5, 7.5) (straddling logit(0.999) = 6.907);
      * back: the rest, log-scales +0.5, depth U(6, 12), raw opacity U(-2, 8); a share `cluster` of it is drawn around
        one point of the image so that some tile lists exceed 512 entries.
    SH DC U(-2.5, 1.5): below -1.77 the colour is negative, so max(c, 0) and the gate of the colour gradient both
    act; higher bands U(-0.25, 0.25)."""
    fov_x = math.radians(60.0)
    focal = fov_to_focal(fov_x, w)
    fov_y = focal_to_fov(focal, h)
    cam = Camera(position=(0.0, 0.0, 0.0), rotation=(0.0, 0.0, 0.0, 1.0), fov_x=fov_x, fov_y=fov_y)
    if n_specks is None:
        n_specks = n // 4
    if n_mid is None:
        n_mid = n // 5
    n_back = n - n_front - n_specks - n_mid
    assert n_back > 0
    per = 3 + 3 + 4 + 1 + 3 * k
    r = splitmix64(seed, n * per).reshape(n, per)
    u = r[:, 0] * 2.1 - 1.05
    v = r[:, 1] * 2.1 - 1.05
    lo, hi = math.log(0.004), math.log(0.03)
    log_scales = lo + r[:, 3:6] * (hi - lo)
    raw = r[:, 10].copy()
    zdep = np.empty(n)
    f, s, m = n_front, n_front + n_specks, n_front + n_specks + n_mid
    zdep[:f] = 2.0 + r[:f, 2]
    log_scales[:f] += 2.5
    raw[:f] = 7.0 + 5.0 * r[:f, 10]
    zdep[f:s] = 2.0 + 4.0 * r[f:s, 2]
    raw[f:s] = 7.0 + 5.0 * r[f:s, 10]
    zdep[s:m] = 3.0 + 3.0 * r[s:m, 2]
    log_scales[s:m] += 1.5
    raw[s:m] = 6.5 + r[s:m, 10]
    zdep[m:] = 6.0 + 6.0 * r[m:, 2]
    log_scales[m:] += 1.0
    raw[m:] = -2.0 + 10.0 * r[m:, 10]
    nc = int(cluster * n_back)
    if nc:   # a dense patch: normal-ish around (0.3, -0.2) in NDC from the sum of three uniforms
        cu = 0.3 + 0.12 * (r[m:m + nc, 0] + r[m:m + nc, 1] + r[m:m + nc, 3] - 1.5)
        cv = -0.2 + 0.12 * (r[m:m + nc, 4] + r[m:m + nc, 5] + r[m:m + nc, 6] - 1.5)
        u[m:m + nc], v[m:m + nc] = cu, cv
    tx, ty = math.tan(fov_x / 2), math.tan(fov_y / 2)
    x = u * zdep * tx
    y = v * zdep * ty
    quats = r[:, 6:10] * 2.0 - 1.0
    # specks: isotropic, ~0.25 px, means on pixel centres (pinhole: px = fx x / z + cx)
    if n_specks:
        cx, cy = 0.5 * w, 0.5 * h
        pxs = np.floor(r[f:s, 0] * w) + 0.5
        pys = np.floor(r[f:s, 1] * h) + 0.5
        x[f:s] = (pxs - cx) * zdep[f:s] / focal
        y[f:s] = (pys - cy) * zdep[f:s] / focal
        log_scales[f:s] = np.log(0.1 * zdep[f:s] / focal)[:, None]
        quats[f:s] = (1.0, 0.0, 0.0, 0.0)
    means = np.stack([x, y, zdep], 1)
    sh = r[:, 11:].reshape(n, k, 3).copy()
    sh[:, 0, :] = sh[:, 0, :] * 4.0 - 2.5
    if k > 1:
        sh[:, 1:, :] = sh[:, 1:, :] * 0.5 - 0.25
    transforms = np.concatenate([means, quats, log_scales], 1).astype(np.float32)
    return cam, transforms, sh.astype(np.float32), raw.astype(np.float32)
