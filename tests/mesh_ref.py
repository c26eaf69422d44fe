"""numpy restatement of the mesh export of DESIGN.md section 4.9 (csrc/mesh.cu): TSDF integration of one pinhole view and
marching-tetrahedra extraction, in float32 with every operation rounded on its own, so that the device results must
match bit for bit."""
from __future__ import annotations

import numpy as np

F = np.float32
DIR_BITS = (1, 2, 4, 3, 5, 6, 7)                       # x, y, z, xy, xz, yz, xyz (x = 1, y = 2, z = 4)
DIR_INDEX = {b: d for d, b in enumerate(DIR_BITS)}
TETS = ((1, 2, 4), (1, 4, 2), (2, 1, 4), (2, 4, 1), (4, 1, 2), (4, 2, 1))   # xyz, xzy, yxz, yzx, zxy, zyx


def new_grid(dims):
    """dims = (dx, dy, dz); arrays in the [dz, dy, dx] layout, zeroed."""
    dx, dy, dz = dims
    return {"tsdf": np.zeros((dz, dy, dx), F), "weight": np.zeros((dz, dy, dx), F), "rgb": np.zeros((dz, dy, dx, 3), F)}


def lattice(origin, h, dims):
    """World positions [dz, dy, dx, 3]: origin + float(i) * h per axis."""
    dx, dy, dz = dims
    ax = [F(origin[a]) + np.arange(n, dtype=F) * F(h) for a, n in enumerate((dx, dy, dz))]
    x = np.broadcast_to(ax[0][None, None, :], (dz, dy, dx))
    y = np.broadcast_to(ax[1][None, :, None], (dz, dy, dx))
    z = np.broadcast_to(ax[2][:, None, None], (dz, dy, dx))
    return np.stack([x, y, z], -1).astype(F)


def integrate(grid, origin, h, trunc, viewmat, fx, fy, cx, cy, img, depth, alpha_min=0.5):
    """One pinhole view: img [H,W,4] (black background), depth [H,W]; updates grid in place."""
    dims = grid["tsdf"].shape[::-1]
    H, W = depth.shape
    p = lattice(origin, h, dims).reshape(-1, 3)
    vm = np.asarray(viewmat, F)
    with np.errstate(all="ignore"):
        xc = [((vm[a] * p[:, 0] + vm[3 + a] * p[:, 1]) + vm[6 + a] * p[:, 2]) + vm[9 + a] for a in range(3)]
        z = xc[2]
        ok = (z >= F(0.01)) & np.isfinite(z)
        inv_z = F(1.0) / z
        u = (F(fx) * xc[0]) * inv_z + F(cx)
        v = (F(fy) * xc[1]) * inv_z + F(cy)
        ok &= (u >= 0) & (u < F(W)) & (v >= 0) & (v < F(H))
        idx = np.nonzero(ok)[0]
        px, py = u[idx].astype(np.int64), v[idx].astype(np.int64)
        c = img[py, px].astype(F)
        a = c[:, 3]
        keep = a >= F(alpha_min)
        ed = depth[py, px].astype(F) / a
        keep &= (ed > 0) & np.isfinite(ed)
        sdf = ed - z[idx]
        keep &= ~(sdf < -F(trunc))
        idx, sdf, c, a = idx[keep], sdf[keep], c[keep], a[keep]
        f = np.fmin(F(1.0), sdf / F(trunc))
        col = np.fmin(np.fmax(c[:, :3] / a[:, None], F(0.0)), F(1.0))
    T, Wt, C = grid["tsdf"].reshape(-1), grid["weight"].reshape(-1), grid["rgb"].reshape(-1, 3)
    w0 = Wt[idx]
    w1 = w0 + F(1.0)
    T[idx] = (T[idx] * w0 + f) / w1
    C[idx] = (C[idx] * w0[:, None] + col) / w1[:, None]
    Wt[idx] = w1


def brick_order(dims, shrink=0):
    """Linear indices of the points (i, j, k) with i < dx - shrink etc., in brick-major order: 8^3 bricks in linear order,
    points x-fastest inside a brick."""
    dx, dy, dz = dims
    k, j, i = np.meshgrid(np.arange(dz - shrink), np.arange(dy - shrink), np.arange(dx - shrink), indexing="ij")
    i, j, k = i.ravel(), j.ravel(), k.ravel()
    nbx, nby = (dx + 7) // 8, (dy + 7) // 8
    key = (((k // 8) * nby + j // 8) * nbx + i // 8) * 512 + ((k % 8) * 8 + j % 8) * 8 + i % 8
    o = np.argsort(key, kind="stable")
    return i[o], j[o], k[o]


def _tet_table():
    """[6 tets][16 sign patterns] -> list of triangles, each three (a, b) tetrahedron corner pairs, wound so that the
    normal points toward T >= 0 (DESIGN.md section 4.9)."""
    table = []
    for t in range(6):
        even = t in (0, 3, 4)                           # xyz, yzx, zxy: positive orientation
        rows = []
        for s in range(16):
            neg = [(s >> v) & 1 for v in range(4)]
            n = sum(neg)
            tris = []
            if n in (1, 3):
                i = neg.index(1) if n == 1 else neg.index(0)
                j, k, l = [v for v in range(4) if v != i]
                det_pos = (i % 2 == 0) == even
                if (n == 1) == det_pos:
                    tris.append(((i, j), (i, k), (i, l)))
                else:
                    tris.append(((i, j), (i, l), (i, k)))
            elif n == 2:
                ni, nj = [v for v in range(4) if neg[v]]
                pk, pl = [v for v in range(4) if not neg[v]]
                perm_even = s not in (5, 10)
                ik, il, jl, jk = (ni, pk), (ni, pl), (nj, pl), (nj, pk)
                if perm_even == even:
                    tris += [(ik, il, jl), (ik, jl, jk)]
                else:
                    tris += [(ik, jl, il), (ik, jk, jl)]
            rows.append(tris)
        table.append(rows)
    return table


TET_TABLE = _tet_table()


def tet_corner_bits(t):
    a, b, _ = TETS[t]
    return (0, a, a | b, 7)


def extract(grid, origin, h):
    """Returns vertices f32 [V,3], colors u8 [V,3], faces i64 [F,3] in the device's order."""
    T, Wt, C = grid["tsdf"], grid["weight"], grid["rgb"]
    dz, dy, dx = T.shape
    dims = (dx, dy, dz)
    obs = Wt != 0
    neg = T < 0
    org = np.asarray(origin, F)
    # edge masks of every point
    mask = np.zeros((dz, dy, dx), np.int64)
    for d, bits in enumerate(DIR_BITS):
        ex, ey, ez = bits & 1, (bits >> 1) & 1, bits >> 2
        if dx - ex <= 0 or dy - ey <= 0 or dz - ez <= 0:
            continue
        sl0 = (slice(0, dz - ez), slice(0, dy - ey), slice(0, dx - ex))
        sl1 = (slice(ez, dz), slice(ey, dy), slice(ex, dx))
        m = obs[sl0] & obs[sl1] & (neg[sl0] != neg[sl1])
        mask[sl0] |= m.astype(np.int64) << d
    i, j, k = brick_order(dims)
    pm = mask[k, j, i]
    cnt = np.array([bin(x).count("1") for x in range(128)], np.int64)[pm]
    vbase = np.zeros((dz, dy, dx), np.int64)
    vbase[k, j, i] = np.cumsum(cnt) - cnt
    # vertices: (point, direction) in point order, then direction order
    bitsel = ((pm[:, None] >> np.arange(7)[None, :]) & 1).astype(bool)
    pidx, didx = np.nonzero(bitsel)
    pi, pj, pk = i[pidx], j[pidx], k[pidx]
    db = np.array(DIR_BITS)[didx]
    qi, qj, qk = pi + (db & 1), pj + ((db >> 1) & 1), pk + (db >> 2)
    tp, tq = T[pk, pj, pi], T[qk, qj, qi]
    with np.errstate(all="ignore"):
        t = tp / (tp - tq)
        verts = np.empty((len(pidx), 3), F)
        cols = np.empty((len(pidx), 3), np.uint8)
        for a, (p_, q_) in enumerate(((pi, qi), (pj, qj), (pk, qk))):
            x0 = org[a] + p_.astype(F) * F(h)
            x1 = org[a] + q_.astype(F) * F(h)
            verts[:, a] = x0 + t * (x1 - x0)
            c0, c1 = C[pk, pj, pi, a], C[qk, qj, qi, a]
            cc = np.fmin(np.fmax(c0 + t * (c1 - c0), F(0.0)), F(1.0))
            cols[:, a] = np.rint(cc * F(255.0)).astype(np.uint8)
    # faces: cells in brick order of their lower corner, 6 tetrahedra each
    faces = []
    if dx >= 2 and dy >= 2 and dz >= 2:
        ci, cj, ck = brick_order(dims, shrink=1)
        ci, cj, ck = _filter_cells(ci, cj, ck, dims)
        corner_obs = np.ones(len(ci), bool)
        cneg = []
        for b in range(8):
            ii, jj, kk = ci + (b & 1), cj + ((b >> 1) & 1), ck + (b >> 2)
            corner_obs &= obs[kk, jj, ii]
            cneg.append(neg[kk, jj, ii].astype(np.int64))
        per_cell = []
        for t in range(6):
            cb = tet_corner_bits(t)
            s = cneg[cb[0]] | (cneg[cb[1]] << 1) | (cneg[cb[2]] << 2) | (cneg[cb[3]] << 3)
            slots = np.full((len(ci), 2, 3), -1, np.int64)
            for sv in range(16):
                tris = TET_TABLE[t][sv]
                sel = np.nonzero(corner_obs & (s == sv))[0]
                if not len(sel) or not tris:
                    continue
                for n_tri, tri in enumerate(tris):
                    for v, (a, b) in enumerate(tri):
                        lo, hi = (a, b) if a < b else (b, a)
                        ca, cbb = cb[lo], cb[hi]
                        oi, oj, ok = ci[sel] + (ca & 1), cj[sel] + ((ca >> 1) & 1), ck[sel] + (ca >> 2)
                        d = DIR_INDEX[ca ^ cbb]
                        om = mask[ok, oj, oi]
                        below = np.array([bin(x).count("1") for x in range(128)], np.int64)[om & ((1 << d) - 1)]
                        slots[sel, n_tri, v] = vbase[ok, oj, oi] + below
            per_cell.append(slots)
        allf = np.stack(per_cell, 1).reshape(-1, 3)     # [cells, 6 tets, 2 slots] flattened in that order
        faces = allf[allf[:, 0] >= 0]
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    return verts, cols, faces


def _filter_cells(ci, cj, ck, dims):
    dx, dy, dz = dims
    m = (ci < dx - 1) & (cj < dy - 1) & (ck < dz - 1)
    return ci[m], cj[m], ck[m]
