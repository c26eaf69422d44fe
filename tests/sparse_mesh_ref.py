"""numpy restatement of the sparse brick TSDF's marking and allocation (DESIGN.md section 4.10, csrc/mesh_sparse.cu):
the near test (through mesh_ref's integration arithmetic), the pinhole candidate test with its expected-depth pyramid,
the one-brick dilation and the slot assignment in linear brick order."""
from __future__ import annotations

import numpy as np

import mesh_ref as mr

F = np.float32
B = 8
UNALLOCATED = 0xFFFFFFFF


def brick_dims(dims):
    return tuple((d + B - 1) // B for d in dims)


def near_points(origin, h, trunc, dims, u, img, depth, alpha_min=0.5):
    """bool [dz, dy, dx]: the points one pinhole view updates with f < 0.  One integration into a fresh grid leaves
    T = (0 * 0 + f) / 1 = f bit for bit (and +0 for f = -0), so T < 0 is exactly the near test."""
    g = mr.new_grid(dims)
    mr.integrate(g, origin, h, trunc, u.viewmat, u.fx, u.fy, u.cx, u.cy, img, depth, alpha_min)
    return g["tsdf"] < 0


def bricks_of(points, dims):
    """bool [nbz, nby, nbx]: bricks holding a True point."""
    nbx, nby, nbz = brick_dims(dims)
    out = np.zeros((nbz, nby, nbx), bool)
    k, j, i = np.nonzero(points)
    out[k // B, j // B, i // B] = True
    return out


def dilate(marked):
    """Bricks with a marked brick in their 3^3 neighbourhood."""
    nbz, nby, nbx = marked.shape
    p = np.zeros((nbz + 2, nby + 2, nbx + 2), bool)
    p[1:-1, 1:-1, 1:-1] = marked
    out = np.zeros_like(marked)
    for dz in range(3):
        for dy in range(3):
            for dx in range(3):
                out |= p[dz:dz + nbz, dy:dy + nby, dx:dx + nbx]
    return out


def assign_slots(alloc):
    """u32 [nbz, nby, nbx]: slots in linear brick order, UNALLOCATED elsewhere."""
    flat = alloc.reshape(-1)
    slots = np.full(flat.shape, UNALLOCATED, np.uint32)
    slots[flat] = np.arange(int(flat.sum()), dtype=np.uint32)
    return slots.reshape(alloc.shape)


# ---------------------------------------------------------------------------------------------- the candidate test
def _rd(x64):
    """float64 -> float32 rounded toward -inf."""
    y = np.asarray(x64, np.float64).astype(F)
    return np.where(y.astype(np.float64) > x64, np.nextafter(y, F(-np.inf)), y).astype(F)


def _ru(x64):
    y = np.asarray(x64, np.float64).astype(F)
    return np.where(y.astype(np.float64) < x64, np.nextafter(y, F(np.inf)), y).astype(F)


def pyramid(img, depth, alpha_min=0.5):
    """Levels of (min, max) of the valid expected depth D / a, each 2 x 2 cells of the one below, down to one cell."""
    a = img[..., 3].astype(F)
    with np.errstate(all="ignore"):
        ed = depth.astype(F) / a
        ok = (a >= F(alpha_min)) & (ed > 0) & np.isfinite(ed)
    lv = [(np.where(ok, ed, F(np.inf)).astype(F), np.where(ok, ed, F(-np.inf)).astype(F))]
    while lv[-1][0].shape != (1, 1):
        mn, mx = lv[-1]
        hh, ww = mn.shape
        H2, W2 = (hh + 1) // 2, (ww + 1) // 2
        pmn = np.full((2 * H2, 2 * W2), F(np.inf), F)
        pmx = np.full((2 * H2, 2 * W2), F(-np.inf), F)
        pmn[:hh, :ww], pmx[:hh, :ww] = mn, mx
        lv.append((pmn.reshape(H2, 2, W2, 2).min(axis=(1, 3)), pmx.reshape(H2, 2, W2, 2).max(axis=(1, 3))))
    return lv


def candidates(origin, h, trunc, dims, u, img, depth, alpha_min=0.5, pinhole=True):
    """bool [nbz, nby, nbx]: the bricks the candidate stage keeps for one view (marks from earlier views aside)."""
    H, W = depth.shape
    lv = pyramid(img, depth, alpha_min)
    nbx, nby, nbz = brick_dims(dims)
    vm = np.asarray(u.viewmat, F)
    out = np.zeros((nbz, nby, nbx), bool)
    org = [F(o) for o in origin]
    for bz in range(nbz):
        for by in range(nby):
            for bx in range(nbx):
                bi = (bx, by, bz)
                lo = [org[a] + F(bi[a] * B) * F(h) for a in range(3)]
                hi = [org[a] + F(min(bi[a] * B + 7, dims[a] - 1)) * F(h) for a in range(3)]
                mag = [max(abs(lo[a]), abs(hi[a])) for a in range(3)]
                cs = []
                for c in range(8):
                    x = np.array([hi[0] if c & 1 else lo[0], hi[1] if c & 2 else lo[1], hi[2] if c & 4 else lo[2]], F)
                    cs.append([((vm[a] * x[0] + vm[3 + a] * x[1]) + vm[6 + a] * x[2]) + vm[9 + a] for a in range(3)])
                cs = np.asarray(cs, F)
                cmin, cmax = cs.min(0), cs.max(0)
                grow = [F(2.0 ** -19) * (((abs(vm[a]) * F(mag[0]) + abs(vm[3 + a]) * F(mag[1])) + abs(vm[6 + a]) * F(mag[2]))
                                          + abs(vm[9 + a])) for a in range(3)]
                zl = _rd(np.float64(cmin[2]) - np.float64(grow[2]))
                zh = _ru(np.float64(cmax[2]) + np.float64(grow[2]))
                if not zh >= F(0.01):
                    continue
                x0, x1, y0, y1 = 0, W - 1, 0, H - 1
                if pinhole and zl >= F(0.01) and u.fx > 0 and u.fy > 0:
                    def bounds(lo_, hi_, f, c0):
                        l64, h64 = np.float64(lo_), np.float64(hi_)
                        rl = min(_rd(l64 / np.float64(zl)), _rd(l64 / np.float64(zh)))
                        rh = max(_ru(h64 / np.float64(zl)), _ru(h64 / np.float64(zh)))
                        ul = _rd(np.float64(_rd(np.float64(F(f)) * np.float64(rl))) + np.float64(F(c0))) - F(1)
                        uh = _ru(np.float64(_ru(np.float64(F(f)) * np.float64(rh))) + np.float64(F(c0))) + F(1)
                        return F(ul), F(uh)
                    ul, uh = bounds(_rd(np.float64(cmin[0]) - grow[0]), _ru(np.float64(cmax[0]) + grow[0]), u.fx, u.cx)
                    vl, vh = bounds(_rd(np.float64(cmin[1]) - grow[1]), _ru(np.float64(cmax[1]) + grow[1]), u.fy, u.cy)
                    if np.isfinite([ul, uh, vl, vh]).all():
                        if uh < 0 or ul >= W or vh < 0 or vl >= H:
                            continue
                        x0, x1 = int(max(ul, 0)), int(min(uh, F(W - 1)))
                        y0, y1 = int(max(vl, 0)), int(min(vh, F(H - 1)))
                ed_lo = _rd(np.float64(zl) - np.float64(_ru(np.float64(F(trunc)) * (1.0 + 2.0 ** -20))))
                L = 0
                while (x1 >> L) - (x0 >> L) > 3 or (y1 >> L) - (y0 >> L) > 3:
                    L += 1
                mn, mx = lv[L]
                sel = (slice(y0 >> L, (y1 >> L) + 1), slice(x0 >> L, (x1 >> L) + 1))
                out[bz, by, bx] = bool(((mn[sel] <= zh) & (mx[sel] >= ed_lo)).any())
    return out
