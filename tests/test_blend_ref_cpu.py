"""The float64 blend reference (tests/blend_ref.py) against the CPU oracle and against central differences of itself,
on the near-opaque scenes of a converged model: clamped alphas, stopped pixels, tile lists longer than 512 entries.

Measured: on opaque_scene(256x256, 20k splats) the oracle's image agrees with the reference to 4e-7 on every
non-flagged pixel, and its backward's per-column relative L2 error against the reference VJP (non-flagged splats) is
1.2e-6 (v_xy), 0.7e-7..1.8e-7 (v_conic), 1.2e-7..1.6e-7 (v_rgb), 1.1e-6 (v_opac), 3.6e-7 (refine).
"""
import numpy as np
import pytest

from blend_ref import blend_reference, opaque_scene, reference_for
from scenes import random_v_output, splitmix64, synthetic_scene

BG = (0.1, 0.2, 0.3)
COLS = ["v_xy_x", "v_xy_y", "v_conic_a", "v_conic_b", "v_conic_c", "v_r", "v_g", "v_b", "v_opac", "refine"]


@pytest.fixture(scope="module")
def orc():
    from oracle import oracle
    return oracle


@pytest.fixture(scope="module")
def orcd():
    from oracle import oracle_depth
    return oracle_depth


def _render(orc, scene, w, h, mip=False):
    from brush_b200.camera import build_uniforms
    cam, tr, sh, op = scene
    return orc.render_forward(build_uniforms(cam, w, h), w, h, tr, sh, op, mip=mip, bg=BG)


def _close(got, ref, mask, rtol=1e-4, atol=1e-5):
    err = np.abs(got.astype(np.float64) - ref)[mask]
    bad = err > atol + rtol * np.abs(ref[mask])
    assert not bad.any(), f"{bad.sum()} of {bad.size} outside tolerance, max err {err.max():.3e}"


@pytest.mark.parametrize("kind,mip", [("synthetic", False), ("opaque", False), ("opaque", True)])
def test_reference_forward_vs_oracle(orc, orcd, kind, mip):
    w, h = 200, 150
    if kind == "synthetic":
        scene = synthetic_scene(8_000, w, h, k=4, seed=0xB1E100)
    else:
        scene = opaque_scene(0xB1E101, 12_000, w, h, k=4)
    o = _render(orc, scene, w, h, mip)
    r = reference_for(o, BG, z=True)
    ok = ~r.ambiguous
    assert ok.mean() > 0.999
    _close(o.out_img, r.img, ok[..., None].repeat(4, -1))
    _close(orcd.render_depth(o), r.depth, ok)
    if kind == "opaque":
        assert r.n_stop > 0.2 * w * h and r.list_len.max() >= 512 and r.n_clamped > 0


def _fd_rows(seed):
    """A 48x48 opaque scene: clamped cores, stops (each speck has a copy behind it on the same pixel ray, whose
    clamped alpha stops the pixel), a negative colour."""
    from oracle import oracle as orc
    w = h = 48
    cam, tr, sh, op = opaque_scene(seed, 60, w, h, k=1, n_front=8, n_specks=16, n_mid=12)
    back = tr[8:24].copy()
    back[:, 0:3] *= 1.3
    tr, sh, op = np.concatenate([tr, back]), np.concatenate([sh, sh[8:24]]), np.concatenate([op, op[8:24]])
    o = _render(orc, (cam, tr, sh, op), w, h)
    P = o.projected.astype(np.float64).copy()
    u = splitmix64(seed + 1, P.shape[0])
    P[:, 6] = u * 1.3 - 0.3   # red in [-0.3, 1): some negative
    return o, P


@pytest.mark.parametrize("seed", [0xFD02, 0xFD03])
def test_reference_vjp_vs_central_differences(orc, seed):
    """Every row entry (xy, conic a/b/c, rgb, opacity) and z of every splat that blends, against float64 central
    differences of the reference forward; entries whose +-eps perturbation flips a decision are skipped."""
    o, P = _fd_rows(seed)
    w, h = o.w, o.h
    cg, toff, z = o.cgid_from_isect, o.tile_offsets_untrimmed, o.depths_sorted.astype(np.float64)
    v_out = random_v_output(h, w, seed + 2).astype(np.float64)
    v_d = splitmix64(seed + 3, h * w).reshape(h, w)
    r = blend_reference(P, cg, toff, w, h, BG, z=z, v_output=v_out, v_depth=v_d)
    assert r.n_clamped > 0 and r.n_stop > 0 and (P[:, 6] < 0).any() and not r.ambiguous.any()

    def loss(P2, z2):
        q = blend_reference(P2, cg, toff, w, h, BG, z=z2)
        return (q.img * v_out).sum() + (q.depth * v_d).sum(), q.decisions

    active = np.unique(np.concatenate([np.flatnonzero(r.v_combined[:, 5:8].any(1)), np.flatnonzero(r.v_z)]))
    assert len(active) >= 20
    checked, skipped = 0, 0
    fails = []
    for i in active:
        for c in list(range(9)) + ["z"]:
            x = z[i] if c == "z" else P[i, c]
            if c == "z":
                eps = 1e-5 * abs(x)
            elif c in (2, 3, 4):   # conic entries: steps on the scale of the row's diagonal
                eps = 1e-5 * max(abs(P[i, 2]), abs(P[i, 4]))
            else:
                eps = 1e-5 * max(abs(x), 0.1 * np.abs(P[:, c]).max())
            if c in (6, 7, 8) and abs(x) <= eps:   # the step would cross the kink of max(c, 0)
                skipped += 1
                continue
            vals = []
            for sgn in (1, -1):
                P2, z2 = P.copy(), z.copy()
                if c == "z":
                    z2[i] += sgn * eps
                else:
                    P2[i, c] += sgn * eps
                vals.append(loss(P2, z2))
            if not (np.array_equal(vals[0][1], r.decisions) and np.array_equal(vals[1][1], r.decisions)):
                skipped += 1
                continue
            num = (vals[0][0] - vals[1][0]) / (2 * eps)
            # v_combined column of each row entry: xy -> 0,1; conic a,b,c -> 2,3,4; opacity -> 8; rgb -> 5,6,7
            an = r.v_z[i] if c == "z" else r.v_combined[i, [0, 1, 2, 3, 4, 8, 5, 6, 7][c]]
            checked += 1
            if abs(num - an) > 1e-6 + 1e-5 * abs(an):
                fails.append(f"splat {i} entry {c}: fd {num:.9g} vjp {an:.9g}")
    assert not fails, "\n".join(fails[:20])
    assert checked >= 10 * len(active) * 0.9, (checked, skipped)


def test_oracle_backward_vs_reference(orc, orcd):
    """The oracle's f32 backward (rem-subtraction replay) against the float64 suffix-sum VJP, on non-flagged splats:
    per-column relative L2 error <= 1e-5 (measured <= 1.4e-6, see the module docstring)."""
    w, h = 256, 256
    o = _render(orc, opaque_scene(0xB1E0 + 20_000, 20_000, w, h), w, h)
    v_out = random_v_output(h, w)
    v_d = splitmix64(0xDE0001, h * w).reshape(h, w).astype(np.float32)
    r = reference_for(o, BG, z=True, v_output=v_out, v_depth=v_d)
    keep = np.ones(o.num_visible, bool)
    keep[r.ambiguous_splats] = False
    assert keep.mean() > 0.9
    ovc = orc.rasterize_backward(o, v_out)
    dvc, dvz = orcd.rasterize_backward_depth(o, v_out, v_d)
    r0 = reference_for(o, BG, v_output=v_out)
    for got, ref, nm in ((ovc, r0.v_combined, ""), (dvc, r.v_combined, " (depth)")):
        for col, name in enumerate(COLS):
            a, b = got[keep, col].astype(np.float64), ref[keep, col]
            rel = np.linalg.norm(a - b) / np.linalg.norm(b)
            assert rel <= 1e-5, f"{name}{nm}: relative L2 {rel:.3e}"
    rel = np.linalg.norm(dvz[keep] - r.v_z[keep]) / np.linalg.norm(r.v_z[keep])
    assert rel <= 1e-5, f"v_z: relative L2 {rel:.3e}"
