"""The numpy restatement of the fused update pass (tests/update_ref.py) pinned against the CPU oracle and float64:
test_gpu_update.py compares the device with it bit for bit, so the restatement itself must be right."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import update_ref as U  # noqa: E402

LRS = dict(lr_mean=3.1e-5, lr_rotation=2e-3, lr_scale=5e-3, lr_coeffs_dc=2e-3, lr_coeffs_sh_scale=20.0, lr_opac=0.012)


_state, _grads = U.random_state, U.random_grads


@pytest.mark.parametrize("k", [1, 9])
def test_restatement_matches_oracle_adam(k):
    """update_ref.update_f32 against oracle.adam_step for t = 1..8, dense (transforms, opacity) and row-reduced (SH).
    The moments are formed by the same f32 operations in the same order: bit-identical.  The parameter update differs
    only where the restatement multiplies by a reciprocal and the oracle divides (m/bc1, v/bc2, the quotient): each of
    the three replaced quotients differs by <= 3 roundings, sqrt halves one of them, and the eps add and the lr product
    round once more, <= 13.5 u = 13.5 * 2^-24 < 2^-20 of the update term in all, plus 1 ulp of p."""
    from oracle import oracle as orc
    rng = np.random.default_rng(k)
    n = 700
    st = _state(n, k, rng)
    for t in range(1, 9):
        gr = _grads(n, k, rng)
        c = U.Consts(t, **LRS)
        new, _ = U.update_f32(st, gr, c)
        checks = []
        p, m, v = st["transforms"].copy(), st["m_t"].copy(), st["v_t"].copy()
        orc.adam_step(p, gr["v_transforms"].copy(), m, v, 1.0, t, lr_scale_per_col=c.lr_t)
        checks.append(("transforms", p, m, v, "m_t", "v_t"))
        sc = np.repeat(np.array([1.0] + [np.float32(1.0) / np.float32(20.0)] * (k - 1), np.float32), 3)
        p, m, v = st["sh"].reshape(n, -1).copy(), st["m_sh"].reshape(n, -1).copy(), st["v_sh"].copy()
        orc.adam_step(p, gr["v_sh_grad"].reshape(n, -1).copy(), m, v, LRS["lr_coeffs_dc"], t, lr_scale_per_col=sc, reduce_v=True)
        checks.append(("sh", p, m, v, "m_sh", "v_sh"))
        p, m, v = st["raw_opac"].reshape(n, 1).copy(), st["m_o"].reshape(n, 1).copy(), st["v_o"].reshape(n, 1).copy()
        orc.adam_step(p, gr["v_raw_opac"].reshape(n, 1).copy(), m, v, LRS["lr_opac"], t)
        checks.append(("raw_opac", p, m, v, "m_o", "v_o"))
        for name, p, m, v, mk, vk in checks:
            assert np.array_equal(new[mk].reshape(-1).view(np.uint32), m.reshape(-1).view(np.uint32)), (t, mk)
            assert np.array_equal(new[vk].reshape(-1).view(np.uint32), v.reshape(-1).view(np.uint32)), (t, vk)
            before = st[name].reshape(-1).astype(np.float64)
            got, want = new[name].reshape(-1).astype(np.float64), p.reshape(-1).astype(np.float64)
            tol = np.spacing(np.abs(p.reshape(-1))).astype(np.float64) + 2.0 ** -20 * np.abs(want - before)
            assert (np.abs(got - want) <= tol).all(), (t, name, np.abs(got - want).max())
        st = {**st, **new}


def test_restatement_matches_float64_adam():
    """update_f32 over eight steps against AdamScaled in float64, within update_ref.adam64_tol (derived there)."""
    rng = np.random.default_rng(3)
    n, k = 900, 16
    st = _state(n, k, rng)
    ref = U.Adam64(st, U.Consts(1, **LRS))
    for t in range(1, 9):
        gr = _grads(n, k, rng)
        c = U.Consts(t, **LRS)
        st, _ = U.update_f32(st, gr, c)
        ref.step_and_check(gr, c, st)


def test_folded_gate_opacity_matches_oracle_fold():
    """The gate opacity with a floor is what fold_min_scale makes of the same row: sigmoid(raw') == clamp(sig coef)."""
    from oracle import oracle as orc
    rng = np.random.default_rng(5)
    n = 5000
    tr = np.zeros((n, 10), np.float32)
    tr[:, 7:10] = np.log(rng.uniform(1e-4, 0.3, (n, 3)))
    raw = rng.uniform(-8, 8, n).astype(np.float32)
    f = rng.uniform(0.0, 0.05, n).astype(np.float32)
    _, raw_f = orc.fold_min_scale(tr, raw, f)
    got = U.fold_opacity64(raw, tr[:, 7:10], f)
    want = 1.0 / (1.0 + np.exp(-raw_f.astype(np.float64)))
    np.testing.assert_allclose(got, want, rtol=2e-5, atol=1e-9)
    # the example of a splat thin on one axis: sigmoid 0.5, coef 0.1 -> weight 0.95^150, not 0.5^150
    f1 = np.array([0.01], np.float32)
    ls = np.log(np.array([[1e4, 1e4, 0.1 * 0.01 / np.sqrt(0.99)]])).astype(np.float32)
    w = U.noise_weight64(np.zeros(1, np.float32), ls, np.ones(1, np.float32), f1)
    assert abs(w[0] / 0.95 ** 150 - 1.0) < 1e-4
    assert U.noise_weight64(np.zeros(1, np.float32), ls, np.ones(1, np.float32))[0] == 0.5 ** 150


def test_powi_and_constants():
    # each squaring doubles the relative error carried in and adds one rounding: <= (t + 2 log2(t+1)) u overall
    for t in (1, 2, 3, 7, 60_000):
        want = float(np.float32(0.999)) ** t
        assert abs(float(U.powi_f32(np.float32(0.999), t)) / want - 1.0) <= (t + 2 * np.log2(t + 1)) * 2.0 ** -24
    c = U.Consts(1, **LRS)
    assert c.f1 == np.float32(1.0) - np.float32(0.9) and c.inv_bc1 == np.float32(1.0) / c.f1
    assert c.lr_rest == np.float32(np.float32(1.0) / np.float32(20.0)) * np.float32(2e-3)
