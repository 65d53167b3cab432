"""First-principles checks of the binary-trait GxE oracle (interaction_bt_oracle.py), without a GPU: the Wald fit is a
zero of the logistic score, V is the inverse of a finite-difference Hessian, HC3 matches a per-sample loop, each Firth
fit is a stationary point of the penalised log-likelihood in its free coordinates, and every LRT is >= 0."""
import numpy as np
import pytest

import interaction_bt_oracle as ibo
from oracle.prep import get_basis
from oracle.step1_bt import get_pvec


def problem(seed, N=600, case_rate=0.3, gxe=0.4):
    rng = np.random.default_rng(seed)
    ia = rng.random(N) > 0.05
    E = np.where(ia, rng.normal(size=N) * 1.5 + 0.3, 0.0)
    cov = rng.normal(size=(N, 2))
    X, _ = get_basis(np.column_stack([np.ones(N), cov, E, E * E]) * ia[:, None])
    g = np.where(ia, rng.binomial(2, 0.3, size=N).astype(float), 0.0)
    mask = ia & (rng.random(N) > 0.05)
    eta = np.log(case_rate / (1 - case_rate)) + 0.3 * cov[:, 0] + 0.2 * g + gxe * g * E / 1.5
    y = (rng.random(N) < 1 / (1 + np.exp(-eta))).astype(float) * mask
    offset = np.log(case_rate / (1 - case_rate)) + 0.3 * cov[:, 0] + rng.normal(size=N) * 0.05
    H, sf, scf = ibo.design(g, E, X, int(ia.sum()))
    return H, y, offset, mask


def loglik(H, y, offset, mask, b):
    p = get_pvec(offset + H @ b)
    return np.where(mask, y * np.log(p) + (1 - y) * np.log(1 - p), 0.0).sum()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_wald_is_a_zero_of_the_score_and_v_the_inverse_hessian(seed):
    H, y, offset, mask = problem(seed)
    st, b, V = ibo.wald(H, y, offset, mask, mac=50.0, rare_mac=1000.0)
    assert st == 3
    p = get_pvec(offset + H @ b)
    assert np.abs(H.T @ np.where(mask, y - p, 0.0)).max() < 1e-7
    e = 1e-4
    hess = np.zeros((2, 2))
    for j in range(2):
        for k in range(2):
            dj, dk = np.eye(2)[j] * e, np.eye(2)[k] * e
            hess[j, k] = (loglik(H, y, offset, mask, b + dj + dk) - loglik(H, y, offset, mask, b + dj - dk)
                          - loglik(H, y, offset, mask, b - dj + dk) + loglik(H, y, offset, mask, b - dj - dk)) / (4 * e * e)
    np.testing.assert_allclose(V, np.linalg.inv(-hess), rtol=1e-4)


def test_hc3_matches_a_per_sample_loop():
    H, y, offset, mask = problem(4)
    st, b, Vr = ibo.wald(H, y, offset, mask, mac=50.0, force_robust=True)
    _, _, V = ibo.wald(H, y, offset, mask, mac=50.0, no_robust=True)
    assert st == 1
    p = get_pvec(offset + H @ b)
    meat = np.zeros((2, 2))
    for i in range(len(y)):
        if not mask[i]:
            continue
        w = p[i] * (1 - p[i])
        h = w * H[i] @ V @ H[i]
        meat += ((y[i] - p[i]) / (1 - h)) ** 2 * np.outer(H[i], H[i])
    np.testing.assert_allclose(Vr, V @ meat @ V, rtol=1e-10)


def pen_loglik(H, y, offset, mask, b):
    return -0.5 * ibo.penalised_dev(y, H, offset, mask, b)


@pytest.mark.parametrize("seed,case_rate", [(5, 0.05), (6, 0.2), (7, 0.03)])
def test_firth_fits_are_stationary_and_lrts_nonnegative(seed, case_rate):
    H, y, offset, mask = problem(seed, case_rate=case_rate, gxe=0.8)
    st, b, se, lrt = ibo.firth(H, y, offset, mask)
    assert st == 0
    assert (lrt >= 0).all()
    e = 1e-5

    def grad(bb, free):
        return np.array([(pen_loglik(H, y, offset, mask, bb + np.eye(2)[j] * e)
                          - pen_loglik(H, y, offset, mask, bb - np.eye(2)[j] * e)) / (2 * e) for j in free])

    assert np.abs(grad(b, [0, 1])).max() < 1e-3                     # full fit: both coordinates free
    ok, bg, dev_g, _, _ = ibo.fit_firth_nr(y, H[:, ::-1], offset, mask, np.array([b[1], 0.0]), 1, False)
    assert ok
    assert np.abs(grad(np.array([0.0, bg[0]]), [1])).max() < 1e-3  # G dropped: only the GxE coefficient is free
    ok, bi, dev_i, _, _ = ibo.fit_firth_nr(y, H, offset, mask, np.array([b[0], 0.0]), 1, False)
    assert ok
    assert np.abs(grad(np.array([bi[0], 0.0]), [0])).max() < 1e-3  # GxE dropped
    # the LRTs are differences of the penalised deviances at the three optima
    dev = ibo.penalised_dev(y, H, offset, mask, b)
    np.testing.assert_allclose(lrt[1], ibo.penalised_dev(y, H, offset, mask, np.array([0.0, bg[0]])) - dev, atol=1e-9)
    np.testing.assert_allclose(lrt[2], ibo.penalised_dev(y, H, offset, mask, np.array([bi[0], 0.0])) - dev, atol=1e-9)
    np.testing.assert_allclose(lrt[0], ibo.penalised_dev(y, H, offset, mask, np.zeros(2)) - dev, atol=1e-9)
