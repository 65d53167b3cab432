"""First-principles checks of interaction_oracle.py that do not go through its restatement of regenie.

- Frisch-Waugh-Lovell: the robust route's BETA of G and G o E equal the OLS coefficients of G and G o E in a fit of the
  residual phenotype on [covariates, G, G o E]; the HLM route's equal the weighted least-squares coefficients of y on
  [X_hlm, G, G o E] with weights exp(-V b).
- The HLM null fit is a stationary point of its likelihood, and its analytic gradient matches finite differences.
"""
import numpy as np

import interaction_oracle as io


def problem(N=600, C=3, seed=1):
    rng = np.random.default_rng(seed)
    cov = np.column_stack([np.ones(N), rng.normal(size=(N, C - 1))])
    X, _ = np.linalg.qr(cov)
    E = cov[:, 1] * 1.3 + 0.5
    g = rng.binomial(2, 0.3, N).astype(float)
    mask = (rng.random((N, 2)) > 0.05).astype(float)
    y = (0.4 * cov[:, 1] + 0.2 * g + 0.15 * g * E + rng.normal(size=N) * np.exp(0.3 * E))[:, None] * mask
    res = y - X @ (X.T @ y)
    res *= mask
    return X, E, g, mask, res, rng


def test_robust_beta_is_ols_coefficient():
    X, E, g, mask, res, _ = problem()
    scf = np.array([1.7, 0.6])
    coef, vcov = io.robust(g, E, X, res, mask, scf, len(g), np.array([300.0, 300.0]))
    A = np.column_stack([X, g, g * E])
    for i in range(2):
        b = np.linalg.lstsq(A, res[:, i] * scf[i], rcond=None)[0]
        assert np.allclose(coef[i], b[-2:], rtol=1e-10)
        assert np.all(np.linalg.eigvalsh(vcov[i]) > 0)


def test_hlm_null_fit_is_stationary():
    X, E, g, mask, res, rng = problem()
    blup = rng.normal(size=len(g)) * 0.1
    V, Xh = io.hlm_design(E, X, blup)
    y = res[:, 0] + 2.0 * mask[:, 0]
    b, grad = io.hlm_fit(y, mask[:, 0], Xh, V)
    assert np.abs(grad).max() < 1e-8

    def nll(bb):                                                  # profile likelihood written out afresh
        dinv = np.exp(-V @ bb) * mask[:, 0]
        W = np.sqrt(dinv)
        a = np.linalg.lstsq(Xh * W[:, None], y * W, rcond=None)[0]
        return 0.5 * np.sum(mask[:, 0] * (V @ bb) + (y - Xh @ a) ** 2 * dinv) / mask[:, 0].sum()

    for k in range(len(b)):
        e = np.zeros(len(b)); e[k] = 1e-5
        assert abs((nll(b + e) - nll(b - e)) / 2e-5) < 1e-6
    # away from the optimum the analytic gradient of the oracle matches finite differences too
    b1 = b + 0.1
    for k in range(len(b)):
        e = np.zeros(len(b)); e[k] = 1e-6
        fd = (nll(b1 + e) - nll(b1 - e)) / 2e-6
        dinv = np.exp(-V @ b1) * mask[:, 0]
        a = np.linalg.lstsq(Xh * np.sqrt(dinv)[:, None], y * np.sqrt(dinv), rcond=None)[0]
        an = V[:, k] @ ((1 - (y - Xh @ a) ** 2 * dinv) * mask[:, 0]) / (2 * mask[:, 0].sum())
        assert abs(fd - an) < 1e-6 * max(1.0, abs(an))


def test_hlm_beta_is_weighted_least_squares():
    X, E, g, mask, res, rng = problem(seed=4)
    blup = rng.normal(size=len(g)) * 0.1
    V, Xh = io.hlm_design(E, X, blup)
    y = res[:, 1]
    b, _ = io.hlm_fit(y, mask[:, 1], Xh, V)
    d, Px, yres = io.hlm_state(y, mask[:, 1], Xh, V, b)
    coef, vcov = io.hlm_test(g, E, d, Px, yres)
    A = np.column_stack([Xh, g, g * E]) * d[:, None]
    want = np.linalg.lstsq(A, y * d, rcond=None)[0][-2:]
    assert np.allclose(coef, want, rtol=1e-8)
    assert np.allclose(vcov, np.linalg.inv(A.T @ A)[-2:, -2:], rtol=1e-8)
