"""numpy restatement of regenie's GxE interaction tests for quantitative traits, E kept as a covariate (gwas_condtl).

- robust route: get_interaction_terms + residualize_geno + apply_interaction_tests_qt (src/Interaction.cpp:44-92,
  :109-286, src/Geno.cpp:3242-3261, src/Pheno.cpp:1836-1852);
- HLM null model: HLM::prep_run / HLM_fitNull / store_null_est (src/HLM.cpp:49-92, :97-198, :222-243), the same
  likelihood minimised with scipy instead of LBFGSpp;
- HLM route: apply_interaction_tests_HLM (src/Interaction.cpp:289-437).
"""
import numpy as np

NUMTOL = 1e-6


def robust(g, E, X, res, mask, scf_sv, n_analyzed, mac, rare_mac=1000.0, force_hc4=False, no_robust=False):
    """g [N] mean-imputed genotype (0 outside the analysis), X [N x C] orthonormal covariate basis, res [N x P] and
    scf_sv [P] as rg_s2_set_chr takes them.  Returns None (skip_int or near-singular) or (coef [P, 2], vcov [P, 2, 2])."""
    N, C = X.shape
    nk = n_analyzed - C
    iM = E * g                                                     # get_interaction_terms: raw G
    iM = iM - X @ (X.T @ iM)
    scf_i = np.linalg.norm(iM) / np.sqrt(nk)
    if scf_i < NUMTOL:
        return None
    iM = iM / scf_i
    G = g - X @ (X.T @ g)                                          # residualize_geno
    sf = np.linalg.norm(G) / np.sqrt(nk)
    G = G / sf
    H = np.stack([G, iM], axis=1)
    w, U = np.linalg.eigh(H.T @ H)
    if w.min() < NUMTOL:
        return None
    Z = U @ np.diag(1.0 / w) @ U.T
    hvec = ((H @ Z) * H).sum(axis=1)
    tau = Z @ H.T @ res
    e_sq = (res - H @ tau) ** 2 * mask
    P = res.shape[1]
    coef, vcov = np.zeros((P, 2)), np.zeros((P, 2, 2))
    neff = mask.sum(axis=0)
    for i in range(P):
        if no_robust:
            V = e_sq[:, i].sum() / (neff[i] - C - 2) * Z
        else:
            if force_hc4 and mac[i] <= rare_mac:
                hc = (1 - hvec) ** np.minimum(N * hvec / 2, 4)
            else:
                hc = (1 - hvec) ** 2
            V = Z @ (H.T * (e_sq[:, i] / hc)) @ H @ Z
        s = np.array([scf_sv[i] / sf, scf_sv[i] / scf_i])          # gscale, iscale
        coef[i] = tau[:, i] * s
        vcov[i] = V * np.outer(s, s)
    return coef, vcov


def _std_cols(M):
    """rescale_mat (src/Pheno.cpp:1887-1900): centre and scale over all rows."""
    n = M.shape[0]
    M = M - M.sum(axis=0) / n
    return M / (np.linalg.norm(M, axis=0) / np.sqrt(n - 1))


def hlm_design(E, X, blup):
    """V = (1, QR(E, E^2)) and X_hlm = (QR(covariates, E^2), blup) of HLM::prep_run for a continuous E."""
    V = np.column_stack([np.ones(len(E)), _std_cols(np.column_stack([E, E * E]))])
    Xh = np.column_stack([X, E * E, blup])
    return V, Xh


def hlm_fit(y, mask, Xh, V, gtol=1e-10):
    """Null HLM y = X a + e, e ~ N(0, exp(V b)) on the masked samples: b by BFGS on the profile likelihood (a by
    weighted least squares, HLM::get_alpha), started from HLM::get_beta_approx.  Returns b and its gradient."""
    from scipy.optimize import minimize
    m = mask.astype(float)
    n = m.sum()

    def alpha(b):
        dinv = np.exp(-V @ b) * m
        Xd = Xh.T * dinv
        return np.linalg.lstsq(Xd @ Xh, Xd @ y, rcond=None)[0], dinv

    def f(b):
        a, dinv = alpha(b)
        esq = (y - Xh @ a) ** 2
        val = 0.5 * np.sum(m * (V @ b) + esq * dinv) / n
        grad = V.T @ ((1 - esq * dinv) * m) / (2 * n)
        return val, grad

    b0 = np.zeros(V.shape[1])
    a, _ = alpha(b0)
    esq = ((y - Xh @ a) * m) ** 2
    b0 = np.linalg.lstsq(V.T @ (V * esq[:, None]), V.T @ ((esq - 1) * m), rcond=None)[0]
    r = minimize(f, b0, jac=True, method="BFGS", options={"gtol": gtol, "maxiter": 10000})
    return r.x, f(r.x)[1]


def hlm_state(y, mask, Xh, V, b):
    """store_null_est: Dinv_sqrt, Px (Xd eigenvectors / sqrt(eigenvalues)) and yres of one trait."""
    d = np.sqrt(np.exp(-V @ b) * mask)
    Xd = Xh * d[:, None]
    w, U = np.linalg.eigh(Xd.T @ Xd)
    Px = (Xd @ U) / np.sqrt(w)
    m = d * y
    return d, Px, m - Px @ (Px.T @ m)


def hlm_test(g, E, d, Px, yres):
    """apply_interaction_tests_HLM for one trait: None when Xres^T Xres is near-singular, else (coef [2], vcov [2, 2])."""
    m = np.stack([g, g * E], axis=1) * d[:, None]
    Xres = m - Px @ (Px.T @ m)
    w, U = np.linalg.eigh(Xres.T @ Xres)
    if w.min() < NUMTOL:
        return None
    Vm = U @ np.diag(1.0 / w) @ U.T
    return Vm @ (Xres.T @ yres), Vm
