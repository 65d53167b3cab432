"""numpy restatement of regenie's GxE interaction tests for binary traits, E kept as a covariate (gwas_condtl).

- design: get_interaction_terms + residualize_geno(force) (src/Interaction.cpp:44-92, src/Geno.cpp:3212-3240,
  src/Pheno.cpp:1836-1852): H = [G_res / scale_fac, resid(E o G) / scf_i];
- wald: apply_interaction_tests_bt (src/Interaction.cpp:441-678) with one interaction term: fit_logistic from beta = 0
  with offset_nullreg (check_hs_dev on, then off), model-based V = (H^T W H)^-1, HC3 on the robust route;
- fit_firth_nr: the penalised Newton fit of src/Step2_Models.cpp:1267-1383 with cols_incl and comp_lrt;
- firth: apply_interaction_tests_firth (src/Interaction.cpp:680-863, beg = 0): full, G-dropped and GxE-dropped fits.

The first fit_logistic attempt is oracle.step1_bt.fit_logistic from beta = 0.  The second one (check_hs_dev off)
continues from the state the first one left, as the reference's does: betavec is the last accepted point, while pivec and
etavec are those of the last evaluation (fit_logistic_continued).
"""
import numpy as np

from oracle.step1_bt import fit_logistic, get_pvec, logist_dev

NUMTOL = 1e-6
LOGIT_TOL = 1e-8                 # fit_logistic numtol (src/Step1_Models.hpp:79)
CHI2_P05 = 3.841458820694124     # chi2_1 statistic of p = 0.05: -log10 p > -log10 0.05 (src/Interaction.cpp:464)
NITER_FIRTH = 250                # src/Regenie.hpp:336
MAXSTEP = 5                      # :339
TOL_FIRTH = 2.5e-4               # :224
NITER_LS = 25                    # :338
ITER_MAX = 50                    # niter_max, :335


def design(g, E, X, n_analyzed):
    """g [N] minor-allele, mean-imputed genotype (0 outside the analysis), E [N] (0 outside), X [N x C] the covariate
    basis (spanning E and E^2).  Returns (H [N x 2], scale_fac, scf_i), or None when either sd is below numtol."""
    nk = n_analyzed - X.shape[1]
    iM = E * g
    iM = iM - X @ (X.T @ iM)
    scf_i = np.linalg.norm(iM) / np.sqrt(nk)
    if scf_i < NUMTOL:
        return None
    G = g - X @ (X.T @ g)
    sf = np.linalg.norm(G) / np.sqrt(nk)
    if sf < NUMTOL:
        return None
    return np.stack([G / sf, iM / scf_i], axis=1), sf, scf_i


def fit_logistic_continued(y, X, offset, mask, beta, eta, p, check_hs_dev, numtol=LOGIT_TOL):
    """fit_logistic (src/Step1_Models.cpp:156-222) entered with betavec = beta and pivec / etavec = p / eta, which need
    not belong to beta.  Returns (ok, beta, eta, p) like oracle.step1_bt.fit_logistic."""
    dev_old = logist_dev(y, p, mask)
    m = mask.astype(float)
    diff_dev = 0.0
    betanew = beta.copy()
    small_score = False
    it = 0
    while it < ITER_MAX:
        it += 1
        w = np.where(mask, p * (1 - p), 1.0)
        if (w == 0).any():
            return False, beta, eta, p
        XtW = X.T * (w * m)
        z = np.where(mask, eta - offset + (y - p) / w, 0.0)
        betanew = np.linalg.solve(XtW @ X, XtW @ z)
        for ls in range(NITER_LS):
            eta = offset + X @ betanew
            p = get_pvec(eta)
            dev_new = logist_dev(y, p, mask)
            if ((p[mask] > 0) & (p[mask] < 1)).all() and ((not check_hs_dev) or dev_new < dev_old):
                break
            betanew = (beta + betanew) / 2
        else:
            return False, beta, eta, p
        score = X.T @ np.where(mask, y - p, 0.0)
        smax = np.abs(score).max()
        if smax < numtol:
            break
        if (not small_score) and it < 20 and smax < 1:
            small_score = True
        if small_score and it > 20 and smax > 5:
            return False, beta, eta, p
        diff_dev = abs(dev_new - dev_old) / (0.1 + abs(dev_new))
        beta = betanew
        dev_old = dev_new
    else:
        it += 1
    if ((diff_dev == 0) or (diff_dev >= numtol)) and it > ITER_MAX:
        return False, beta, eta, p
    return True, betanew, eta, p


def wald(H, y, offset, mask, mac, rare_mac=1000.0, force_robust=False, no_robust=False):
    """One trait.  Returns (status, beta [2], V [2, 2]) on the scale of H: status 1 robust, 3 model-based, -1 near-singular
    H^T W H or a negative robust variance, -2 the logistic regression failed (beta and V are None unless 1 or 3)."""
    ok, b, eta, p = fit_logistic(y, H, offset, mask, np.zeros(2), True, numtol=LOGIT_TOL)
    if not ok:
        ok, b, eta, p = fit_logistic_continued(y, H, offset, mask, b.copy(), eta, p, False)
    if not ok:
        return -2, None, None
    w = np.where(mask, p * (1 - p), 0.0)
    WX = H * np.sqrt(w)[:, None]
    ev, U = np.linalg.eigh(WX.T @ WX)
    if ev.min() < NUMTOL:
        return -1, None, None
    V = U @ np.diag(1.0 / ev) @ U.T
    robust = force_robust or (not no_robust and mac > rare_mac and bool((b * b / np.diag(V) > CHI2_P05).any()))
    if robust:
        V = V @ hc3_meat(H, y, p, mask, V) @ V
    if np.diag(V).min() < 0:
        return -1, None, None
    return (1 if robust else 3), b, V


def hc3_meat(H, y, p, mask, V):
    """H^T diag(mask ((y - p) / (1 - h))^2) H, h = rowsum((W^1/2 H V) o W^1/2 H) (src/Interaction.cpp:472-474)."""
    WX = H * np.sqrt(np.where(mask, p * (1 - p), 0.0))[:, None]
    h = ((WX @ V) * WX).sum(axis=1)
    r2 = np.where(mask, (y - p) / (1 - h), 0.0) ** 2
    return H.T @ (H * r2[:, None])


def printed(beta, V, sf, scf_i, flipped):
    """(coef [2], vcov [2, 2]) of the printed rows: divided by scale_fac and scf_i, sign-corrected for a flip."""
    s = np.array([1.0 / sf, 1.0 / scf_i])
    return (-1.0 if flipped else 1.0) * beta * s, V * np.outer(s, s)


def penalised_dev(y, X, offset, mask, beta):
    """-2 log-lik - log det(X^T W X), W = p (1 - p) on the mask and 1 off it (get_wvec for Firth)."""
    p = get_pvec(offset + X @ beta)
    w = np.where(mask, p * (1 - p), 1.0)
    XtW = X.T * np.sqrt(w)
    return logist_dev(y, p, mask) - np.linalg.slogdet(XtW @ XtW.T)[1]


def fit_firth_nr(y, X, offset, mask, beta, cols_incl, comp_lrt, maxstep=MAXSTEP, niter=NITER_FIRTH, tol=TOL_FIRTH,
                 check_score_inc=True):
    """fit_firth_nr: the first cols_incl columns are free, the other coefficients stay at their (zero) start.
    Returns (ok, beta, dev, dev0, se); dev0 and se only with comp_lrt."""
    nc = X.shape[1]
    beta = np.array(beta, dtype=float)
    it, n_inc, score_old, dev_new, dev0 = 0, 0, 1e16, 0.0, None
    Ainv = None
    while it < niter:
        it += 1
        p = get_pvec(offset + X @ beta)
        w = np.where(mask, p * (1 - p), 1.0)
        XtW = X.T * np.sqrt(w)
        A = XtW @ XtW.T
        dev_old = logist_dev(y, p, mask) - np.linalg.slogdet(A)[1]
        if comp_lrt and it == 1:
            dev0 = dev_old
        Ainv = np.linalg.inv(A)
        h = ((Ainv @ XtW) * XtW).sum(axis=0)
        u = np.where(mask, y - p + h * (0.5 - p), 0.0)
        mod = X[:, :cols_incl].T @ u
        step = np.linalg.solve(A[:cols_incl, :cols_incl], mod)
        smax = np.abs(mod).max()
        if smax < tol and it >= 2:
            break
        if not comp_lrt:
            n_inc = n_inc + 1 if smax > score_old else 0
            if check_score_inc and n_inc > 25:
                return False, beta, None, None, None
        mx = np.abs(step).max() / maxstep
        if mx > 1:
            step = step / mx
        for ls in range(1, NITER_LS + 1):
            if ls > 1:
                step = step / 2
            bnew = np.zeros(nc)
            bnew[:cols_incl] = beta[:cols_incl] + step
            dev_new = penalised_dev(y, X, offset, mask, bnew)
            if dev_new < dev_old:
                break
        else:
            if not comp_lrt:
                return False, beta, None, None, None
            step[0] += 1e-6
        beta[:cols_incl] += step
        score_old = smax
    else:
        return False, beta, None, None, None
    if comp_lrt:
        if dev0 - dev_new < 0:
            return False, beta, None, None, None
        return True, beta, dev_new, dev0, np.sqrt(np.diag(Ainv))
    return True, beta, dev_new, None, None


def firth(H, y, offset, mask):
    """apply_interaction_tests_firth for one pair: (status, beta [2], se [2], lrt [3] = (2DF, SNP, SNPxVAR)) on the scale
    of H; status 0 = rows, 1 / 2 / 3 = the full / G-dropped / GxE-dropped fit failed, 4 = a negative LRT."""
    ok, b, dev, dev0, se = fit_firth_nr(y, H, offset, mask, np.zeros(2), 2, True)
    if not ok:
        return 1, None, None, None
    ok, _, dev_s, _, _ = fit_firth_nr(y, H[:, ::-1], offset, mask, np.array([b[1], 0.0]), 1, False)   # G last
    if not ok:
        return 2, None, None, None
    lrt_g = dev_s - dev
    if lrt_g < 0:
        return 4, None, None, None
    ok, _, dev_s, _, _ = fit_firth_nr(y, H, offset, mask, np.array([b[0], 0.0]), 1, False)
    if not ok:
        return 3, None, None, None
    lrt_i = dev_s - dev
    if lrt_i < 0:
        return 4, None, None, None
    return 0, b, se, np.array([dev0 - dev, lrt_g, lrt_i])
