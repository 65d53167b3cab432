"""Step-2 binary-trait score test with approximate Firth fallback (oracle only; test infrastructure).

Restates rgcgithub/regenie v4.1.2 so the oracle can be checked against the ONE golden output file the
reference ships (example/test_bin_out_firth_Y1.regenie, docs/docs/options.md:20-51):
  fit_null_logistic (Step-2 use)     src/Step1_Models.cpp:54-140
  Data::compute_res_bin              src/Data.cpp:2439-2455
  fit_approx_firth_null / fit_firth_nr   src/Step2_Models.cpp:899-983, 1267-1383
  fit_null_firth (cov_blup_offset)   src/Step2_Models.cpp:985-1060
  parseSnpfromBGEN stats + flip      src/Geno.cpp:2186-2413, 3077-3163
  check_sparse_G                     src/Geno.cpp:3165-3178
  compute_score_bt                   src/Step2_Models.cpp:470-556
  check_pval_snp / get_sumstats      src/Step2_Models.cpp:1988-2041
  fit_firth_logistic_snp_fast        src/Step2_Models.cpp:1158-1252
  fit_firth_pseudo / fit_firth (1 SNP)   src/Step2_Models.cpp:1527-1737
"""
import math

import numpy as np

from .prep import get_basis
from .step1_bt import NUMTOL_EPS, L1_RIDGE_EPS, fit_logistic, get_pvec, logist_dev
from .step2 import MIN_MAC, PROP_ZERO_THR, get_logp

NUMTOL = 1e-6
NUMTOL_FIRTH = 2.5e-4       # src/Regenie.hpp:224
MAXSTEP = 5                 # :339
MAXSTEP_NULL = 25           # :340
NITER_FIRTH = 250           # :336
NITER_FIRTH_NULL = 1000     # :337
NITER_LS = 25               # :338
NITER_MAX = 50              # :335


def null_logistic_offset(y, X, offset, mask):
    """fit_null_logistic in test mode: returns (beta, eta, p).  src/Step1_Models.cpp:79-86."""
    b0 = np.zeros(X.shape[1])
    for chk in (True, False):
        ok, b, eta, p = fit_logistic(y, X, offset, mask, b0.copy(), chk)
        if ok:
            return b, eta, p
    raise ValueError("null logistic regression did not converge")


def firth_nr(y, X, offset, mask, beta, maxstep, niter, tol, check_score_inc=True):
    """fit_firth_nr with all columns included, comp_lrt = False (null model).  :1267-1383."""
    m = mask
    score_old = 1e16
    n_inc = 0
    it = 0
    dev_new = 0.0
    while it < niter:
        it += 1
        eta = offset + X @ beta
        p = get_pvec(eta)
        dev_old = logist_dev(y, p, m)
        w = np.where(m, p * (1 - p), 1.0)
        XtW = X.T * np.sqrt(w)
        XtWX = XtW @ XtW.T
        sign, logdet = np.linalg.slogdet(XtWX)
        dev_old -= logdet
        h = (np.linalg.solve(XtWX, XtW) * XtW).sum(axis=0)
        mod_score = X.T @ np.where(m, y - p + h * (0.5 - p), 0.0)
        step = np.linalg.solve(XtWX, mod_score)
        smax = np.abs(mod_score).max()
        if smax < tol and it >= 2:
            break
        n_inc = n_inc + 1 if smax > score_old else 0
        if check_score_inc and n_inc > 25:
            return False, beta
        mx = np.abs(step).max() / maxstep
        if mx > 1:
            step = step / mx
        ok = False
        for ls in range(1, NITER_LS + 1):
            if ls > 1:
                step = step / 2
            bn = beta + step
            p2 = get_pvec(offset + X @ bn)
            dev_new = logist_dev(y, p2, m)
            w2 = np.where(m, p2 * (1 - p2), 1.0)
            XtW2 = X.T * np.sqrt(w2)
            dev_new -= np.linalg.slogdet(XtW2 @ XtW2.T)[1]
            if dev_new < dev_old:
                ok = True
                break
        if not ok:
            return False, beta
        beta = beta + step
        score_old = smax
    else:
        return False, beta
    return True, beta


def firth_pseudo_1snp(dev0, y, g, offset, mask, carriers, beta, niter, tol):
    """fit_firth_pseudo, single SNP (src/Step2_Models.cpp:1527-1641).  Returns (state, beta, se, lrt); state 0 converged,
    1 beta moved by more than 0.1 between iterations 14 and 15 or the iteration cap (:1582, :1633), 2 the inner step
    grew (:1595), 3 a zero weight p (1 - p) (:1616), 4 converged with LRT < 0 (:1636).

    State 3 cannot happen: get_pvec clamps eta to [-30, 30] and returns eps / (1 + eps) beyond it (eps = 10 DBL_EPSILON),
    so every p (1 - p) is at least about 2.2e-15 (and 1 - 1 / (exp(30) + 1) is 9.4e-14 below 1); masked-out samples
    have weight 1."""
    fast = carriers is not None and len(carriers) > 0
    if fast:
        p = get_pvec(offset + g * beta)
        dev_new = logist_dev(y, p, mask)
        dev_nc = dev_new - logist_dev(y[carriers], p[carriers], mask[carriers])
        gm = g[carriers]; yy = y[carriers]; off = offset[carriers]; mk = mask[carriers]
    else:
        gm = np.where(mask, g, 0.0); yy = y; off = offset; mk = mask
        dev_nc = 0.0
    gsq = gm * gm
    it = 0
    b14 = 0.0
    XtWX = 1.0
    dev_new = 0.0
    betanew = beta
    while it < niter:
        it += 1
        p = get_pvec(off + (g[carriers] if fast else g) * beta)
        dev_new = dev_nc + logist_dev(yy, p, mk)
        w = np.where(mk, p * (1 - p), 1.0)
        d = gsq * w
        XtWX = d.sum()
        dev_new -= math.log(XtWX)
        h = d / XtWX
        ystar = yy + h * (0.5 - p)
        score = (gm * (ystar - p)).sum()
        if abs(score) < tol and it >= 2:
            break
        if it == 14:
            b14 = beta
        if it == 15 and abs(beta - b14) > 0.1:
            return 1, beta, 0.0, 0.0
        nl = 0
        bdiff = 1e16
        while nl < 25:
            nl += 1
            step = score / XtWX
            bnew = abs(step)
            if bnew > bdiff:
                return 2, beta, 0.0, 0.0
            mx = bnew / 5.0
            betanew = beta + (step / mx if mx > 1 else step)
            p = get_pvec(off + (g[carriers] if fast else g) * betanew)
            score = (gm * (ystar - p)).sum()
            if abs(score) < tol:
                break
            w = np.where(mk, p * (1 - p), 1.0)
            if (w == 0).any():
                return 3, beta, 0.0, 0.0
            XtWX = (gsq * w).sum()
            beta = betanew
            bdiff = bnew
        else:
            nl += 1
        if nl > NITER_MAX:
            return 1, beta, 0.0, 0.0
        beta = betanew
    else:
        return 1, beta, 0.0, 0.0
    lrt = dev0 - dev_new
    if lrt < 0:
        return 4, beta, 0.0, lrt
    return 0, beta, math.sqrt(1 / XtWX), lrt


NR_CONVERGED, NR_NO_CONV, NR_LRT_NEG = 0, 1, 2     # outcomes of firth_nr_1snp (the reference returns false for both)


def firth_nr_1snp(dev0, y, g, offset, mask, carriers, beta, maxstep, niter, tol):
    """fit_firth, single SNP Newton-Raphson (src/Step2_Models.cpp:1644-1737).  Returns (outcome, beta, se, lrt, smin)
    with outcome NR_CONVERGED, NR_NO_CONV (iteration cap, :1728) or NR_LRT_NEG (converged with LRT < 0, :1731), and
    smin the smallest |modified score| the stopping test saw (from iteration 2): how far a fit that did not converge
    stayed from the tolerance."""
    fast = carriers is not None and len(carriers) > 0
    p = get_pvec(offset + g * beta)
    dev_old = logist_dev(y, p, mask)
    if fast:
        gm = g[carriers]; yy = y[carriers]; off = offset[carriers]; mk = mask[carriers]; gg = g[carriers]
        p = get_pvec(off + gg * beta)
        dev_nc = dev_old - logist_dev(yy, p, mk)
    else:
        gm = np.where(mask, g, 0.0); yy = y; off = offset; mk = mask; gg = g
        dev_nc = 0.0
    w = np.where(mk, p * (1 - p), 1.0)
    gsq = gm * gm
    d = gsq * w
    XtWX = d.sum()
    dev_old -= math.log(XtWX)
    it = 0
    dev_new = dev_old
    smin = math.inf
    while it < niter:
        it += 1
        h = d / XtWX
        score = (gm * (yy - p + h * (0.5 - p))).sum()
        if it >= 2:
            smin = min(smin, abs(score))
        if abs(score) < tol and it >= 2:
            break
        step = score / XtWX
        mx = abs(step) / maxstep
        if mx > 1:
            step /= mx
        ok = False
        for ls in range(1, NITER_LS + 1):
            if ls > 1:
                step /= 2
            bn = beta + step
            p = get_pvec(off + gg * bn)
            dev_new = dev_nc + logist_dev(yy, p, mk)
            w = np.where(mk, p * (1 - p), 1.0)
            d = gsq * w
            XtWX = d.sum()
            dev_new -= math.log(XtWX)
            if dev_new < dev_old:
                ok = True
                break
        if not ok:
            step += 1e-6
        beta += step
        dev_old = dev_new
    else:
        return NR_NO_CONV, beta, 0.0, 0.0, smin
    lrt = dev0 - dev_new
    if lrt < 0:
        return NR_LRT_NEG, beta, 0.0, lrt, smin
    return NR_CONVERGED, beta, math.sqrt(1 / XtWX), lrt, smin


class BtChrom:
    """Per-chromosome null state of one binary trait (compute_res_bin + fit_null_firth)."""

    def __init__(self, y_raw, X, blup, mask):
        loco = blup * mask
        self.beta0, eta, p = null_logistic_offset(y_raw, X, loco, mask)
        w = np.where(mask, p * (1 - p), 1.0)                       # get_wvec, src/Step1_Models.cpp:1760
        self.gamma_sqrt = np.sqrt(w)
        self.gamma_sqrt_mask = self.gamma_sqrt * mask
        self.Xg, _ = get_basis(self.gamma_sqrt_mask[:, None] * X)  # X_Gamma, :130-131
        self.yres = (y_raw - p) / self.gamma_sqrt * mask           # src/Data.cpp:2443-2445
        self.phat = p                                              # m_ests.Y_hat_p, src/Step1_Models.cpp:128
        # null approximate Firth: covariate effects become an offset (src/Step2_Models.cpp:899-983, 1014-1017)
        ok, bf = firth_nr(y_raw, X, blup, mask, self.beta0.copy(), MAXSTEP_NULL, NITER_FIRTH_NULL, 50 * NUMTOL)
        if not ok:
            raise ValueError("null Firth did not converge")
        self.cov_blup_offset = X @ bf + blup


# ------------------------------------------------------------------------------------------------ saddlepoint (SPA)
TOL_SPA = float(np.finfo(float).eps) ** 0.25        # src/Regenie.hpp:330
NITER_SPA = 1000                                    # :329
MAX_EXP_LIM = 708                                   # src/Step2_Models.hpp:30
NL_DBL_DMIN = 10.0 * np.finfo(float).tiny           # src/Regenie.hpp:229


def _norm_cdf(x):
    return 0.5 * math.erfc(-x / math.sqrt(2.0))


def chisq1_from_pvalue(pv):
    """quantile(complement(chi2_1, p)) = (Phi^-1(1 - p/2))^2, by Newton on the erfc tail (src/Regenie.cpp:1859-1873)."""
    target = math.log(pv)
    z = math.sqrt(max(-2.0 * math.log(pv) - math.log(max(-2.0 * math.log(pv), 1.0)), 0.0)) if pv < 0.5 else 0.5
    for _ in range(200):
        f = math.erfc(z / math.sqrt(2.0))
        if f <= 0.0:
            z *= 0.5
            continue
        d = math.log(f) - target
        dz = d / (-math.sqrt(2.0 / math.pi) * math.exp(-0.5 * z * z) / f)
        z -= dz
        if abs(dz) < 1e-14 * max(1.0, abs(z)):
            break
    return z * z


SPA_OK, SPA_LIMITS, SPA_NITER, SPA_K2_SEARCH, SPA_K2_ROOT, SPA_PTOT = 0, 1, 2, 3, 4, 5   # s2_spa_kernel's codes


def spa_test(stat, denum, gres, st, mask, nz, fast):
    """run_SPA_test_snp + solve_K1_snp + get_SPA_pvalue_snp (src/Step2_Models.cpp:2072-2294).
    gres: residualised genotype (length N); nz: g != 0 (the entries of Gsparse); fast = is_sparse.
    Returns (reason, chisq, logp, nan_tail); reason SPA_OK, or why the test failed: SPA_LIMITS s outside the limits
    of K' (:2101), SPA_NITER the root search hit NITER_SPA (:2191), SPA_K2_SEARCH K'' = 0 during the search (:2163),
    SPA_K2_ROOT K'' = 0 at the root (:2282), SPA_PTOT p1 + p2 > 1 or not a number (:2135); nan_tail: SPA_PTOT
    because a tail was NaN.

    A tail that is not a number.  w = sgn(r) sqrt(2 (r s - K(r))) at the root r of K'(r) = s.  Because K is convex
    with K(0) = 0, r s - K(r) = sup_t (t s - K(t)) >= 0 in exact arithmetic.  In floating point it goes negative in
    two ways.  (a) K(r) overflows: exp(r g / c) is inf for a sample with r g / c > 709.  K'' guards only the opposite
    sign (-r g / c > 708), so this happens when the root lies far out, e.g. when the carriers carry little weight
    and c = sqrt(G'WG) is small (firth_spa_cases.nan_candidates).  (b) Cancellation when s ~ 0: r s - K(r) ~ s^2 / 2
    is then below the rounding of K; both tails are then near 1/2, so this lands in SPA_PTOT as p1 + p2 > 1 does.
    Then w is NaN, and so are r = w + log(v / w) / w and the tail p-value.  The reference passes that r to
    boost::math::cdf(normal), whose default policy throws domain_error on a non-finite variate.  compute_tests_mt
    catches it and rethrows it as the run's error (src/Data.cpp:2537-2551), so the run ends.  So the reference never
    reaches `(pval1 + pval2) > 1` or get_logp(pv) with a NaN.  Its max(nl_dbl_dmin, NaN) = nl_dbl_dmin would report a
    "success" with the largest chi-square, and that path is unreachable.  A per-variant test cannot end the run, so
    here (as in s2_spa_kernel) both tails are computed with IEEE arithmetic: sqrt of a negative number is NaN, and
    x / 0 is +-inf.  A NaN tail makes p1 + p2 NaN, and `not (p1 + p2 <= 1)` reports it as a failed test with
    SPA_PTOT.  That is the TEST_FAIL row in place of the reference's abort, and never a p-value.  An infinite r gives
    the tail 0 or 1, as boost's cdf does."""
    cgf = SpaCgf(stat, denum, gres, st, mask, nz, fast)
    if not cgf.solvable():
        return SPA_LIMITS, 0.0, 0.0, False
    tval = -stat if stat >= 0 else stat
    ptot = 0.0
    for lam in (1, -1):
        reason, root = solve_k1(cgf, tval, lam)
        if reason != SPA_OK:
            return reason, 0.0, 0.0, False
        kval = cgf.K(lam * root)
        k2 = cgf.K2(lam * root)
        if k2 == 0:
            return SPA_K2_ROOT, 0.0, 0.0, False
        ptot += spa_tail(root, tval, kval, k2)
    if not ptot <= 1:
        return SPA_PTOT, 0.0, 0.0, math.isnan(ptot)
    pval = max(NL_DBL_DMIN, ptot)
    return SPA_OK, chisq1_from_pvalue(pval), -math.log10(pval), False


class SpaCgf:
    """The cumulant generating function K of the score and its derivatives K', K'' (compute_K*_snp,
    src/Step2_Models.cpp:2200-2272), over the masked samples, or over the non-zero genotypes plus a normal remainder
    when fast."""

    def __init__(self, stat, denum, gres, st, mask, nz, fast):
        self.stat, self.denum, self.fast = stat, denum, fast
        self.c = c = math.sqrt(denum)
        gmod = np.where(mask, gres / st.gamma_sqrt, 0.0)
        gmu = gmod * st.phat
        self.a = gmu.sum()
        sel = (mask & nz) if fast else mask
        self.gm, self.ph, self.gs = gmod[sel], st.phat[sel], st.gamma_sqrt[sel]
        if fast:
            self.b = denum - float((gres[sel] ** 2).sum())
            self.d = float(gmu[sel].sum())
        self.lim_lo = gmod[gmod < 0].sum() - self.a
        self.lim_hi = gmod[gmod > 0].sum() - self.a

    def solvable(self):
        """K'(t) = s has a finite root (:2099-2105)."""
        score_num = self.stat * self.c
        return not (score_num < self.lim_lo or score_num > self.lim_hi)

    def K(self, t):
        c, gm, ph = self.c, self.gm, self.ph
        with np.errstate(over="ignore"):
            v = np.log(1 - ph + ph * np.exp(t / c * gm)).sum()
        return v - t * self.d / c + t * t / 2 / self.denum * self.b if self.fast else v - t * self.a / c

    def K1(self, t):
        c, gm, ph = self.c, self.gm, self.ph
        with np.errstate(over="ignore"):
            v = ((gm * ph / c) / (ph + (1 - ph) * np.exp(-t / c * gm))).sum()
        return v - self.d / c + t / self.denum * self.b if self.fast else v - self.a / c

    def K2(self, t):
        c, gm, ph, gs = self.c, self.gm, self.ph, self.gs
        vexp = -t / c * gm
        if (vexp > MAX_EXP_LIM).any():
            return 0.0
        e = np.exp(vexp)
        with np.errstate(over="ignore"):                                           # e^2 = inf: the term is 0
            v = ((gm * gm * gs * gs / (c * c) * e) / (ph + (1 - ph) * e) ** 2).sum()
        return v + self.b / self.denum if self.fast else v


def solve_k1(cgf, tval, lam):
    """solve_K1_snp (src/Step2_Models.cpp:2146-2198): the root of lam K'(lam t) = tval by Newton steps, bisecting when a
    step leaves the bracket.  Returns (reason, root): SPA_OK, SPA_NITER or SPA_K2_SEARCH."""
    K1, K2 = cgf.K1, cgf.K2
    if tval >= 0:
        min_x, max_x = 0.0, float(np.finfo(float).max)
    else:
        min_x, max_x = -float(np.finfo(float).max), 0.0
    t_old = 0.0
    f_old = lam * K1(lam * t_old) - tval
    t_new = -1.0
    it = 0
    while True:
        it += 1
        if it > NITER_SPA:
            return SPA_NITER, 0.0
        hess = K2(lam * t_old)
        if hess == 0:
            return SPA_K2_SEARCH, 0.0
        t_new = t_old - f_old / hess
        f_new = lam * K1(lam * t_new) - tval
        if abs(f_new) < TOL_SPA:
            return SPA_OK, t_new
        if t_new and min_x < t_new < max_x:
            if f_new > 0:
                max_x = t_new
            else:
                min_x = t_new
        else:
            t_new = (min_x + max_x) / 2
            f_new = lam * K1(lam * t_new) - tval
            if f_new <= 0:
                min_x = t_new
            else:
                max_x = t_new
        t_old, f_old = t_new, f_new


def spa_tail(root, tval, kval, k2):
    """One tail of get_SPA_pvalue_snp (src/Step2_Models.cpp:2287-2295) in IEEE arithmetic: NaN when 2 (r s - K(r)) < 0
    or K(r) is not finite (see spa_test)."""
    with np.errstate(all="ignore"):
        wval = np.float64(math.copysign(1.0, root) if root != 0 else 0.0) * np.sqrt(np.float64(2 * (root * tval - kval)))
        vval = np.float64(root * math.sqrt(k2))
        if vval == 0:
            return 0.5
        rval = wval + np.log(vval / wval) / wval
    return float("nan") if math.isnan(rval) else _norm_cdf(float(rval))


def score_bt(g_raw, info_term, in_analysis, mask, y_raw, st: BtChrom, z_thr, n_samples, male=None, non_par=False,
             correction="firth", min_mac=None):
    """One variant, one trait.  g_raw: dosages with -3 = missing.  Returns dict or None if ignored.

    Beside the values, a tested variant (|stat| > z_thr) reports the branch its correction took.  SPA: spa_reason
    (SPA_OK or a failure code of spa_test) and spa_nan_tail (SPA_PTOT because a tail was NaN).  Firth: firth_state,
    the pseudo-Firth state 0-4 of firth_pseudo_1snp; nr, None when the pseudo-Firth converged (state 0), else the
    outcome of the Newton-Raphson fit (NR_CONVERGED, NR_NO_CONV, NR_LRT_NEG), and nr_min_score, the smallest
    |modified score| it reached; carriers_only, whether both fits ran over the carriers alone; and the fits' inputs
    gvec (G_res / Gamma^1/2) and offset (the null covariate + LOCO offset)."""
    ok = in_analysis & (g_raw != -3.0)
    ns1 = int(ok.sum())
    total = float(g_raw[ok].sum())
    okp = ok & mask
    ns = int(okp.sum())
    tot_p = float(g_raw[okp].sum())
    info_p = float(info_term[okp].sum())
    if non_par and male is not None:                          # see step2.variant_stats
        mval = np.where(ok, g_raw, 0.0) * 0.5 * (2 - male.astype(float))
        m1, mp = float(mval.sum()), float(mval[mask].sum())
        mac1 = min(m1, 2 * ns1 - int((ok & male).sum()) - m1)
        mac = min(mp, 2 * ns - int((okp & male).sum()) - mp)
    else:
        mac1 = min(total, 2 * ns1 - total)
        mac = min(tot_p, 2 * ns - tot_p)
    min_mac = MIN_MAC if min_mac is None else min_mac                              # --minMAC
    if mac1 < min_mac or mac < min_mac:
        return None
    af = tot_p / (2.0 * ns)
    info = 1.0 if af in (0.0, 1.0) else 1 - info_p / (2 * ns * af * (1 - af))     # src/Geno.cpp:3140
    mean = total / ns1
    flipped = mean > 1                                                             # flip_geno :3150-3163
    g = g_raw.copy()
    if flipped:
        g = np.where(g != -3.0, 2 - g, g)
        mean = 2 - mean
    g = np.where(g == -3.0, mean, g)
    g = np.where(in_analysis, g, 0.0)
    is_sparse = int(((g != 0) & in_analysis).sum()) <= n_samples * (1 - PROP_ZERO_THR)
    gw = g * st.gamma_sqrt_mask
    if is_sparse:
        xtwg = st.Xg.T @ gw
        den = gw @ gw - xtwg @ xtwg
    else:
        gres = gw - st.Xg @ (st.Xg.T @ gw)
        den = gres @ gres
    sq = math.sqrt(den)
    if sq < NUMTOL:
        return None
    stat = (gw @ st.yres if is_sparse else gres @ st.yres) / sq
    out = dict(af=af, info=info, n=ns, flipped=flipped, stat=stat, test_fail=False, is_sparse=is_sparse)
    if abs(stat) <= z_thr:
        se = 1 / sq
        out.update(beta=stat * se, se=se, chisq=stat * stat, logp=get_logp(stat * stat))
    elif correction == "spa":
        if is_sparse:
            gres = gw - st.Xg @ xtwg
        reason, chisq, logp, nan_tail = spa_test(stat, den, gres, st, mask, (g != 0), is_sparse)
        out.update(spa_reason=reason, spa_nan_tail=nan_tail)
        se0 = 1 / sq
        if reason != SPA_OK:
            out.update(beta=stat * se0, se=se0, chisq=float("nan"), logp=float("nan"), test_fail=True)
        else:                                                                      # check_pval_snp :2021-2029
            out.update(beta=math.copysign(1.0, stat) * math.sqrt(chisq) * se0, se=se0, chisq=chisq, logp=logp)
    else:
        if is_sparse:
            gres = gw - st.Xg @ xtwg
        gvec = gres / st.gamma_sqrt                                               # :2056
        carriers = None
        if is_sparse and mac < 50:
            carriers = np.nonzero(mask & in_analysis & (g > 1e-4))[0]
        off = st.cov_blup_offset
        p = get_pvec(off)
        dev0 = logist_dev(y_raw, p, mask)
        if carriers is not None and len(carriers) > 0:
            pc = get_pvec(off[carriers])
            wc = np.where(mask[carriers], pc * (1 - pc), 1.0)
            dev0 -= math.log(((gvec[carriers] ** 2) * wc).sum())
            niter_pseudo = NITER_FIRTH // 2
        else:
            wv = np.where(mask, p * (1 - p), 1.0)
            dev0 -= math.log(((np.where(mask, gvec, 0.0) ** 2) * wv).sum())
            niter_pseudo = min(NITER_FIRTH // 2, 50)
        state, b, se, lrt = firth_pseudo_1snp(dev0, y_raw, gvec, off, mask, carriers, 0.0, niter_pseudo, NUMTOL_FIRTH)
        out.update(firth_state=state, nr=None, carriers_only=carriers is not None and len(carriers) > 0, gvec=gvec,
                   offset=off)
        if state != 0:
            nr, b, se, lrt, smin = firth_nr_1snp(dev0, y_raw, gvec, off, mask, carriers, 0.0, MAXSTEP,
                                                 NITER_FIRTH // 2, NUMTOL_FIRTH)
            out.update(nr=nr, nr_min_score=smin)
            if nr != NR_CONVERGED:
                se0 = 1 / sq
                out.update(beta=stat * se0, se=se0, chisq=float("nan"), logp=float("nan"), test_fail=True)
                out["beta"] = -out["beta"] if flipped else out["beta"]
                return out
        out.update(beta=b, se=se, chisq=lrt, logp=get_logp(lrt))
    if flipped:
        out["beta"] = -out["beta"]
    return out
