"""The branch reports of the Firth and SPA oracle (oracle/step2_bt.py), checked from first principles on the
constructed block of firth_spa_cases, the same inputs the GPU branch test feeds to s2_firth_kernel and s2_spa_kernel.

  * A converged Firth fit maximises the one-parameter penalised log-likelihood
        f(b) = l(b) + 1/2 log sum_S g^2 w(b),   eta = offset + g b,
    over all masked samples, or, carriers-only, over the carriers with the non-carriers held at b = 0; and its
    LRT is 2 (f(b_hat) - f(0)).
  * K' and K'' of the SPA cumulant generating function are the central differences of K and K', and the root of the
    search solves K'(t) = s (brentq).
  * Every branch that the GPU test asserts a count for is hit here, and the NaN edge of a tail is decided: a tail
    whose 2 (r s - K(r)) is negative or not finite is NaN, and p1 + p2 = NaN fails the test (SPA_PTOT).  The block
    holds variants whose K(r) overflows, so the GPU test checks the kernel's side of that decision too.
"""
import math

import numpy as np
import pytest
from scipy import optimize

import firth_spa_cases as fc
from oracle import step2_bt
from oracle.step1_bt import get_pvec


@pytest.fixture(scope="module")
def block():
    pb = fc.problem()
    return pb, fc.oracle_rows(pb)


def test_branches_hit(block):
    """The counts the GPU test asserts.  Pseudo state 3 (w == 0) cannot happen (get_pvec clamps eta).  The rows picked
    for the Newton-Raphson cap and the NaN tail sit there with a margin that rounding cannot take away: |score| stays
    above 2.5 times the tolerance, and r g / c passes 709 (where exp overflows) by more than 25 %."""
    pb, rows = block
    fc.check_floors(fc.branch_counts(rows))
    for i in range(128, 128 + len(fc.NR_KEEP)):
        rf = rows[(i, 0)][0]
        assert rf["nr"] == step2_bt.NR_NO_CONV and rf["nr_min_score"] > 2.5 * step2_bt.NUMTOL_FIRTH, (i, rf["nr"])
    n_nan = 0
    for (i, j), (_, rs) in sorted(rows.items()):
        if not rs["spa_nan_tail"]:
            continue
        assert i >= 128 + len(fc.NR_KEEP)
        cgf = _cgf(fc.dosage(pb["g"][i]), pb, j, pb["sts"][j], rs)
        tval = -abs(rs["stat"])
        x = []
        for lam in (1, -1):
            reason, root = step2_bt.solve_k1(cgf, tval, lam)
            assert reason == step2_bt.SPA_OK and cgf.K2(lam * root) > 0
            x.append(float(np.max(lam * root / cgf.c * cgf.gm)))
            assert (x[-1] > 709.79) == math.isinf(cgf.K(lam * root))
        assert max(x) > 1.25 * 709.79, (i, j, x)
        n_nan += 1
    assert n_nan >= len(fc.NAN_KEEP)


def _fits(block, carriers_only):
    pb, rows = block
    out = []
    for (i, j), (rf, _) in sorted(rows.items()):
        if "firth_state" not in rf or rf["test_fail"] or rf["carriers_only"] != carriers_only:
            continue
        out.append((i, j, rf))
    return out


@pytest.mark.parametrize("carriers_only", [False, True])
def test_firth_maximises_penalised_likelihood(block, carriers_only):
    pb, rows = block
    fits = _fits(block, carriers_only)
    assert len(fits) >= 40
    n_nr = 0
    for i, j, rf in fits:
        mask, y = pb["mask"][:, j], pb["Y"][:, j]
        g, off = rf["gvec"], rf["offset"]
        if carriers_only:                                  # score_bt: carriers after the flip and the imputation
            gi = fc.dosage(pb["g"][i])
            mean = gi[pb["ia"] & (gi != -3)].mean()
            gi = np.where(gi == -3, 2 - mean if rf["flipped"] else mean, np.where(rf["flipped"], 2 - gi, gi))
            S = mask & pb["ia"] & (gi > 1e-4)
        else:
            S = mask.copy()
        ll0 = np.where(y == 0, np.log(1 - get_pvec(off)), np.log(get_pvec(off)))

        def f(b):
            p = get_pvec(off + g * b)
            ll = np.where(S, np.where(y == 0, np.log(1 - p), np.log(p)), ll0)[mask].sum()
            return ll + 0.5 * math.log((g[S] ** 2 * (p * (1 - p))[S]).sum())

        b_hat = rf["beta"] * (-1 if rf["flipped"] else 1)
        info = (g[S] ** 2 * (lambda p: p * (1 - p))(get_pvec(off + g * b_hat))[S]).sum()
        half = 5.0 / math.sqrt(info)
        r = optimize.minimize_scalar(lambda b: -f(b), bounds=(b_hat - half, b_hat + half), method="bounded",
                                     options=dict(xatol=1e-10))
        # the fits stop at |modified score| < 2.5e-4: b_hat is within about tol / I of the maximum
        assert abs(r.x - b_hat) <= 4 * step2_bt.NUMTOL_FIRTH / info + 1e-7, (i, j, r.x, b_hat, info)
        assert f(b_hat) >= -r.fun - 1e-7 * max(1.0, abs(r.fun)), (i, j)
        lrt = 2 * (f(b_hat) - f(0.0))
        assert abs(rf["chisq"] - lrt) <= 1e-9 * max(1.0, abs(lrt)), (i, j, rf["chisq"], lrt)
        n_nr += rf["nr"] is not None
    assert n_nr >= (10 if carriers_only else 0)            # the Newton-Raphson fallback converged on these


def test_spa_cumulants_and_root(block):
    pb, rows = block
    n = 0
    for (i, j), (_, rs) in sorted(rows.items()):
        if rs.get("spa_reason") != step2_bt.SPA_OK or n >= 60:
            continue
        st = pb["sts"][j]
        gd = fc.dosage(pb["g"][i])
        cgf = _cgf(gd, pb, j, st, rs)
        s = rs["stat"]
        tval = -abs(s)
        for lam in (1, -1):
            reason, root = step2_bt.solve_k1(cgf, tval, lam)
            assert reason == step2_bt.SPA_OK
            assert abs(lam * cgf.K1(lam * root) - tval) < step2_bt.TOL_SPA
            lo, hi = (root * 2 - 1, 0.0) if root < 0 else (0.0, root * 2 + 1)
            r_ref = optimize.brentq(lambda t: lam * cgf.K1(lam * t) - tval, lo, hi, xtol=1e-14)
            k2 = cgf.K2(lam * root)
            assert abs(root - r_ref) <= 2 * step2_bt.TOL_SPA / k2 + 1e-12, (i, j, root, r_ref)
            for t in (lam * root, 0.5 * lam * root, 0.0):
                h = 1e-4 * max(1.0, abs(t))
                d1 = (cgf.K(t + h) - cgf.K(t - h)) / (2 * h)
                d2 = (cgf.K1(t + h) - cgf.K1(t - h)) / (2 * h)
                assert abs(d1 - cgf.K1(t)) <= 1e-6 * max(1.0, abs(d1)), (i, j, t, d1, cgf.K1(t))
                assert abs(d2 - cgf.K2(t)) <= 1e-5 * max(1e-3, abs(d2)), (i, j, t, d2, cgf.K2(t))
        n += 1
    assert n == 60


def _cgf(gd, pb, j, st, rs):
    """SpaCgf of one selection, rebuilt the way score_bt builds it."""
    ia, mask = pb["ia"], pb["mask"][:, j]
    ok = ia & (gd != -3)
    mean = gd[ok].sum() / ok.sum()
    g = gd.copy()
    if rs["flipped"]:
        g = np.where(g != -3, 2 - g, g)
        mean = 2 - mean
    g = np.where(g == -3, mean, g)
    g = np.where(ia, g, 0.0)
    gw = g * st.gamma_sqrt_mask
    gres = gw - st.Xg @ (st.Xg.T @ gw)
    den = (gw @ gw - (st.Xg.T @ gw) @ (st.Xg.T @ gw)) if rs["is_sparse"] else gres @ gres
    return step2_bt.SpaCgf(rs["stat"], den, gres, st, mask, g != 0, rs["is_sparse"])


def test_spa_tail_nan_edge():
    """get_SPA_pvalue_snp in IEEE arithmetic: a negative or non-finite 2 (r s - K(r)) makes the tail NaN (the reference
    throws in boost's cdf there and ends the run); NaN tails fail the test through `not (p1 + p2 <= 1)`; a zero w with a
    non-zero v gives an infinite r and a tail of 0 or 1; r = 0 gives 1/2."""
    assert math.isnan(step2_bt.spa_tail(-2.0, -3.0, 6.5, 1.0))                 # r s - K = -0.5
    assert math.isnan(step2_bt.spa_tail(-2.0, -3.0, math.inf, 1.0))            # K(r) overflowed
    assert step2_bt.spa_tail(0.0, -3.0, 0.0, 1.0) == 0.5
    assert step2_bt.spa_tail(-2.0, -3.0, 6.0, 1.0) in (0.0, 1.0)               # w = 0, v != 0
    p = step2_bt.spa_tail(-2.0, -3.0, 3.0, 1.5)
    w = -math.sqrt(6.0)
    v = -2.0 * math.sqrt(1.5)
    assert p == pytest.approx(0.5 * math.erfc(-(w + math.log(v / w) / w) / math.sqrt(2)), rel=1e-15)
    ptot = step2_bt.spa_tail(-2.0, -3.0, 6.5, 1.0) + 0.3
    assert not ptot <= 1                                                       # the SPA_PTOT test of spa_test
