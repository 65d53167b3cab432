"""Constructed binary-trait blocks whose Firth and SPA fits leave the converged path (shared by the CPU oracle test and
the GPU branch test, which must see the same inputs).

Two traits: one with a prevalence of 0.5 %, one with 50 %.  Some samples carry LOCO offsets of +-34 or +-50 on the side
of their phenotype, past the |eta| = 30 clamp of get_pvec, and twelve more +-24.  The first 128 rows mix single- and
two-carrier variants, rare variants whose carriers are all cases or all controls of a trait, carriers among the clamped
samples, rare variants with missing calls (mean-imputed, so counted as carriers), common variants with no effect (small
LRTs, the smallest about 1.6e-3; no converged LRT in the block is negative, the smallest is about 1e-4) and common
ones with large effects.  Then come rows picked from two candidate streams by the oracle on the CPU: carriers-only fits whose Newton-Raphson
fallback stops at the iteration cap with |score| at least 2.7 times the tolerance (NR_KEEP), and variants whose second
SPA tail is NaN because K(r) overflows, with r g / c above 900 for a carrier (NAN_KEEP).  Odd rows are coded on the
major allele, so they are flipped.
"""
import numpy as np

from oracle import step2_bt

N = 2000
P = 2
C = 3
MIN_MAC = 1.0          # single carriers are tested
SEED = 20261018
# the draws of nr_candidates / nan_candidates that the oracle sends down the branch each stream is for
NR_KEEP = (124, 172, 174, 302, 714, 718)
NAN_KEEP = (444, 828, 1041, 1092, 1134, 1344, 1560, 1605)
BS = 128 + len(NR_KEEP) + len(NAN_KEEP)


def problem(seed=SEED):
    rng = np.random.default_rng(seed)
    ia = np.ones(N, dtype=bool)
    ia[rng.choice(N, N // 100, replace=False)] = False
    cov = rng.standard_normal((N, C - 1))
    X = np.hstack([np.ones((N, 1)), cov]) * ia[:, None]
    mask = ia[:, None] & (rng.random((N, P)) > 0.03)
    Y = np.zeros((N, P))
    live0 = np.nonzero(mask[:, 0])[0]
    Y[rng.choice(live0, int(round(0.005 * len(live0))), replace=False), 0] = 1.0        # 0.5 % cases
    Y[:, 1] = (rng.random(N) < 1 / (1 + np.exp(-0.5 * cov[:, 0]))) & mask[:, 1]           # ~50 % cases
    blup = 0.3 * rng.standard_normal((N, P))
    far = rng.choice(np.nonzero(ia)[0], 40, replace=False)                                # |eta| > 30
    depth = np.where(np.arange(40) < 20, 34.0, 50.0)[:, None]
    blup[far] = np.where(Y[far] == 1, depth, -depth)                                     # on the side of y
    rng2 = np.random.default_rng(seed + 1)                                               # the rows chosen by draw
    mid = rng2.choice(np.setdiff1d(np.nonzero(ia)[0], far), 12, replace=False)           # |eta| ~ 24: w ~ 4e-11
    blup[mid] = np.where(Y[mid] == 1, 24.0, -24.0)
    blup *= mask
    sts = [step2_bt.BtChrom(Y[:, j], X, blup[:, j], mask[:, j]) for j in range(P)]
    g = _block(rng, rng2, ia, mask, Y, far, mid)
    return dict(N=N, P=P, C=C, ia=ia, X=X, mask=mask, Y=Y, blup=blup, sts=sts, far=far, mid=mid, g=g,
                n_an=int(ia.sum()))


def _block(rng, rng2, ia, mask, Y, far, mid):
    """Hard calls [BS, N] (ALT allele counts, 3 = missing) of the rows described in the module docstring."""
    live = np.nonzero(ia)[0]
    g = np.zeros((BS, N), dtype=np.uint8)
    cases = [np.nonzero((Y[:, j] == 1) & mask[:, j])[0] for j in range(P)]
    ctrls = [np.nonzero((Y[:, j] == 0) & mask[:, j])[0] for j in range(P)]

    def put(r, idx, hom_frac=0.2):
        g[r, idx] = np.where(rng.random(len(idx)) < hom_frac, 2, 1)

    for r in range(0, 8):                                              # one carrier: a case, a control, anyone
        pool = (cases[r % 2], ctrls[r % 2], live)[r % 3]
        put(r, rng.choice(pool, 1), hom_frac=0.5)
    for r in range(8, 16):                                             # two carriers
        pool = (cases[r % 2], ctrls[r % 2], live)[r % 3]
        put(r, rng.choice(pool, 2, replace=False))
    for r in range(16, 28):                                            # all carriers are cases of one trait
        j = r % 2
        put(r, rng.choice(cases[j], min(len(cases[j]), 3 + r % 7), replace=False))
    for r in range(28, 40):                                            # all carriers are controls of one trait
        put(r, rng.choice(ctrls[r % 2], 3 + r % 9, replace=False))
    for r in range(40, 44):                                            # one carrier at |eta| = 50: G'WG ~ 1e-14, ignored
        put(r, far[20 + 5 * (r - 40):21 + 5 * (r - 40)], hom_frac=0.5)
    for r in range(44, 48):                                            # carriers among the clamped samples
        k = 2 + r % 5
        put(r, np.concatenate([rng.choice(far, k, replace=False), rng.choice(live, r % 3, replace=False)]))
    for r in range(48, 60):                                            # rare, with missing calls (mean > 1e-4)
        put(r, rng.choice(live, 4 + r % 6, replace=False))
        g[r, rng.choice(live, 2 + r % 5, replace=False)] = 3
    for r in range(60, 76):                                            # rare, a few cases among the carriers
        j = r % 2
        idx = np.concatenate([rng.choice(cases[j], 1 + r % 3, replace=False),
                              rng.choice(ctrls[j], 2 + r % 11, replace=False)])
        put(r, idx)
    for r in range(76, 96):                                            # common, no effect: small LRTs
        g[r] = rng.binomial(2, rng.uniform(0.05, 0.5), size=N)
    for r in range(96, 108):                                           # common, large effect on a trait
        j = r % 2
        pr = np.where(Y[:, j] == 1, 0.6, 0.1)
        g[r] = rng.binomial(2, pr)
    for r in range(108, 116):                                          # MAC just under / over 50, sparse
        put(r, rng.choice(live, 20 + 2 * (r - 108), replace=False))
    for r in range(116, 128):                                          # rare case-enriched with a missing call
        j = r % 2
        put(r, np.concatenate([rng.choice(cases[j], min(len(cases[j]), 2 + r % 4), replace=False),
                               rng.choice(ctrls[j], r % 3, replace=False)]))
        g[r, rng.choice(live, 1 + r % 3, replace=False)] = 3
    g[128:] = np.concatenate([nr_candidates(rng2, mask, Y, N_NR_DRAWS)[list(NR_KEEP)],
                              nan_candidates(rng2, ia, far, mid, N_NAN_DRAWS)[list(NAN_KEEP)]])
    g[~ia[None, :].repeat(BS, 0)] = np.where(rng.random(((~ia).sum() * BS,)) < 0.5, 1, 0)
    # half of the rows coded on the major allele: the kernels flip them back
    flip = np.arange(BS) % 2 == 1
    g[flip] = np.where(g[flip] == 3, 3, 2 - np.minimum(g[flip], 2))
    return g


def nr_candidates(rng2, mask, Y, n):
    """n candidate rows: two or three carriers, all controls of the 0.5 % trait.  The Newton-Raphson step
    score / sum g^2 w leaves out the curvature of the Firth penalty, so on some of them the fit oscillates about its
    root and |score| is still above the tolerance after 125 iterations."""
    ctrl0 = np.nonzero((Y[:, 0] == 0) & mask[:, 0])[0]
    out = np.zeros((n, N), dtype=np.uint8)
    for k in range(n):
        idx = rng2.choice(ctrl0, 2 + k % 2, replace=False)
        out[k, idx] = np.where(rng2.random(len(idx)) < 0.2, 2, 1)
    return out


def nan_candidates(rng2, ia, far, mid, n):
    """n candidate rows: one to four carriers among the samples at |eta| >= 24, and on every third row one more
    carrier anywhere.  With so little weight on the carriers c = sqrt(G'WG) is small, the root of the second tail lies
    far out, and t g / c passes 709 for a carrier: K(r) = inf."""
    pool = np.concatenate([mid, far])
    live = np.nonzero(ia)[0]
    out = np.zeros((n, N), dtype=np.uint8)
    for k in range(n):
        idx = rng2.choice(pool, 1 + k % 4, replace=False)
        out[k, idx] = rng2.integers(1, 3, len(idx))
        if k % 3 == 0:
            out[k, rng2.choice(live, 1)] = 1
    return out


N_NR_DRAWS, N_NAN_DRAWS = 1200, 1800


def dosage(g_row):
    """Oracle dosage of one hard-call row: ALT allele count, -3 = missing."""
    return np.where(g_row == 3, -3.0, g_row.astype(np.float64))


def oracle_rows(pb, z_thr=0.0):
    """score_bt with Firth and with SPA for every (variant, trait) of the block: {(i, j): (firth, spa)} over the
    pairs that are not ignored."""
    out = {}
    for i in range(BS):
        gd = dosage(pb["g"][i])
        for j in range(P):
            args = (gd, np.zeros(N), pb["ia"], pb["mask"][:, j], pb["Y"][:, j], pb["sts"][j], z_thr, N)
            rf = step2_bt.score_bt(*args, min_mac=MIN_MAC)
            if rf is None:
                continue
            rs = step2_bt.score_bt(*args, correction="spa", min_mac=MIN_MAC)
            out[(i, j)] = (rf, rs)
    return out


def branch_counts(rows):
    """Counts of each Firth pseudo state, Newton-Raphson outcome and SPA reason among rows (oracle_rows)."""
    c = dict(pseudo=np.zeros(5, int), nr=np.zeros(3, int), spa=np.zeros(6, int), carriers=0, nan_tail=0)
    for rf, rs in rows.values():
        if "firth_state" in rf:
            c["pseudo"][rf["firth_state"]] += 1
            if rf["nr"] is not None:
                c["nr"][rf["nr"]] += 1
            c["carriers"] += rf["carriers_only"]
        if "spa_reason" in rs:
            c["spa"][rs["spa_reason"]] += 1
            c["nan_tail"] += rs["spa_nan_tail"]
    return c


def check_floors(c):
    """The branch counts both the CPU test of the oracle and the GPU test assert on this block."""
    assert c["pseudo"][0] >= 150 and c["pseudo"][1] >= 10 and c["pseudo"][2] >= 40, c
    assert c["pseudo"][3] == 0, c
    assert c["nr"][step2_bt.NR_CONVERGED] >= 40 and c["nr"][step2_bt.NR_NO_CONV] >= len(NR_KEEP), c
    assert c["carriers"] >= 150, c
    for reason, least in ((step2_bt.SPA_OK, 120), (step2_bt.SPA_K2_SEARCH, 3), (step2_bt.SPA_K2_ROOT, 8),
                          (step2_bt.SPA_PTOT, 60)):
        assert c["spa"][reason] >= least, (reason, c)
    assert c["nan_tail"] >= len(NAN_KEEP), c
