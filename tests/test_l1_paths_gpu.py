"""Level 1, the LOCO assembly and the LOOCV route at the shapes that select their chunking and tiling, each against the
numpy oracle and against plain long-double references.

Level 1 picks its work split from the shape of the input:
  * sample chunks (l1_setup_chunks): len = round_up(max(2048, ceil(Npad / (max_chunks - K + 1))), 128) samples with
    max_chunks = max(K, 2^30 / (8 nC^2)), so a fold spans several chunks once it is longer than 2048 samples, and the
    1 GiB cap on the chunk partials sets the length once nC is large (nC = 2560: max_chunks = 20);
  * l1_pred_sums_kernel stages beta 256 columns at a time, with R1 * 256 doubles of dynamic shared memory;
  * l1_assemble_kernel, which also assembles the dense level-0 route's systems, keeps one partial per fold (K <= 16);
  * l0_loocv_pred_kernel loops over tiles of 8 phenotypes; the LOOCV fill kernels put the sample axis on grid.x.
Level 1 is fed straight through rg_l0_load_W with a synthetic W shaped like level 0's output: every case asserts
through the "l1_dims" / "l1_chunks" hooks which split ran.  The synthetic W holds multiples of 2^-8 below 8 in
magnitude and y multiples of 2^-10 below 8, so W^T W and W^T y are exact in FP64 in any summation order (products
below 2^22 units of 2^-16 and 2^24 units of 2^-18, sums over at most 60 000 samples below 2^40 units): the Gram and
right-hand-side partials of every chunk, their fold sums and the held-out differences the kernels form are exact, and
only the ridge shift adds a rounding to the systems.  W beta is exact in long double (11 + 53 significant bits): the
long-double references below are exact up to their own 2^-64 roundings.
"""
import numpy as np
import pytest

import helpers
from oracle import prep, step1, step1_bt
from regenie_b200 import capi, hostprep

pytestmark = pytest.mark.gpu
U = 2.0 ** -53              # unit round-off of FP64
LD = np.longdouble
NV = 3 * 8 + 2              # l1_sums row: kMaxRidge = 8 triples (Sx, Sx2, Sxy), then Sy, Sy2


def rel(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def gamma(n):
    return n * U / (1 - n * U)


def round_up(x, m):
    return (x + m - 1) // m * m


def ld_mm(A, Bm, rows=2000):
    """A @ Bm in long double, a few rows of A at a time."""
    Bl = Bm.astype(LD)
    return np.concatenate([A[r:r + rows].astype(LD) @ Bl for r in range(0, A.shape[0], rows)], axis=0)


def ld_tmv(A, v, rows=2000):
    """A^T v in long double, a few rows of A at a time."""
    return sum(A[r:r + rows].astype(LD).T @ v[r:r + rows].astype(LD) for r in range(0, A.shape[0], rows))


# ------------------------------------------------------------------------------------------------ synthetic level 1
def synth_W(N, nblocks, R, mask, rng):
    """W the way level 0 shapes it: per block R nearly collinear columns (one latent signal plus noise), each column
    standardised over the masked samples and zero on the others, rounded to a multiple of 2^-8."""
    m = mask.astype(bool)
    W = np.zeros((N, nblocks * R))
    for b in range(nblocks):
        cols = rng.standard_normal(N)[:, None] + 0.3 * rng.standard_normal((N, R))
        mu, sd = cols[m].mean(axis=0), cols[m].std(axis=0, ddof=1)
        cols = np.where(m[:, None], (cols - mu) / sd, 0.0)
        W[:, b * R:(b + 1) * R] = np.clip(np.round(cols * 256), -2000, 2000) / 256
    return W


class L1Case:
    """A Step-1 handle whose W was loaded directly (no level-0 run), with its W, y and tau grid."""

    def __init__(self, N, nblocks, R=5, P=2, R1=5, K=5, loocv=False, seed=0, chrs=None, bt=False, fold_sizes=None):
        rng = np.random.default_rng(seed)
        mask = (rng.random((N, P)) > 0.02).astype(np.uint8, order="F")
        self.W = [synth_W(N, nblocks, R, mask[:, p], rng) for p in range(P)]
        sig = np.stack([self.W[p][:, ::R].sum(axis=1) for p in range(P)], axis=1)
        X, Y, _, in_an, _ = hostprep.prepare_qt(0.05 * sig + rng.standard_normal((N, P)), np.zeros((N, 0)))
        Y = np.clip(np.round(Y * 1024), -8000, 8000) / 1024            # on the 2^-10 grid (module docstring)
        self.X, self.Y, self.mask = X, np.asfortranarray(Y * mask), mask
        self.neff = mask.sum(axis=0).astype(float)
        self.N, self.P, self.R, self.R1, self.B = N, P, R, R1, nblocks * R
        self.loocv = loocv
        self.fold_sizes = (np.array([N]) if loocv else
                           np.asarray(fold_sizes if fold_sizes is not None else hostprep.fold_sizes(N, K), dtype=np.int64))
        self.K = len(self.fold_sizes)
        self.chrs = list(chrs) if chrs is not None else [1 + b * 3 // nblocks for b in range(nblocks)]
        self.tau = self.B * (1 - hostprep.ridge_grid(R1)) / hostprep.ridge_grid(R1)
        if bt:
            self.y_raw = ((self.Y + 0.3 * rng.standard_normal((N, P)) > 0.4) * mask).astype(float)
            self.off = np.stack([step1_bt.null_offset(self.y_raw[:, p], X, mask[:, p].astype(bool)) for p in range(P)],
                                axis=1)
            self.tau = self.tau * 3 / np.pi ** 2
        self.st = self.handle()

    def handle(self, R1=None):
        st = capi.Step1(self.X, self.Y, self.mask, np.ones(self.N, np.uint8), self.fold_sizes, np.ones(self.R),
                        self.neff, self.N, 1, self.B // self.R, n_ridge_l1=R1 or self.R1, loocv=self.loocv)
        for p in range(self.P):
            for b in range(self.B // self.R):
                st.load_W(b, p, self.W[p][:, b * self.R:(b + 1) * self.R])
        return st

    def fit(self, st=None, tau=None):
        st = st or self.st
        cs, best = st.l1_fit(np.tile(self.tau if tau is None else tau, (self.P, 1)))
        return cs, best, st.loco(self.chrs)

    def fit_bt(self, st=None):
        st = st or self.st
        cs, best = st.l1_fit_bt(self.y_raw, self.off, np.tile(self.tau, (self.P, 1)))
        return cs, best, st.loco(self.chrs)

    def chr_cols(self):
        return [(c, self.chrs.index(c) * self.R, self.chrs.count(c) * self.R) for c in sorted(set(self.chrs))]

    def dims(self, st=None):
        return dict(zip(("B", "nC", "R1", "K", "nmat", "n_aug", "nch", "len"),
                        (int(x) for x in (st or self.st).debug("l1_dims", np.int64, 8))))


# ------------------------------------------------------------------------------------------------------- checks
def check_chunks(case, st=None):
    """The chunk table partitions every padded fold exactly, in order, into chunks of the rule's length (a multiple of
    128; only a fold's last chunk may be shorter), and stays within max_chunks."""
    d = case.dims(st)
    ch = (st or case.st).debug("l1_chunks", np.int32, 4 * d["nch"]).reshape(d["nch"], 4).astype(np.int64)
    pad = round_up(case.fold_sizes, 256)
    start = np.concatenate([[0], np.cumsum(pad)])
    Npad, K, nC = int(start[-1]), case.K, d["nC"]
    max_chunks = max(K, 2 ** 30 // (8 * nC * nC))
    want = round_up(max(2048, -(-Npad // (max_chunks - K + 1))), 128)
    assert d["len"] == want and want % 128 == 0, (d, want)
    assert d["nch"] <= max_chunks
    for f in range(K):
        c = ch[ch[:, 2] == f]
        assert len(c) == -(-pad[f] // want), (f, len(c))
        assert c[0, 0] == start[f] and (c[1:, 0] == c[:-1, 0] + c[:-1, 1]).all() and c[:, 1].sum() == pad[f], f
        assert (c[:-1, 1] == want).all() and 0 < c[-1, 1] <= want and (c[:, 1] % 128 == 0).all(), f
    assert (np.diff(ch[:, 2]) >= 0).all()
    return d, ch


def fold_starts(case):
    return np.concatenate([[0], np.cumsum(case.fold_sizes)])


def check_beta(case, p, betas, taus, C_BW=4.0):
    """Normwise backward error of the solutions betas [K][R1][nC] (one system per fold f and tau):
        eta = |A_f x - b_f| / (|A_f| |x| + |b_f|) <= C_BW nC u,   A_f = W^T W - W_f^T W_f + tau I (LOOCV: nothing held
    out), b_f = W^T y - W_f^T y_f, both exact here (module docstring).  The systems the kernels solve are exact but for
    the ridge shift, which adds at most u |A_f| to eta; the rest is the solve.  For the Cholesky solve Higham's
    Theorem 10.4 gives eta below 3 n^2 u in the worst case (n = nC); the error growth seen in practice is linear in n
    and far smaller (Higham, Accuracy and Stability, sec. 10.1.1).  C_BW = 4 holds the blocked Cholesky with its
    64 x 64 diagonal-block inverses to 4 nC u (1.4e-13 at nC = 320), while a system assembled without one of its
    sample chunks is off by that chunk's Gram, a relative change of about (chunk length) / N, 1e-2 or more in these
    cases.  Norms: Frobenius for A, 2-norm for vectors.  Returns the largest eta in units of nC u."""
    W, y = case.W[p], case.Y[:, p]
    B = case.B
    nC = betas.shape[-1]
    G = W.T @ W                                    # exact (see the module docstring)
    b = ld_tmv(W, y)
    st = fold_starts(case)
    worst = 0.0
    for f in range(len(betas)):
        if case.loocv:
            Af, bf = G.astype(LD), b
        else:
            Wf = W[st[f]:st[f + 1]]
            Af = (G - Wf.T @ Wf).astype(LD)
            bf = b - ld_tmv(Wf, y[st[f]:st[f + 1]])
        for r, tau in enumerate(taus):
            x = betas[f][r]
            assert not x[B:].any(), "padding coefficients of fold %d, tau %d are not zero" % (f, r)
            xl = x[:B].astype(LD)
            res = float(np.linalg.norm((Af @ xl + LD(tau) * xl - bf).astype(np.float64)))
            nA = float(np.linalg.norm(Af.astype(np.float64) + tau * np.eye(B)))
            eta = res / (nA * np.linalg.norm(x) + float(np.linalg.norm(bf.astype(np.float64))))
            worst = max(worst, eta / (nC * U))
    print("beta backward error: %.3g nC u (nC = %d, bound %g nC u)" % (worst, nC, C_BW))
    assert worst <= C_BW, "beta backward error %.3g nC u (bound %g nC u)" % (worst, C_BW)
    return worst


def check_sums(case, p, betas, sums):
    """CV sums of l1_pred_sums_kernel (Sx, Sx2, Sxy per tau; Sy, Sy2) recomputed in long double from the fetched beta.
    p1 = W_f beta_f is a sequential FMA dot product over B columns, |dp| <= e = gamma_B |W_f| |beta_f|; the per-sample
    terms p1, p1^2, p1 y, y, y^2 (one more rounding for a product) are then summed over Npad samples in a fixed order,
    within gamma_Npad of the sum of their magnitudes."""
    W, y, R1 = case.W[p], case.Y[:, p].astype(LD), case.R1
    Npad = int(round_up(case.fold_sizes, 256).sum())
    gB, gN = gamma(case.B), gamma(Npad)
    st = fold_starts(case)
    ref = np.zeros(NV, dtype=LD)
    bnd = np.zeros(NV)
    ay = np.abs(y.astype(np.float64))
    for f in range(case.K):
        sl = slice(st[f], st[f + 1])
        Bt = betas[f][:, :case.B].T
        p1 = ld_mm(W[sl], Bt)                                          # exact products
        e = gB * (np.abs(W[sl]) @ np.abs(Bt))
        a = np.abs(p1.astype(np.float64)) + e
        yf = y[sl][:, None]
        ref[0:3 * R1:3] += p1.sum(axis=0)
        ref[1:3 * R1:3] += (p1 * p1).sum(axis=0)
        ref[2:3 * R1:3] += (p1 * yf).sum(axis=0)
        bnd[0:3 * R1:3] += (e + gN * a).sum(axis=0)
        bnd[1:3 * R1:3] += ((2 * a) * e + (U + gN * (1 + U)) * a * a).sum(axis=0)
        bnd[2:3 * R1:3] += ((e + (U + gN * (1 + U)) * a) * ay[sl][:, None]).sum(axis=0)
    ref[24], ref[25] = y.sum(), (y * y).sum()
    bnd[24], bnd[25] = gN * ay.sum(), (U + gN * (1 + U)) * (ay * ay).sum()
    live = np.r_[np.arange(3 * R1), 24, 25]
    err = np.abs(sums[live].astype(LD) - ref[live]).astype(np.float64)
    ex = float((err / np.maximum(bnd[live], 1e-300)).max())
    assert ex <= 1.0, "CV sums exceed their error bound %.3g-fold (%s)" % (ex, np.argmax(err / bnd[live]))
    assert not sums[3 * R1:24].any(), "CV sums of unused ridge slots are not zero"


def check_kfold(case, cs, best, loco, d, beta_folds=None):
    """Oracle (cs 1e-8, best, LOCO 1e-7) and the long-double checks for every phenotype."""
    K, R1, nC, P = case.K, case.R1, d["nC"], case.P
    beta = case.st.debug("l1_beta", np.float64, P * K * R1 * nC).reshape(P, K, R1, nC)
    sums = case.st.debug("l1_sums", np.float64, P * NV).reshape(P, NV)
    for p in range(P):
        check_beta(case, p, beta[p], case.tau)
        check_sums(case, p, beta[p], sums[p])
        y = case.Y[:, p]
        if beta_folds is None:
            cs_o, betas_o = step1.level1_kfold(case.W[p], y, case.fold_sizes, case.tau)
            assert rel(cs[:, p, :], cs_o) < 1e-8
            assert best[p] == step1.pick_tau(cs_o, case.neff[p])
            pred = step1.predictions_kfold(case.W[p], betas_o, case.fold_sizes, best[p], case.chr_cols())
            assert rel(loco[p], step1.loco_matrix(pred, case.chr_cols())) < 1e-7
        else:
            # the oracle on a subset of folds: beta against a plain FP64 solve, cs against the GPU's own sums
            st = fold_starts(case)
            G, b = case.W[p].T @ case.W[p], case.W[p].T @ y
            for f in beta_folds:
                Wf = case.W[p][st[f]:st[f + 1]]
                A, bf = G - Wf.T @ Wf, b - Wf.T @ y[st[f]:st[f + 1]]
                for r, tau in enumerate(case.tau):
                    assert rel(beta[p, f, r, :case.B], np.linalg.solve(A + tau * np.eye(case.B), bf)) < 1e-8, (f, r)
            s = sums[p]
            assert np.array_equal(cs[:, p, :], np.stack([s[0:3 * R1:3], np.full(R1, s[24]), s[1:3 * R1:3],
                                                         np.full(R1, s[25]), s[2:3 * R1:3]]))
            assert best[p] == step1.pick_tau(cs[:, p, :], case.neff[p])
    return beta


# --------------------------------------------------------------------------------------------- (a) sample chunks
def test_folds_span_several_chunks():
    """N = 23 000 in K = 5 folds of 4600 samples, padded to 4608: chunks of 2048, 2048 and 512 per fold."""
    case = L1Case(23000, 8, seed=1)
    cs, best, loco = case.fit()
    d, ch = check_chunks(case)
    assert (d["B"], d["nC"], d["len"], d["nch"]) == (40, 64, 2048, 15), d
    assert list(ch[ch[:, 2] == 4][:, 1]) == [2048, 2048, 512]
    check_kfold(case, cs, best, loco, d)


def test_chunk_length_set_by_the_partial_cap():
    """B = 500 blocks x 5 = 2500 (nC = 2560): max_chunks = 2^30 / (8 * 2560^2) = 20, so the chunk length is
    round_up(ceil(60160 / 16), 128) = 3840 > 2048 and each fold of 12 032 padded samples takes 4 chunks, the last
    of 512.  25 systems at nC = 2560, 10 passes of the beta loop of l1_pred_sums_kernel.  The oracle's
    eigendecompositions at B = 2500 are slow, so beta is compared with an FP64 solve on folds 0 and 4 only; the
    long-double checks cover every fold."""
    case = L1Case(60000, 500, P=1, seed=2)
    cs, best, loco = case.fit()
    d, ch = check_chunks(case)
    assert (d["nC"], d["nmat"], d["len"], d["nch"]) == (2560, 25, 3840, 20), d
    assert list(ch[ch[:, 2] == 0][:, 1]) == [3840, 3840, 3840, 512]
    check_kfold(case, cs, best, loco, d, beta_folds=(0, 4))
    # LOCO rows are the per-chromosome parts of W beta_f at tau*: recomputed in FP64 from the fetched beta
    beta = case.st.debug("l1_beta", np.float64, case.K * case.R1 * d["nC"]).reshape(case.K, case.R1, d["nC"])
    pred = step1.predictions_kfold(case.W[0], [beta[f, :, :case.B].T for f in range(case.K)], case.fold_sizes,
                                   best[0], case.chr_cols())
    assert rel(loco[0], step1.loco_matrix(pred, case.chr_cols())) < 1e-10


# ----------------------------------------------------------------------------------------------- (b) column tiling
@pytest.mark.parametrize("B,R,R1,K", [(5, 5, 2, 2), (64, 4, 8, 16), (65, 5, 2, 16), (300, 5, 8, 2)])
def test_column_tiling_ridge_and_fold_counts(B, R, R1, K):
    """B = 5 (one partial DMMA tile), 64 (one exact tile), 65 (a tile and one column), 300 (two beta passes of 256 and
    44 columns); R1 = 2 and 8 (the smallest and largest dynamic shared memory of l1_pred_sums_kernel); K = 2 and
    16 (the bounds of fold_v in l1_assemble_kernel, which level 0's dense route shares).  Uneven folds."""
    N = 4100
    rng = np.random.default_rng(B)
    fs = rng.multinomial(N - 150 * K, np.ones(K) / K) + 150
    case = L1Case(N, B // R, R=R, R1=R1, seed=B + K, fold_sizes=fs)
    cs, best, loco = case.fit()
    d, _ = check_chunks(case)
    assert (d["B"], d["nC"], d["R1"], d["K"], d["nmat"]) == (B, round_up(B, 64), R1, K, K * R1), d
    check_kfold(case, cs, best, loco, d)


def test_refusals():
    """R1 = 9 ridge values, K = 17 folds and a logistic level 1 over 6005 predictors are refused with a clear error
    before anything is launched.  A refused fit leaves no fit behind: after the logistic refusal on a handle that had
    a QT fit, rg_loco and the level-1 hooks refuse instead of reading the earlier fit's buffers."""
    case = L1Case(600, 2, P=1, R1=9, seed=3)
    n0 = case.st.launch_count()
    with pytest.raises(capi.RgError, match="n_ridge_l1 out of range"):
        case.fit()
    assert case.st.launch_count() == n0
    with pytest.raises(capi.RgError, match="n_folds out of range"):
        capi.Step1(case.X, case.Y, case.mask, np.ones(600, np.uint8), hostprep.fold_sizes(600, 17), np.ones(5),
                   case.neff, 600, 1, 2)
    case = L1Case(600, 1201, P=1, R1=2, seed=3)
    case.fit()
    assert case.dims()["B"] == 6005
    n0 = case.st.launch_count()
    y = (case.Y > 0).astype(float)
    with pytest.raises(capi.RgError, match="up to 6000"):
        case.st.l1_fit_bt(y, np.zeros_like(y), np.ones((1, 2)))
    assert case.st.launch_count() == n0
    with pytest.raises(capi.RgError, match="must run before rg_loco"):
        case.st.loco(case.chrs)
    with pytest.raises(capi.RgError, match="no level-1 fit"):
        case.dims()
    case.st.close()


# ---------------------------------------------------------------------------------------------------------- (c) LOCO
def test_loco_chromosome_gaps_and_x():
    """Blocks on chromosomes 1, 7 and 23: gaps between chromosomes, chromosome 23's row, the absent chromosomes'
    rows equal to the whole-genome prediction, which is what rg_prs returns."""
    case = L1Case(3000, 12, chrs=[1] * 3 + [7] * 5 + [23] * 4, seed=4)
    cs, best, loco = case.fit()
    d, _ = check_chunks(case)
    check_kfold(case, cs, best, loco, d)
    prs = case.st.prs()
    for p in range(case.P):
        for c in set(range(1, 24)) - {1, 7, 23}:
            assert np.array_equal(loco[p][:, c - 1], prs[p])
        # the three per-chromosome parts add up to the whole-genome prediction
        parts = prs[p][:, None] - loco[p][:, [0, 6, 22]]
        assert np.abs(parts.sum(axis=1) - prs[p]).max() <= 1e-12 * np.abs(parts).sum(axis=1).max()


def test_loco_single_chromosome():
    """One chromosome: its own LOCO row is exactly zero, every other row is the whole-genome prediction."""
    case = L1Case(3000, 6, chrs=[5] * 6, seed=5)
    cs, best, loco = case.fit()
    d, _ = check_chunks(case)
    check_kfold(case, cs, best, loco, d)
    prs = case.st.prs()
    for p in range(case.P):
        assert not loco[p][:, 4].any()
        assert all(np.array_equal(loco[p][:, c], prs[p]) for c in range(23) if c != 4)
        assert np.abs(prs[p]).max() > 0


# --------------------------------------------------------------------------------------------------------- (d) LOOCV
def test_loocv_level0_and_level1_past_65535_samples(tmp_path):
    """Full LOOCV run from a .bed at N = 66 000 (Npad = 66 048 > 65 535, the old gridDim.y limit of the fill
    kernels), P = 9 traits (two phenotype tiles of l0_loocv_pred_kernel, the second with one trait)."""
    pb = helpers.synthetic_problem(tmp_path, N=66000, M=100, P=9, C=3, bsize=50, miss=0.02, loocv=True, seed=11)
    st = pb.gpu_step1()
    for b in range(len(pb.blocks)):
        pb.gpu_l0_block(st, b)
    assert st.status() == 0
    assert int(st.debug("dims", np.int64, 8)[0]) == 66048
    P, R = 9, 5
    B = len(pb.blocks) * R
    tau = B * (1 - pb.h0) / pb.h0
    cs, best = st.l1_fit(np.tile(tau, (P, 1)))
    loco = st.loco([c for c, _, _ in pb.blocks])
    assert st.status() == 0
    d = dict(zip(("B", "nC", "R1", "K", "nmat", "n_aug", "nch", "len"), st.debug("l1_dims", np.int64, 8)))
    assert (d["nmat"], d["n_aug"]) == (5, d["nC"] + 64 + 66048), d

    def gen():
        for b in range(len(pb.blocks)):
            yield pb.oracle_block(b)[0]
    o = step1.run_step1_qt(gen(), pb.blocks, pb.prep, pb.fold_sizes, pb.M, loocv=True)
    for ph in range(P):
        for b in range(len(pb.blocks)):
            assert rel(st.fetch_W(b, ph), o["W"][ph][:, b * R:(b + 1) * R]) < 1e-8, (b, ph)
        assert rel(cs[:, ph, :], o["cs"][ph]) < 1e-7, ph
        assert best[ph] == o["best"][ph]
        assert rel(loco[ph], o["loco"][ph]) < 1e-6, ph
    st.close()


def test_loocv_level1_wide():
    """B = 300 loaded predictors (nC = 320) at N = 3000: l1_loocv_sums, the row backsolve and l1_loocv_chr_pred over
    five 64-wide column panels; the coefficients at tau* against the long-double backward-error bound and the
    leverages against an FP64 solve."""
    case = L1Case(3000, 60, loocv=True, seed=6)
    cs, best, loco = case.fit()
    d, _ = check_chunks(case)
    assert (d["nC"], d["nmat"], d["n_aug"]) == (320, 5, 320 + 64 + 3072), d
    bvec = case.st.debug("l1_bvec", np.float64, case.P * 320).reshape(case.P, 320)
    hvec = case.st.debug("l1_hvec", np.float64, case.P * 3072).reshape(case.P, 3072)
    for p in range(case.P):
        W, y = case.W[p], case.Y[:, p]
        cs_o = step1.level1_loocv(W, y, case.tau, case.neff[p], 1)
        assert rel(cs[:, p, :], cs_o) < 1e-7
        assert best[p] == step1.pick_tau(cs_o, case.neff[p])
        pred = step1.predictions_loocv(W, y, case.tau[best[p]], case.chr_cols())
        assert rel(loco[p], step1.loco_matrix(pred, case.chr_cols())) < 1e-6
        tb = case.tau[best[p]]
        check_beta(case, p, bvec[p][None, None, :], [tb])
        A = W.T @ W + tb * np.eye(case.B)
        h = (W * np.linalg.solve(A, W.T).T).sum(axis=1)
        assert rel(hvec[p][:case.N], h) < 1e-10 and not hvec[p][case.N:].any()


# ------------------------------------------------------------------------------------------------ (e) binary traits
def _check_bt(case, cs, best, loco):
    for p in range(case.P):
        W, y, off, m = case.W[p], case.y_raw[:, p], case.off[:, p], case.mask[:, p].astype(bool)
        if case.loocv:
            cs_o = step1_bt.level1_logistic_loocv(W, y, off, m, case.tau)
        else:
            cs_o, betas = step1_bt.level1_logistic_kfold(W, y, off, m, case.tau, case.fold_sizes)
        np.testing.assert_allclose(cs[:, p, :], cs_o, rtol=1e-7, atol=1e-9)
        best_o, _ = step1_bt.output_table(cs_o, case.neff[p], case.B, case.tau)
        assert best[p] == best_o
        if case.loocv:
            pred = step1_bt.predictions_binary_loocv(W, y, off, m, case.tau[best_o], case.chr_cols())
        else:
            pred = step1_bt.predictions_binary_kfold(W, betas, best_o, case.fold_sizes, case.chr_cols())
        np.testing.assert_allclose(loco[p], step1.loco_matrix(pred, case.chr_cols()), rtol=1e-6, atol=1e-8)


def test_logistic_kfold_folds_span_two_chunks():
    """The k-fold logistic level 1 the driver runs for N >= 5000: N = 12 000, K = 5 folds of 2400 samples padded to
    2560, each two chunks (2048 + 512), B = 100."""
    case = L1Case(12000, 20, P=1, bt=True, seed=7)
    cs, best, loco = case.fit_bt()
    d, ch = check_chunks(case)
    assert (d["nC"], d["len"], d["nch"]) == (128, 2048, 10), d
    _check_bt(case, cs, best, loco)


def test_logistic_loocv_wide():
    """LOOCV logistic level 1 at N = 4900, B = 1500: l1_bt_eta_kernel with 12 000 bytes of shared memory, leverages
    from 5120 sample rows riding along the factorisation at nC = 1536."""
    case = L1Case(4900, 300, P=1, R1=2, loocv=True, bt=True, seed=8)
    cs, best, loco = case.fit_bt()
    d, _ = check_chunks(case)
    assert (d["B"], d["nC"], d["n_aug"]) == (1500, 1536, 1536 + 64 + 5120), d
    _check_bt(case, cs, best, loco)


# ------------------------------------------------------------------------------------------------------- (f) refits
def test_refit_equals_a_fresh_handle():
    """rg_l1_fit twice on one handle with different tau grids gives what a fresh handle gives for the second grid,
    bit for bit; a QT fit after a logistic one on a LOOCV handle takes the QT LOCO route."""
    case = L1Case(3000, 13, seed=9)
    case.fit(tau=case.tau * 3)
    got = case.fit()
    beta = case.st.debug("l1_beta", np.float64, case.P * case.K * case.R1 * 128)
    fresh = case.handle()
    want = case.fit(st=fresh)
    for a, b in zip(got, want):
        assert np.array_equal(a, b)
    assert np.array_equal(beta, fresh.debug("l1_beta", np.float64, beta.size))
    fresh.close()

    case = L1Case(2000, 10, P=1, loocv=True, bt=True, seed=10)
    case.fit_bt()
    got = case.fit()
    fresh = case.handle()
    want = case.fit(st=fresh)
    for a, b in zip(got, want):
        assert np.array_equal(a, b)
    fresh.close()
