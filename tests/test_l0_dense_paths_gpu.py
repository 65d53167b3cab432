"""The dense FP64 level-0 route (rg_l0_block_dosage_u8 / rg_l0_block_f64: every Step-1 block read from a .bgen file) at
the shapes that select its chunking, tiling and solver.

The route decodes the probability pairs into an FP64 [bs][Npad] matrix, imputes / residualises / scales it
(dense_prepare), sums per-chunk Gram partials of kStatChunk = 2048 padded samples per fold (level 1's l1_assemble), factors the
K*R shifted systems (batched Cholesky) and predicts in tiles of DQ = 25 outputs (dense_predict); LOOCV carries the samples
as extra right-hand-side rows of the factorisation and predicts in tiles of at most 8 phenotypes (l0_loocv_pred).
Every case asserts through the "dims" hook (Npad, rp, nC, n_aug, nmat, K, cpp, nchunks) which shape ran, and compares
the level-0 predictors with the oracle fed with the oracle's own dosage decode, at 1e-9 relative unless it says otherwise.
"""
import numpy as np
import pytest

import helpers
from oracle import bgen as obgen
from oracle import plink, prep, step1
from regenie_b200 import capi, synth


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except ImportError:
        return False


pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not _has_gpu(), reason="needs a CUDA device")]
TOL = 1e-9
LD = np.longdouble
STAT_CHUNK = 2048           # samples per Gram partial (kStatChunk)
FOLD_PAD = 256              # folds start on 256-sample boundaries (kFoldPad)


def rel(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def round_up(x, m):
    return (x + m - 1) // m * m


def _fileset(d, n_file, P, C=3, n_snp=6, seed=5, drop=True):
    """PLINK fileset of n_file samples whose phenotype / covariate files lack a few of them.  Only the sample list, the
    phenotypes and the covariates matter here: the level-0 blocks are synthetic probability pairs."""
    g = synth.genotypes(n_file, n_snp, seed=seed, miss=0.0)
    Y, cov, na = synth.phenotypes(g, P, C, seed=seed, n_causal=n_snp, na_frac=0.03)
    drop_p = {5, 77, n_file - 3} if drop else ()
    drop_c = {11} if drop else ()
    return helpers.write_fileset(str(d), g, Y, cov, na, drop_pheno=drop_p, drop_cov=drop_c)


class Case:
    """One Step-1 configuration: the prepared samples, folds and ridge grid, and a handle factory."""

    def __init__(self, prefix, K=5, loocv=False, remove=None, R=5, m_eff=20000):
        self.pb = helpers.Problem(prefix, prefix.rsplit("/", 1)[0] + "/pheno.txt", prefix.rsplit("/", 1)[0] + "/covar.txt",
                                  64, K=K, loocv=loocv, remove=remove)
        h0 = prep.set_ridge_params(5) if R == 5 else np.linspace(0.01, 0.99, R)
        self.lam = m_eff * (1 - h0) / h0
        self.loocv = loocv
        self.idx = None if self.pb.keep.all() else self.pb.sample_idx

    @property
    def pr(self):
        return self.pb.prep

    def step1(self, bs_max, total_blocks=1):
        pr = self.pr
        return capi.Step1(pr.X, pr.Y, pr.mask, pr.in_analysis, self.pb.fold_sizes, self.lam, pr.neff, pr.n_analyzed,
                          bs_max, total_blocks, loocv=self.loocv)

    def expected_dims(self, bs, nmat):
        pad = [round_up(int(f), FOLD_PAD) for f in self.pb.fold_sizes]
        Npad = sum(pad)
        nC, Ppad = round_up(bs, 64), round_up(self.pr.Y.shape[1], 64)
        n_aug = nC + Ppad + (Npad if self.loocv else 0)
        return Npad, round_up(bs, 128), nC, n_aug, nmat, sum((p + STAT_CHUNK - 1) // STAT_CHUNK for p in pad)

    def check_dims(self, st, bs):
        d = [int(x) for x in st.debug("dims", np.int64, 8)]
        K = 1 if self.loocv else len(self.pb.fold_sizes)
        Npad, rp, nC, n_aug, nmat, nch = self.expected_dims(bs, K * len(self.lam))
        assert d[:5] == [Npad, rp, nC, n_aug, nmat] and d[5] == K and d[7] == nch, d
        assert d[6] == round_up(self.pr.X.shape[1] + self.pr.Y.shape[1], 16)
        return dict(Npad=d[0], nC=d[2], nchunks=d[7])

    def oracle_W(self, probs, miss, ref_first=False):
        g = _decode(probs, miss, ref_first)[:, self.pb.keep]
        gi, _ = plink.mean_impute_block(g, self.pr.in_analysis)
        Gt, _ = step1.residualize_genotypes(gi, self.pr.X, self.pr.in_analysis, self.pr.n_analyzed, self.pr.ncov)
        if self.loocv:
            return step1.level0_loocv(Gt, self.pr.Y, self.pr.mask, self.lam, self.pr.neff)
        return step1.level0_kfold(Gt, self.pr.Y, self.pr.mask, self.pb.fold_sizes, self.lam, self.pr.neff)


def _decode(probs, miss, ref_first=False):
    """Dosages of the probability pairs as the oracle reads a BGEN file (-3 = missing), [bs][n_file]."""
    return np.stack([obgen.dosage(probs[v, :, 0].astype(np.float64), probs[v, :, 1].astype(np.float64),
                                  (miss[v] & 0x80) != 0, ref_first=ref_first)[0] for v in range(probs.shape[0])])


def _probs(rng, bs, n, miss_frac=0.02):
    """8-bit probability pairs: most calls (nearly) hard, the rest fractional; about miss_frac of them missing."""
    p0 = rng.integers(0, 256, size=(bs, n))
    p1 = (rng.random((bs, n)) * (256 - p0)).astype(np.int64)
    certain = rng.random((bs, n)) < 0.7
    maf = rng.uniform(0.05, 0.5, size=(bs, 1))
    g = rng.binomial(2, maf, size=(bs, n))
    p0 = np.where(certain, (g == 2) * 255, p0)
    p1 = np.where(certain, (g == 1) * 255, p1)
    probs = np.stack([p0, p1], axis=2).astype(np.uint8)
    miss = np.where(rng.random((bs, n)) < miss_frac, 0x82, 0x02).astype(np.uint8)
    return probs, miss


def _hard_calls(rng, bs, n, miss_frac=0.02):
    """Hard calls in {0, 1, 2} and 3 = missing, as 0/255 probability pairs + missing flags and as 2-bit .bed rows."""
    g = synth.genotypes(n, bs, seed=int(rng.integers(1 << 30)), miss=miss_frac)
    probs = np.stack([(g == 2) * 255, (g == 1) * 255], axis=2).astype(np.uint8)
    miss = np.where(g == 3, 0x82, 0x02).astype(np.uint8)
    return probs, miss, synth.pack_bed(g)


def _check_W(st, W_o, block_id=0, tol=TOL):
    for ph in range(len(W_o)):
        W = st.fetch_W(block_id, ph)
        assert np.isfinite(W).all()
        assert rel(W, W_o[ph]) < tol, (block_id, ph, rel(W, W_o[ph]))


# ------------------------------------------------------------------------------------------------------ fixtures
N_BIG = 30001               # samples kept of the 30 004 in the file


@pytest.fixture(scope="module")
def big(tmp_path_factory):
    d = tmp_path_factory.mktemp("big")
    return _fileset(d, N_BIG + 3, P=6, seed=21)


@pytest.fixture(scope="module")
def big_case(big):
    return Case(big, K=5, remove={"F2_I2", "F15000_I15000", "F30003_I30003"})


@pytest.fixture(scope="module")
def big_block(big_case):
    """Case 1's block and its handle, shared by the checks that read the same run."""
    bs = 1000
    probs, miss = _probs(np.random.default_rng(101), bs, big_case.pb.n_file)
    st = big_case.step1(bs)
    st.l0_block_dosage_u8(probs, miss, 0, sample_idx=big_case.idx, ref_first=True)
    assert st.status() == 0
    yield probs, miss, st
    st.close()


# ------------------------------------------------------------------------------------- A. dense route vs the oracle
def test_chunked_gram_second_predict_tile_wide_cholesky(big_case, big_block):
    """N = 30 001 over 5 folds of 3 Gram chunks each (nchunks = 15), R * P = 30 outputs (a second dense_predict tile with
    5 live outputs), nC = 1024 (16 Cholesky panels); a sample subset of the file, ref-first dosages."""
    probs, miss, st = big_block
    assert big_case.pr.Y.shape[1] * len(big_case.lam) == 30
    dims = big_case.check_dims(st, 1000)
    assert dims["nchunks"] == 15 and dims["nC"] == 1024
    _check_W(st, big_case.oracle_W(probs, miss, ref_first=True))


def test_two_folds_short_last_chunk(big):
    """K = 2: 7 full chunks + one of 768 per fold; bs = 65 -> nC = 128, prediction loop of 64 + 1 rows."""
    c = Case(big, K=2)
    pad = [round_up(int(f), FOLD_PAD) for f in c.pb.fold_sizes]
    assert all(p % STAT_CHUNK == 768 and p // STAT_CHUNK == 7 for p in pad), pad
    bs = 65
    probs, miss = _probs(np.random.default_rng(102), bs, c.pb.n_file)
    st = c.step1(bs)
    st.l0_block_dosage_u8(probs, miss, 0, sample_idx=c.idx)
    assert st.status() == 0
    dims = c.check_dims(st, bs)
    assert dims["nchunks"] == 16 and dims["nC"] == 128
    _check_W(st, c.oracle_W(probs, miss))
    st.close()


@pytest.mark.parametrize("R", [1, 8])
def test_sixteen_folds(tmp_path, R):
    """K = kMaxFolds = 16 fills the assembler's per-fold registers; nmat = 16 R systems."""
    c = Case(_fileset(tmp_path, 20000, P=3, seed=22), K=16, R=R)
    bs = 64
    probs, miss = _probs(np.random.default_rng(103 + R), bs, c.pb.n_file)
    st = c.step1(bs)
    st.l0_block_dosage_u8(probs, miss, 0, sample_idx=c.idx)
    assert st.status() == 0
    c.check_dims(st, bs)
    assert int(st.debug("dims", np.int64, 8)[4]) == 16 * R
    _check_W(st, c.oracle_W(probs, miss))
    st.close()


def test_loocv_many_chunks_two_pheno_tiles(tmp_path):
    """LOOCV at N = 66 000 (past the 65 280 padded samples that once capped a grid axis): the sample rows of
    l1_loocv_fill span many chunks, and P = 9 runs l0_loocv_pred in two phenotype tiles (8 + 1)."""
    c = Case(_fileset(tmp_path, 66000, P=9, seed=23), loocv=True)
    bs = 64
    probs, miss = _probs(np.random.default_rng(104), bs, c.pb.n_file)
    st = c.step1(bs)
    st.l0_block_dosage_u8(probs, miss, 0, sample_idx=c.idx)
    assert st.status() == 0
    dims = c.check_dims(st, bs)
    assert dims["Npad"] > 65280 and dims["nchunks"] == 33
    _check_W(st, c.oracle_W(probs, miss))
    st.close()


def test_short_blocks_after_long_ones_and_lanes(tmp_path, monkeypatch):
    """Blocks of 1000, 1, 37 and 1000 SNPs on one handle: the short ones run in the scratch (gd, cm, dpart) the long one
    sized.  Each against the oracle with one lane, and bit-identical with three lanes."""
    c = Case(_fileset(tmp_path, 9000, P=4, seed=24), remove={"F8_I8", "F4000_I4000"})
    sizes = [1000, 1, 37, 1000]
    rng = np.random.default_rng(105)
    blocks = [_probs(rng, bs, c.pb.n_file) for bs in sizes]
    W = {}
    for lanes in (1, 3):
        monkeypatch.setenv("RG_B200_LANES", str(lanes))
        st = c.step1(1000, total_blocks=len(sizes))
        for b, (probs, miss) in enumerate(blocks):
            st.l0_block_dosage_u8(probs, miss, b, sample_idx=c.idx, ref_first=(b == 2))
            c.check_dims(st, sizes[b])
        assert st.status() == 0
        W[lanes] = [[st.fetch_W(b, ph) for ph in range(4)] for b in range(len(sizes))]
        st.close()
    for b, (probs, miss) in enumerate(blocks):
        W_o = c.oracle_W(probs, miss, ref_first=(b == 2))
        for ph in range(4):
            assert rel(W[1][b][ph], W_o[ph]) < TOL, (b, ph)
            assert np.array_equal(W[1][b][ph], W[3][b][ph]), (b, ph)


# ---------------------------------------------------------------------------------- B. cross-checks without an oracle
@pytest.mark.parametrize("N,bs", [(8000, 1000), (12000, 2500)])
def test_dense_route_matches_2bit_route_on_hard_calls(tmp_path, monkeypatch, N, bs):
    """The same hard calls as 0/255 probability pairs through the dense route and as 2-bit rows through the .bed route.
    bs = 1000: the mixed solver on the 2-bit side; bs = 2500: FP64 Cholesky and FP64 prediction on both sides."""
    monkeypatch.delenv("RG_B200_SOLVER", raising=False)
    c = Case(_fileset(tmp_path, N, P=3, seed=25))
    probs, miss, packed = _hard_calls(np.random.default_rng(106), bs, c.pb.n_file)
    st_d = c.step1(bs)
    st_d.l0_block_dosage_u8(probs, miss, 0, sample_idx=c.idx)
    assert st_d.status() == 0
    c.check_dims(st_d, bs)
    st_b = c.step1(bs)
    st_b.l0_block_bed(packed, bs, 0, sample_idx=c.idx)
    assert st_b.status() == 0
    paths = tuple(int(x) for x in st_b.debug("paths", np.int64, 3))
    if bs <= 2048:
        assert paths[2] > 0 and st_b.solver_stats() == (1, 0)          # mixed solver, no FP64 re-solve
    else:
        assert paths[1:] == (0, 0)                                      # FP64 prediction, FP64 Cholesky
    assert tuple(int(x) for x in st_d.debug("paths", np.int64, 3))[1:] == (0, 0)
    for ph in range(3):
        Wb = st_b.fetch_W(0, ph)
        assert rel(st_d.fetch_W(0, ph), Wb) < 2e-9, ph
    st_d.close()
    st_b.close()


def test_f64_entry_point_is_bit_identical(big_case, big_block):
    """G = p1/255 + 2 (p0/255) (-3 = missing) built in numpy, as dense_from_dosage does it: rg_l0_block_f64 on it gives
    the very W of rg_l0_block_dosage_u8 on the pairs (the factor 2 is exact, so any difference is in the decode)."""
    probs, miss, _ = big_block
    bs = probs.shape[0]
    p0, p1 = probs[:, :, 0].astype(np.float64), probs[:, :, 1].astype(np.float64)
    G = np.where(miss & 0x80, -3.0, p1 / 255.0 + 2.0 * (p0 / 255.0))
    st_u8 = big_case.step1(bs)
    st_u8.l0_block_dosage_u8(probs, miss, 0, sample_idx=big_case.idx)
    st_f = big_case.step1(bs)
    st_f.l0_block_f64(G, 0, sample_idx=big_case.idx)
    assert st_u8.status() == 0 and st_f.status() == 0
    big_case.check_dims(st_f, bs)
    for ph in range(6):
        assert np.array_equal(st_f.fetch_W(0, ph), st_u8.fetch_W(0, ph)), ph
    st_u8.close()
    st_f.close()


def test_prepared_statistics(big_case, big_block):
    """mu and inv_sd of the block against a long-double recomputation: the mean over analysed non-missing samples, and
    1 / sd with the N_analyzed - C divisor (inv_sd holds 1 / sd on both level-0 routes)."""
    probs, miss, st = big_block
    bs = probs.shape[0]
    rp = int(st.debug("dims", np.int64, 8)[1])
    mu = st.debug("mu", np.float64, rp)[:bs]
    inv_sd = st.debug("inv_sd", np.float64, rp)[:bs]
    pr = big_case.pr
    g = _decode(probs, miss, ref_first=True)[:, big_case.pb.keep].astype(LD)
    ia = pr.in_analysis.astype(bool)
    ok = ia[None, :] & (g != -3)
    mu_o = np.where(ok, g, 0).sum(axis=1) / ok.sum(axis=1)
    gi = np.where(g == -3, mu_o[:, None], g) * ia[None, :]
    X = pr.X.astype(LD)
    r = gi - (gi @ X) @ X.T
    inv_sd_o = np.sqrt(LD(pr.n_analyzed - pr.ncov)) / np.sqrt((r * r).sum(axis=1))
    assert float(np.abs(mu - mu_o).max() / np.abs(mu_o).max()) < 1e-13
    assert float(np.abs((inv_sd - inv_sd_o) / inv_sd_o).max()) < 1e-13


# --------------------------------------------------------------------------------------- C. limits and reports
@pytest.mark.parametrize("route", ["dense", "bed_f64", "bed_mixed"])
def test_two_hundred_phenotypes(tmp_path, monkeypatch, route):
    """P = 200 in k-fold: the FP64 backward substitution takes the right-hand sides in chunks of a fixed shared-memory
    size, on the dense route and on the 2-bit route with the FP64 or the mixed solver."""
    if route == "bed_f64":
        monkeypatch.setenv("RG_B200_SOLVER", "f64")
    else:
        monkeypatch.delenv("RG_B200_SOLVER", raising=False)
    N, bs, P = 6000, 256, 200
    c = Case(_fileset(tmp_path, N, P=P, seed=26))
    st = c.step1(bs)
    rng = np.random.default_rng(107)
    if route == "dense":
        probs, miss = _probs(rng, bs, c.pb.n_file)
        st.l0_block_dosage_u8(probs, miss, 0, sample_idx=c.idx)
        W_o = c.oracle_W(probs, miss)
    else:
        _, _, packed = _hard_calls(rng, bs, c.pb.n_file)
        st.l0_block_bed(packed, bs, 0, sample_idx=c.idx)
        g = plink.decode_bed(packed, c.pb.n_file, keep=c.pb.keep)
        gi, _ = plink.mean_impute_block(g, c.pr.in_analysis)
        Gt, _ = step1.residualize_genotypes(gi, c.pr.X, c.pr.in_analysis, c.pr.n_analyzed, c.pr.ncov)
        W_o = step1.level0_kfold(Gt, c.pr.Y, c.pr.mask, c.pb.fold_sizes, c.lam, c.pr.neff)
        paths = tuple(int(x) for x in st.debug("paths", np.int64, 3))
        assert (paths[2] > 0) == (route == "bed_mixed")
    assert st.status() == 0
    c.check_dims(st, bs)
    _check_W(st, W_o)
    st.close()


@pytest.mark.parametrize("route", ["dense", "bed"])
def test_loocv_wide_block(tmp_path, route):
    """LOOCV with bsize = 3600 (nC = 3648) and P = 8: eight u rows of 3648 doubles exceed the shared memory a block may
    opt into on an H100 (227 KiB), so l0_loocv_pred runs the phenotypes in tiles that fit (7 + 1)."""
    N, bs, P = 4500, 3600, 8
    c = Case(_fileset(tmp_path, N, P=P, seed=27), loocv=True)
    st = c.step1(bs)
    rng = np.random.default_rng(108)
    if route == "dense":
        probs, miss = _probs(rng, bs, c.pb.n_file)
        st.l0_block_dosage_u8(probs, miss, 0, sample_idx=c.idx)
        W_o = c.oracle_W(probs, miss)
    else:
        _, _, packed = _hard_calls(rng, bs, c.pb.n_file)
        st.l0_block_bed(packed, bs, 0, sample_idx=c.idx)
        g = plink.decode_bed(packed, c.pb.n_file, keep=c.pb.keep)
        gi, _ = plink.mean_impute_block(g, c.pr.in_analysis)
        Gt, _ = step1.residualize_genotypes(gi, c.pr.X, c.pr.in_analysis, c.pr.n_analyzed, c.pr.ncov)
        W_o = step1.level0_loocv(Gt, c.pr.Y, c.pr.mask, c.lam, c.pr.neff)
    assert st.status() == 0
    assert c.check_dims(st, bs)["nC"] == 3648
    _check_W(st, W_o)
    st.close()


@pytest.mark.parametrize("kind", ["constant", "all_missing"])
def test_low_variance_row_is_reported(tmp_path, kind):
    """A constant or an all-missing dosage row (row 17 of block 2, max_block_size 64) is reported like the 2-bit route
    reports a monomorphic SNP: status = block * 64 + row + 1; the block's predictors stay finite."""
    c = Case(_fileset(tmp_path, 3000, P=2, seed=28))
    rng = np.random.default_rng(109)
    st = c.step1(64, total_blocks=3)
    for b in range(3):
        probs, miss = _probs(rng, 64, c.pb.n_file)
        if b == 2:
            if kind == "constant":
                probs[17, :, 0], probs[17, :, 1] = 0, 255          # dosage 1 everywhere (and imputed to 1)
            else:
                miss[17, :] = 0x82
        st.l0_block_dosage_u8(probs, miss, b, sample_idx=c.idx)
    assert st.status() == 2 * 64 + 17 + 1
    for b in range(3):
        for ph in range(2):
            assert np.isfinite(st.fetch_W(b, ph)).all(), (b, ph)
    st.close()
