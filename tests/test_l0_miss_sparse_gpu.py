"""The Miss rows of the level-0 integer Gram as sparse sums over per-(SNP, fold) missing lists (miss_gram.cu).

The sparse path must leave `zz` bit-identical to the dense tensor-core tiles (RG_B200_GRAM=dense), to the CUDA-core
reference and to numpy over every entry the dense tile list writes, and take the dense tiles itself once a block has more
missing calls than its list holds.
"""
import numpy as np
import pytest

import helpers
from oracle import plink
from regenie_b200 import synth

pytestmark = pytest.mark.gpu


def dense_tile_mask(rp):
    """Entries of one fold's [2 rp][2 rp] Gram that gram_tile_list's 128 x 256 tiles write."""
    m = np.zeros((2 * rp, 2 * rp), dtype=bool)
    for nj in range(2 * rp // 256):
        for mi in range(2 * nj, 2 * rp // 128):
            m[128 * mi:128 * mi + 128, 256 * nj:256 * nj + 256] = True
    return m


def make_problem(tmp, g, bs, K=5, remove=None, loocv=False, n_chr=3):
    Y, cov, na = synth.phenotypes(g, 3, 3, seed=7, na_frac=0.03)
    prefix = helpers.write_fileset(str(tmp), g, Y, cov, na, n_chr=n_chr)
    return helpers.Problem(prefix, str(tmp) + "/pheno.txt", str(tmp) + "/covar.txt", bs, K=K, loocv=loocv,
                           remove=remove)


def numpy_zz(pb, b, rp):
    """[K][2 rp][2 rp] exact Z_f Z_f^T from the raw calls, Z = [G0; Miss] (missing calls: G0 = 0, Miss = 1)."""
    _, s, bs = pb.blocks[b]
    g = plink.decode_bed(pb.packed[s:s + bs], pb.n_file, keep=pb.keep)
    g = np.where(pb.prep.in_analysis[None, :], g, 0.0)
    cut = np.concatenate([[0], np.cumsum(pb.fold_sizes)])
    out = []
    for f in range(len(pb.fold_sizes)):
        gf = g[:, cut[f]:cut[f + 1]]
        Z = np.zeros((2 * rp, gf.shape[1]), dtype=np.int64)
        Z[:bs] = np.where(gf == -3, 0, gf)
        Z[rp:rp + bs] = gf == -3
        out.append(Z @ Z.T)
    return np.stack(out)


def run(pb, mode, monkeypatch, blocks=None, check=None):
    """Level 0 on the given blocks with RG_B200_GRAM=mode ("dense" or unset); check(st, b) after each block."""
    if mode == "dense":
        monkeypatch.setenv("RG_B200_GRAM", "dense")
    else:
        monkeypatch.delenv("RG_B200_GRAM", raising=False)
    st = pb.gpu_step1()
    W = []
    for b in (range(len(pb.blocks)) if blocks is None else blocks):
        pb.gpu_l0_block(st, b)
        assert st.status() == 0
        if check:
            check(st, b)
        W.append([st.fetch_W(b, ph) for ph in range(pb.prep.Y.shape[1])])
    return W


def last_zz(st):
    Npad, rp, nC, n_aug, nmat, K, cpp, nch = [int(x) for x in st.debug("dims", np.int64, 8)]
    zz = st.debug("zz", np.float32, K * 4 * rp * rp).reshape(K, 2 * rp, 2 * rp)
    return rp, zz


def check_block(pb, st, b, sparse, zz_dense=None):
    """zz of the last block against numpy, the CUDA-core reference and (if given) the forced-dense zz; the path taken."""
    sparse_path, total, cap = [int(x) for x in st.debug("gram_path", np.int64, 3)]
    if sparse is None:
        assert total == -1 and sparse_path == 0
    else:
        assert sparse_path == int(sparse) and (total <= cap) == sparse
    rp, zz = last_zz(st)
    m = dense_tile_mask(rp)
    ref = numpy_zz(pb, b, rp)
    assert np.array_equal(zz[:, m], ref[:, m].astype(np.float32))
    zr = st.debug("zz_ref", np.float32, zz.size).reshape(zz.shape)
    tri = np.tril(np.ones(m.shape, dtype=bool))
    assert np.array_equal(zz[:, tri], zr[:, tri])
    if zz_dense is not None:
        assert np.array_equal(zz[:, m], zz_dense[:, m])
    return zz


# (N, M, bs, missing rate, folds, sample subset, LOOCV, sparse expected)
CASES = [
    (1203, 200, 100, 0.0, 5, False, False, True),
    (1203, 260, 130, 0.001, 3, False, False, True),      # N not a multiple of 16, 3 uneven folds
    (2000, 1000, 1000, 0.01, 5, False, False, True),
    (1500, 260, 130, 0.012, 5, True, False, True),        # --remove style subset
    (1000, 2048, 2048, 0.01, 3, False, False, True),     # two 1024-column chunks per row in the sparse kernel
    (1000, 260, 130, 0.01, 1, False, True, True),        # LOOCV: one fold of every sample
    (900, 200, 100, 0.04, 5, False, False, False),       # above the threshold: the dense tiles run
]


@pytest.mark.parametrize("N,M,bs,miss,K,subset,loocv,sparse", CASES)
def test_sparse_zz_is_exact(tmp_path, monkeypatch, N, M, bs, miss, K, subset, loocv, sparse):
    g = synth.genotypes(N, M, seed=11, miss=miss)
    remove = None
    if subset:
        keys, _ = plink.read_fam(helpers.write_fileset(str(tmp_path / "k"), g[:1], np.zeros((N, 1)), np.zeros((N, 1)),
                                                       np.zeros((N, 1), bool)) + ".fam")
        remove = {keys[3], keys[400], keys[N - 1], keys[N // 2]}
    pb = make_problem(tmp_path, g, bs, K=K, remove=remove, loocv=loocv)
    dense = {}
    run(pb, "dense", monkeypatch, blocks=[0], check=lambda st, b: dense.update(zz=check_block(pb, st, b, None)))
    run(pb, "auto", monkeypatch, blocks=[0], check=lambda st, b: check_block(pb, st, b, sparse, dense["zz"]))


def test_sparse_zz_skewed_missingness(tmp_path, monkeypatch):
    """One SNP missing at every sample of one fold, and the missing calls of the block concentrated in one fold."""
    N, M, bs = 1500, 256, 256
    g = synth.genotypes(N, M, seed=5, miss=0.002)
    pb = make_problem(tmp_path, g, bs, K=5)
    cut = np.concatenate([[0], np.cumsum(pb.fold_sizes)])
    g[17, cut[1]:cut[2]] = 3
    rng = np.random.default_rng(3)
    f3 = slice(cut[3], cut[4])
    g[:, f3][rng.random(size=(M, cut[4] - cut[3])) < 0.03] = 3
    pb = make_problem(tmp_path, g, bs, K=5)
    dense = {}
    run(pb, "dense", monkeypatch, blocks=[0], check=lambda st, b: dense.update(zz=check_block(pb, st, b, None)))
    run(pb, "auto", monkeypatch, blocks=[0], check=lambda st, b: check_block(pb, st, b, True, dense["zz"]))


def test_path_switch_on_one_lane(tmp_path, monkeypatch):
    """Blocks alternating between the dense and the sparse path on one lane (zz is reused): no stale entry survives,
    and the predictors equal the forced-dense run's."""
    monkeypatch.setenv("RG_B200_LANES", "1")
    N, bs = 1100, 128
    rates = [0.05, 0.005, 0.05, 0.0, 0.01]
    g = np.concatenate([synth.genotypes(N, bs, seed=20 + k, miss=r) for k, r in enumerate(rates)])
    pb = make_problem(tmp_path, g, bs, K=5, n_chr=1)
    assert [b[2] for b in pb.blocks] == [bs] * len(rates)
    paths = []

    def check(st, b):
        paths.append(int(st.debug("gram_path", np.int64, 3)[0]))
        check_block(pb, st, b, bool(paths[-1]))

    W_sparse = run(pb, "auto", monkeypatch, check=check)
    assert paths == [0, 1, 0, 1, 1]
    W_dense = run(pb, "dense", monkeypatch)
    for a, b in zip(W_sparse, W_dense):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)


def test_multiblock_W_identical(tmp_path, monkeypatch):
    """A multi-block level 0 on the default lanes gives identical W on both paths, within the oracle's tolerance."""
    pb = helpers.synthetic_problem(tmp_path, N=1700, M=700, bsize=200, miss=0.01)
    W_sparse = run(pb, "auto", monkeypatch)
    W_dense = run(pb, "dense", monkeypatch)
    for b, (a, d) in enumerate(zip(W_sparse, W_dense)):
        W_o = pb.oracle_l0(b)[0]
        for ph in range(len(a)):
            assert np.array_equal(a[ph], d[ph])
            assert np.abs(a[ph] - W_o[ph]).max() / np.abs(W_o[ph]).max() < 1e-9
