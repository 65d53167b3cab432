"""Level-0 Gram and statistics tiles with their genotype operand built on chip from the block's 2-bit rows.

The Z Z^T tiles and the Z [X | Y]-digit statistics tiles are exact integer sums, Z = [G0; Miss] (missing calls: G0 = 0,
Miss = 1).  Both must equal numpy's integer products of the codes fetched from "gp", for every fold, and zz must equal
the CUDA-core reference.  The cases cover a 256-row B tile with G0 and Miss halves (rows_p 128), the sparse and the dense
Miss rows, sample counts that are not multiples of 16 or 128, a sample subset, uneven folds, LOOCV, and 1, 2 and 3 digit
groups of (X | Y) (128 x 128 and 128 x 256 statistics tiles).
"""
import numpy as np
import pytest

import helpers
from oracle import plink
from regenie_b200 import synth

pytestmark = pytest.mark.gpu


def fold_ranges(st, pb, npad):
    """(first padded sample, padded length) of every fold, from the padded index of each fold's first sample."""
    pad_of = st.debug("pad_of", np.int32, int(np.sum(pb.fold_sizes)))
    starts = [int(pad_of[c]) for c in np.concatenate([[0], np.cumsum(pb.fold_sizes)[:-1]])] + [npad]
    return [(starts[f], starts[f + 1] - starts[f]) for f in range(len(pb.fold_sizes))]


def z_rows(st, rp, npad):
    """Z = [G0; Miss] as float64 [2 rp][Npad] from the block's 2-bit rows (code 3 = missing)."""
    words = st.debug("gp", np.uint32, rp * (npad // 16)).reshape(rp, npad // 16)
    codes = ((words[:, :, None] >> (2 * np.arange(16, dtype=np.uint32))) & 3).reshape(rp, npad)
    return np.concatenate([np.where(codes == 3, 0, codes), codes == 3]).astype(np.float64)


def dense_tile_mask(rp):
    """Entries of one fold's [2 rp][2 rp] Gram that gram_tile_list's 128 x 256 tiles write."""
    m = np.zeros((2 * rp, 2 * rp), dtype=bool)
    for nj in range(2 * rp // 256):
        for mi in range(2 * nj, 2 * rp // 128):
            m[128 * mi:128 * mi + 128, 256 * nj:256 * nj + 256] = True
    return m


def check_block(pb, st, ncol, sparse_expected):
    npad, rp, nC, n_aug, nmat, K, cpp, nch = [int(x) for x in st.debug("dims", np.int64, 8)]
    assert pb.prep.X.shape[1] + pb.prep.Y.shape[1] == ncol
    stats_tc = int(st.debug("paths", np.int64, 3)[0])
    assert stats_tc == 1
    sparse_path = int(st.debug("gram_path", np.int64, 3)[0])
    assert sparse_path == int(sparse_expected)
    Z = z_rows(st, rp, npad)
    zz = st.debug("zz", np.float32, K * 4 * rp * rp).reshape(K, 2 * rp, 2 * rp)
    zr = st.debug("zz_ref", np.float32, zz.size).reshape(zz.shape)
    drows = 128 * (-(-ncol // 14))                  # 14 columns of (X | Y) per 128-row digit group
    D = st.debug("xyD", np.int8, drows * npad).reshape(drows, npad).astype(np.float64)
    T = st.debug("tstat", np.float32, K * 2 * rp * drows).reshape(K, 2 * rp, drows)
    m = dense_tile_mask(rp)
    tri = np.tril(np.ones(m.shape, dtype=bool))
    for f, (s0, n) in enumerate(fold_ranges(st, pb, npad)):
        Zf = Z[:, s0:s0 + n]
        assert np.array_equal(zz[f][m], (Zf @ Zf.T)[m].astype(np.float32)), "zz, fold %d" % f
        assert np.array_equal(zz[f][tri], zr[f][tri]), "zz against zz_ref, fold %d" % f
        assert np.array_equal(T[f], (Zf @ D[:, s0:s0 + n].T).astype(np.float32)), "statistics tiles, fold %d" % f


# (N, M, bs, missing rate, folds, sample subset, LOOCV, C + P, P, RG_B200_GRAM, sparse Miss rows expected)
CASES = [
    (1203, 200, 100, 0.0, 5, False, False, 13, 3, None, True),       # rows_p 128: a B tile of G0 and Miss halves
    (1203, 260, 130, 0.01, 3, False, False, 20, 3, None, True),      # N not a multiple of 16, 3 uneven folds
    (2000, 1000, 1000, 0.01, 5, False, False, 30, 4, None, True),
    (1500, 260, 130, 0.01, 5, True, False, 20, 2, None, True),       # a sample subset
    (1000, 2048, 2048, 0.01, 3, False, False, 13, 3, None, True),
    (1000, 260, 130, 0.01, 1, False, True, 13, 3, None, True),       # LOOCV: one fold of every sample
    (900, 200, 100, 0.03, 5, False, False, 30, 3, None, False),      # above the sparse threshold: dense Miss tiles
    (1100, 300, 300, 0.01, 5, False, False, 20, 3, "dense", False),  # dense Miss tiles on request
]


@pytest.mark.parametrize("N,M,bs,miss,K,subset,loocv,cp,P,mode,sparse", CASES)
def test_gram_and_stats_tiles_exact(tmp_path, monkeypatch, N, M, bs, miss, K, subset, loocv, cp, P, mode, sparse):
    if mode:
        monkeypatch.setenv("RG_B200_GRAM", mode)
    else:
        monkeypatch.delenv("RG_B200_GRAM", raising=False)
    monkeypatch.delenv("RG_B200_STATS", raising=False)
    g = synth.genotypes(N, M, seed=13, miss=miss)
    Y, cov, na = synth.phenotypes(g, P, cp - P, seed=7, na_frac=0.03)
    prefix = helpers.write_fileset(str(tmp_path), g, Y, cov, na, n_chr=1)
    remove = None
    if subset:
        keys, _ = plink.read_fam(prefix + ".fam")
        remove = {keys[3], keys[400], keys[N - 1], keys[N // 2]}
    pb = helpers.Problem(prefix, str(tmp_path / "pheno.txt"), str(tmp_path / "covar.txt"), bs, K=K, loocv=loocv,
                         remove=remove)
    st = pb.gpu_step1()
    try:
        pb.gpu_l0_block(st, 0)
        assert st.status() == 0
        check_block(pb, st, cp, sparse)
    finally:
        st.close()
