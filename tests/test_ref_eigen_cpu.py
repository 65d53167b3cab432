"""The compiled Eigen/OpenMP restatement (oracle/ref_eigen, built against the reference's vendored Eigen 3.4.0) and
the numpy oracle are two independent restatements of the same reference functions; they must agree.  This gives the
QT k-fold level-0 arithmetic (which has no golden vector in the reference's tests, SURVEY 8c) a second pin that uses
the reference's own SelfAdjointEigenSolver, and the Step-2 QT score test a second implementation.

The Eigen restatement needs the reference's sources to build, so its outputs on these seeded problems are stored under
tests/golden/ref_eigen/ (level-0 predictors at a fixed sample of 64 rows, Step-2 results in full)."""
import os

import numpy as np
import pytest

import helpers
from oracle import plink, step2

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_eigen")


def _rows(n):
    """The sample rows the stored level-0 predictors were taken at."""
    return np.sort(np.random.default_rng(0).choice(n, 64, replace=False))


@pytest.mark.parametrize("seed,N,M,bsize", [(3, 1200, 160, 80), (11, 2051, 130, 130)])
def test_level0_kfold_eigen_matches_numpy_oracle(tmp_path, seed, N, M, bsize):
    pb = helpers.synthetic_problem(tmp_path, N=N, M=M, P=3, C=3, bsize=bsize, miss=0.02, seed=seed)
    W_eigen = np.load(os.path.join(GOLD, "l0_kfold_seed%d.npy" % seed))
    assert W_eigen.shape[0] == len(pb.blocks)
    for b in range(len(pb.blocks)):
        W_np, _, _, _ = pb.oracle_l0(b)
        for ph in range(3):
            W_e = W_eigen[b, ph]
            want = W_np[ph][_rows(W_np[ph].shape[0])]
            err = np.abs(W_e - want).max() / np.abs(W_np[ph]).max()
            assert err < 1e-9, (b, ph, err)


def test_level0_eigen_is_thread_count_invariant_to_rounding(tmp_path):
    """The stored outputs of the Eigen restatement run with 1 and with 4 OpenMP threads (equal to 1e-10 when they were
    stored) both match the numpy oracle, which runs live here."""
    pb = helpers.synthetic_problem(tmp_path, N=900, M=64, P=2, C=3, bsize=64, seed=5)
    W1 = np.load(os.path.join(GOLD, "l0_threads1.npy"))
    W4 = np.load(os.path.join(GOLD, "l0_threads4.npy"))
    W_np, _, _, _ = pb.oracle_l0(0)
    for ph in range(len(W_np)):
        want = W_np[ph][_rows(W_np[ph].shape[0])]
        for W in (W1, W4):
            assert np.abs(W[ph] - want).max() / np.abs(W_np[ph]).max() < 1e-9, ph


def test_step2_qt_eigen_matches_numpy_oracle(tmp_path):
    pb = helpers.synthetic_problem(tmp_path, N=1500, M=120, P=3, C=3, bsize=120, miss=0.03, seed=9)
    pr = pb.prep
    rng = np.random.default_rng(1)
    res = rng.normal(size=(pb.n_file, 3)) * pr.mask
    res /= np.linalg.norm(res, axis=0) / np.sqrt(pr.neff - pr.ncov)
    scf = np.array([1.3, 0.7, 2.0])
    YtX = res.T @ pr.X
    out = np.load(os.path.join(GOLD, "s2_qt_seed9.npy"))
    assert out.shape[0] == pb.M
    n_checked = 0
    for i in range(pb.M):
        graw = plink.decode_bed(pb.packed[i:i + 1], pb.n_file)[0]
        vs = step2.variant_stats(graw, pr.in_analysis, pr.mask)
        if vs["ignored"]:
            assert out[i, 0] == -1
            continue
        sc = step2.score_qt(vs["g"], pr.X, res, pr.mask, pr.in_analysis, pr.n_analyzed, pr.ncov, scf, YtX, False)
        assert out[i, 0] == vs["af1"] and out[i, 1] == vs["ns1"] and out[i, 3] == sc["is_sparse"]
        for ph in range(3):
            q = out[i, 4 + 5 * ph: 9 + 5 * ph]
            assert q[0] == vs["af"][ph] and q[1] == vs["ns"][ph]
            np.testing.assert_allclose(q[2:], [sc["beta"][ph], sc["se"][ph], sc["chisq"][ph]], rtol=1e-9)
        n_checked += 1
    assert n_checked > 50
