"""The factor of the mixed-precision ridge solver as it is stored (csrc/chol_mixed.cu): one FP32 matrix per system with
L in the lower triangle, L_kk on the diagonal tiles and the transposes of the off-diagonal tiles above them. The TF32
hi/lo pairs that the tensor cores multiply exist only inside the GEMM tiles (csrc/tf32_gemm.cu), so what these tests
see is everything the solver keeps."""
import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu

T = 128


def _spd(n, K, P, seed):
    rng = np.random.default_rng(seed)
    Af = np.zeros((K, n, n)); b = np.zeros((K, P, n))
    for f in range(K):
        Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
        ev = np.exp(rng.uniform(0, np.log(50.0), size=n)) * 1000.0
        A = (Q * ev) @ Q.T
        Af[f] = (A + A.T) / 2
        b[f] = rng.standard_normal((P, n)) * 100.0
    return Af, b


@pytest.mark.parametrize("n,K,R", [(128, 2, 2), (256, 1, 3), (1024, 2, 2), (2048, 1, 2)])
def test_stored_factor_is_the_cholesky_factor_with_mirrored_tiles(n, K, R):
    from regenie_b200 import capi
    Af, b = _spd(n, K, 2, seed=7 * n + K)
    lam = np.array([5000.0, 50.0, 0.5])[:R]
    x, fail, F = capi.mixed_solve(Af, lam, b, steps=3, tol=1e-9, want_inverse=True)
    assert fail == 0
    nt = n // T
    for f in range(K):
        for r in range(R):
            Fm = F[f * R + r]
            Lref = np.linalg.cholesky(Af[f] + lam[r] * np.eye(n))
            # whole lower triangle, diagonal tiles included, at an FP32 bound (3xTF32 products, FP32 accumulation)
            low = np.tril(Fm).astype(np.float64)
            assert np.abs(low - Lref).max() / np.abs(Lref).max() < 2e-5, (f, r)
            for k in range(nt):
                d = Fm[k * T:(k + 1) * T, k * T:(k + 1) * T]
                assert not np.triu(d, 1).any(), (f, r, k)               # diagonal tiles: zeros above the diagonal
                for i in range(k + 1, nt):                               # what the backward substitution streams
                    assert np.array_equal(Fm[k * T:(k + 1) * T, i * T:(i + 1) * T],
                                          Fm[i * T:(i + 1) * T, k * T:(k + 1) * T].T), (f, r, i, k)
    x2, fail2, F2 = capi.mixed_solve(Af, lam, b, steps=3, tol=1e-9, want_inverse=True)
    assert fail2 == 0
    assert np.array_equal(F.view(np.uint32), F2.view(np.uint32))
    assert np.array_equal(x.view(np.uint64), x2.view(np.uint64))


def test_level0_blocks_of_dimension_1024_stay_on_the_mixed_solver(tmp_path):
    pb = helpers.synthetic_problem(tmp_path, N=1500, M=2 * 600, P=3, C=3, bsize=600, miss=0.02, seed=11)
    st = pb.gpu_step1()
    for blk in range(len(pb.blocks)):
        pb.gpu_l0_block(st, blk)
    assert st.status() == 0
    mixed, fallbacks = st.solver_stats()
    assert mixed == len(pb.blocks) and fallbacks == 0
    W_o = pb.oracle_l0(1)[0]
    for ph in range(3):
        W = st.fetch_W(1, ph)
        assert np.abs(W - W_o[ph]).max() / np.abs(W_o[ph]).max() < 1e-9
    st.close()
