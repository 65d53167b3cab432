"""The mixed-precision ridge solver (csrc/chol_mixed.cu + csrc/tf32_gemm.cu): 3xTF32 wgmma factorisation / inverse +
FP64 iterative refinement, against numpy's FP64 solve; its convergence flag; and the FP64 fallback of the level-0 path.

What the reference computes here: beta = V (D + lambda I)^-1 V^T (GtY - GtY_f), src/Step1_Models.cpp:484-494."""
import os

import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu


def _systems(n, K, P, seed, cond=50.0, n_real=None):
    """K SPD matrices with eigenvalues spread over [1, cond] * scale (identity on the padded rows, like the product path)."""
    rng = np.random.default_rng(seed)
    n_real = n_real or n
    Af = np.zeros((K, n, n)); b = np.zeros((K, P, n))
    for f in range(K):
        Q, _ = np.linalg.qr(rng.standard_normal((n_real, n_real)))
        ev = np.exp(rng.uniform(0, np.log(cond), size=n_real)) * 1000.0
        A = (Q * ev) @ Q.T
        Af[f, :n_real, :n_real] = (A + A.T) / 2
        for i in range(n_real, n):
            Af[f, i, i] = 1.0
        b[f, :, :n_real] = rng.standard_normal((P, n_real)) * 100.0
    return Af, b


@pytest.mark.parametrize("n,K,R,P,n_real", [(128, 2, 2, 3, 100), (256, 2, 3, 2, 256), (512, 1, 2, 10, 450), (1024, 2, 2, 10, 1000),
                                             (2048, 1, 2, 3, 1900)])   # the largest dimension (bsize 1025 .. 2048)
def test_mixed_solve_matches_numpy(n, K, R, P, n_real):
    from regenie_b200 import capi
    Af, b = _systems(n, K, P, seed=n + K, n_real=n_real)
    lam = np.array([5000.0, 50.0, 0.5])[:R]
    # default stopping rule (correction size OR its quadratic predictor, chol_mixed.cu): the accepted iterate is within
    # the 1e-9 class; the strict rule (negative tol = correction size only) runs one more correction and reaches round-off
    x, fail, Lt = capi.mixed_solve(Af, lam, b, steps=3, tol=1e-9, want_inverse=True)
    xs, fail_s, _ = capi.mixed_solve(Af, lam, b, steps=3, tol=-1e-9)
    assert fail == 0 and fail_s == 0
    for f in range(K):
        for r in range(R):
            A = Af[f] + lam[r] * np.eye(n)
            ref = np.linalg.solve(A, b[f].T).T
            err = np.abs(x[f * R + r] - ref).max() / np.abs(ref).max()
            assert err < 2e-10, (f, r, err)
            err_s = np.abs(xs[f * R + r] - ref).max() / np.abs(ref).max()
            assert err_s < 1e-11, (f, r, err_s)
            if n > 128:
                # the FP32-accurate factor the refinement solves with: tile (1, 0) of L vs numpy's Cholesky (diagnostic)
                Lref = np.linalg.cholesky(A)
                t = Lt[f * R + r][128:256, 0:128].astype(np.float64)
                assert np.abs(t - Lref[128:256, 0:128]).max() / np.abs(Lref[128:256, 0:128]).max() < 1e-4


def test_mixed_solve_flags_an_ill_conditioned_system():
    from regenie_b200 import capi
    Af, b = _systems(256, 1, 2, seed=3, cond=1e12)
    x, fail, _ = capi.mixed_solve(Af, np.array([1e-9]), b, steps=3, tol=1e-9)
    assert fail != 0


def test_level0_uses_the_mixed_solver_and_matches_the_oracle(tmp_path):
    pb = helpers.synthetic_problem(tmp_path, N=2051, M=260, P=3, C=3, bsize=130, miss=0.02, seed=5)
    st = pb.gpu_step1()
    for b in range(len(pb.blocks)):
        pb.gpu_l0_block(st, b)
    assert st.status() == 0
    mixed, fallbacks = st.solver_stats()
    assert mixed == len(pb.blocks) and fallbacks == 0
    for b in range(len(pb.blocks)):
        W_o = pb.oracle_l0(b)[0]
        for ph in range(3):
            W = st.fetch_W(b, ph)
            assert np.abs(W - W_o[ph]).max() / np.abs(W_o[ph]).max() < 1e-9
    st.close()


def test_level0_fp64_fallback_when_the_refinement_does_not_converge(tmp_path, monkeypatch):
    """An unreachable tolerance raises every block's flag: each block must be re-solved by the FP64 Cholesky from the
    lane's scratch (also when the lane is reused before anyone synchronises) and still match the oracle."""
    monkeypatch.setenv("RG_B200_MX_TOL", "1e-30")
    monkeypatch.setenv("RG_B200_LANES", "2")
    pb = helpers.synthetic_problem(tmp_path, N=1500, M=5 * 96, P=2, C=3, bsize=96, miss=0.02, seed=8)
    st = pb.gpu_step1()
    for b in range(len(pb.blocks)):
        pb.gpu_l0_block(st, b)
    assert st.status() == 0
    mixed, fallbacks = st.solver_stats()
    assert mixed == len(pb.blocks) and fallbacks == len(pb.blocks)
    for b in (0, 1, len(pb.blocks) - 1):
        W_o = pb.oracle_l0(b)[0]
        for ph in range(2):
            W = st.fetch_W(b, ph)
            assert np.abs(W - W_o[ph]).max() / np.abs(W_o[ph]).max() < 1e-9
    st.close()


def test_fp64_solver_is_still_selectable(tmp_path, monkeypatch):
    monkeypatch.setenv("RG_B200_SOLVER", "f64")
    pb = helpers.synthetic_problem(tmp_path, N=900, M=128, P=2, C=3, bsize=64, seed=2)
    st = pb.gpu_step1()
    pb.gpu_l0_block(st, 0)
    assert st.status() == 0
    assert st.solver_stats() == (0, 0)
    W_o = pb.oracle_l0(0)[0]
    assert np.abs(st.fetch_W(0, 0) - W_o[0]).max() / np.abs(W_o[0]).max() < 1e-9
    st.close()
