"""Numerical study for DESIGN.md section 8 (1): can the level-0 ridge systems (A_-f + lambda_j I) beta = b be factorised in
reduced precision on the tensor cores and polished by FP64 iterative refinement?

Synthetic block as bench.py builds it (MAF ~ U(0.01, 0.5), 1 % missing, mean-imputed, residualised on C = 3 covariates,
unit variance), N samples, bs SNPs, K = 5 folds, the reference's lambda grid M (1 - h) / h, h in {0.01, .25, .5, .75, .99}.
For every (fold, lambda) system: condition number, and the number of refinement steps needed to reach the FP64 Cholesky
solution to 1e-12 (relative, max norm) when the factor is computed in
  fp32          plain single precision (what an FP32-accumulating tensor-core path with split operands delivers)
  tf32          operands rounded to 10 mantissa bits before an fp32 factorisation (one-pass TF32 MMA)
CPU only (numpy); prints a table.
"""
import sys

import numpy as np


def tf32_round(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    u = a.view(np.uint32)
    u = (u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)
    return u.view(np.float32)


def chol_solve(L, b):
    from scipy.linalg import solve_triangular
    y = solve_triangular(L, b, lower=True)
    return solve_triangular(L.T, y, lower=False)


def main():
    N = int(sys.argv[1]) if len(sys.argv) > 1 else 100000
    bs = int(sys.argv[2]) if len(sys.argv) > 2 else 1000
    M = int(sys.argv[3]) if len(sys.argv) > 3 else 50000
    P, K, C = 10, 5, 3
    rng = np.random.default_rng(20260924)
    maf = rng.uniform(0.01, 0.5, bs)
    G = rng.binomial(2, maf[:, None], (bs, N)).astype(np.float64)
    # a block of LD: neighbouring SNPs share haplotypes
    for j in range(1, bs):
        if rng.random() < 0.6:
            keep = rng.random(N) < 0.8
            G[j, keep] = G[j - 1, keep]
    miss = rng.random((bs, N)) < 0.01
    mu = (G * ~miss).sum(1) / (~miss).sum(1)
    G = np.where(miss, mu[:, None], G)
    X = np.linalg.qr(np.hstack([np.ones((N, 1)), rng.normal(size=(N, C - 1))]))[0]
    G -= (G @ X) @ X.T
    G /= np.linalg.norm(G, axis=1, keepdims=True) / np.sqrt(N - C)
    Y = rng.normal(size=(N, P))
    Y -= X @ (X.T @ Y)
    Y /= Y.std(0)
    folds = np.array_split(np.arange(N), K)
    A = G @ G.T
    b = G @ Y
    h = np.array([0.01, 0.25, 0.5, 0.75, 0.99])
    lam = M * (1 - h) / h
    print("N=%d bs=%d M=%d; eigenvalues of G G^T: min %.3g max %.3g" % ((N, bs, M) + tuple(np.linalg.eigvalsh(A)[[0, -1]])))
    print("%4s %10s %9s | %-22s | %-22s" % ("fold", "lambda", "cond", "fp32: err0, steps", "tf32: err0, steps"))
    worst = {"fp32": 0, "tf32": 0}
    for f in range(K):
        Gf = G[:, folds[f]]
        Af = A - Gf @ Gf.T
        bf = b - Gf @ Y[folds[f]]
        for lj in lam:
            S = Af + lj * np.eye(bs)
            ev = np.linalg.eigvalsh(S)
            x_ref = chol_solve(np.linalg.cholesky(S), bf)
            row = "%4d %10.4g %9.3g |" % (f, lj, ev[-1] / ev[0])
            for kind in ("fp32", "tf32"):
                S32 = S.astype(np.float32) if kind == "fp32" else tf32_round(S)
                try:
                    L = np.linalg.cholesky(S32).astype(np.float64)
                except np.linalg.LinAlgError:
                    row += " %-22s |" % "not positive definite"
                    worst[kind] = 99
                    continue
                x = chol_solve(L, bf)
                err0 = np.abs(x - x_ref).max() / np.abs(x_ref).max()
                steps, err = 0, err0
                while err > 1e-12 and steps < 30:
                    r = bf - S @ x
                    x = x + chol_solve(L, r)
                    err = np.abs(x - x_ref).max() / np.abs(x_ref).max()
                    steps += 1
                worst[kind] = max(worst[kind], steps)
                row += " %8.1e, %2d steps     |" % (err0, steps)
            print(row)
    print("worst case refinement steps:", worst)


if __name__ == "__main__":
    main()
