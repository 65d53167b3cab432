"""The mixed-precision level-0 ridge solver (csrc/chol_mixed.cu) at every launch shape it selects and on LD-conditioned
systems, against an FP64 Cholesky solve refined with long-double residuals.

MixedSolver::solve picks its kernels from n, P, R and K:
  * the right-hand sides go in chunks of rhs_chunk(n) = 12 up to n = 1024 and 6 at n = 2048;
  * a chunk of np <= 10 vectors runs mx_trisolve_kernel<10>, np = 11..12 runs <12>;
  * the residual pass is mx_residual_fused_kernel when R * np <= 64, else the per-system mx_residual_kernel<10> / <12>.
_launches() restates those rules; every test names the kernels its shapes run.

Stopping-rule contract: a solve that leaves the fallback flag clear has every system within 2 * tol of the exact
solution (relative to the system's largest |x|), whatever its conditioning.  The level-0 path relies on it: a clear flag
means the block is not re-solved in FP64.
"""
import numpy as np
import pytest
import scipy.linalg

import helpers
from oracle import prep
from regenie_b200 import synth

gpu = pytest.mark.gpu
LD = np.longdouble
STEPS = 3                  # refinement steps of the level-0 path (kMxSteps, rg_api.cu)
MAX_STEPS = 6              # kMxMaxSteps


def _rhs_chunk(n):
    return max(1, min(12, 98304 // (8 * n)))


def _launches(n, P, R):
    """[(np, trisolve kernel, residual kernel)] per right-hand-side chunk, as MixedSolver::solve selects them."""
    out = []
    pc = _rhs_chunk(n)
    for p0 in range(0, P, pc):
        m = min(pc, P - p0)
        res = "fused" if R * m <= 64 else "residual<%d>" % (10 if m <= 10 else 12)
        out.append((m, "trisolve<%d>" % (10 if m <= 10 else 12), res))
    return out


def _lam_grid(M, R):
    """Level-0 ridge values lambda = M (1 - h) / h over the h grid of R values (src/Regenie.cpp, src/Data.cpp)."""
    h = prep.set_ridge_params(R)
    return M * (1 - h) / h


def _spectral(n, K, P, seed, lo, hi):
    """K SPD matrices Q diag(ev) Q^T with ev log-uniform on [lo, hi] (both ends included), and right-hand sides."""
    rng = np.random.default_rng(seed)
    Af = np.empty((K, n, n))
    ev = np.exp(rng.uniform(np.log(lo), np.log(hi), size=(K, n)))
    ev[:, 0], ev[:, 1] = lo, hi
    for f in range(K):
        Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
        A = (Q * ev[f]) @ Q.T
        Af[f] = (A + A.T) / 2
    b = rng.standard_normal((K, P, n)) * 100.0
    return Af, b, ev


def _ld_genotypes(rng, N, n_snp, cluster, redraw):
    """n_snp hard calls [n_snp, N] in clusters of `cluster` SNPs: a base SNP and copies of it with a fraction `redraw`
    (scalar or per copy) of the calls drawn again from the base's allele frequency."""
    g = np.empty((n_snp, N), dtype=np.uint8)
    redraw = np.broadcast_to(np.asarray(redraw, dtype=np.float64), (n_snp,))
    for c0 in range(0, n_snp, cluster):
        maf = rng.uniform(0.05, 0.5)
        base = rng.binomial(2, maf, size=N).astype(np.uint8)
        for i in range(c0, min(c0 + cluster, n_snp)):
            g[i] = base
            if i > c0:
                sel = rng.random(N) < redraw[i]
                g[i, sel] = rng.binomial(2, maf, size=int(sel.sum()))
    return g


def _ld_gram(n, K, P, seed, redraw, n_nominal, cluster, N):
    """Fold Grams of a standardised genotype block with LD clusters, rows scaled to norm^2 = n_nominal (oracle/step1.py
    scales to N - C), and right-hand sides G y of a random trait.  Returns (Af [K, n, n], b [K, P, n], eigenvalues)."""
    rng = np.random.default_rng(seed)
    g = _ld_genotypes(rng, N, n, cluster, redraw).astype(np.float64)
    g -= g.mean(axis=1, keepdims=True)
    g *= np.sqrt(n_nominal) / np.linalg.norm(g, axis=1, keepdims=True)
    y = rng.standard_normal((N, P))
    folds = np.array_split(np.arange(N), K + 1)          # fold f's system leaves out fold f (the last chunk is shared)
    Af, b, ev = np.empty((K, n, n)), np.empty((K, P, n)), []
    for f in range(K):
        keep = np.setdiff1d(np.arange(N), folds[f])
        G = g[:, keep]
        A = G @ G.T
        Af[f] = (A + A.T) / 2
        b[f] = (G @ y[keep]).T
        ev.append(np.linalg.eigvalsh(Af[f]))
    return Af, b, np.array(ev)


def _reference(Af, lam, b):
    """x [K*R, P, n] of (Af[f] + lam[r] I) x = b[f]: FP64 Cholesky, then corrections from residuals computed in long
    double until the correction is below 1e-14 of max |x| or stops shrinking.  A long-double residual carries an error
    of about kappa * 1e-19 relative to x, so at kappa = 1e7 the corrections level off near 1e-13; anything above 1e-12
    (far below every tolerance checked here) is refused."""
    K, n, _ = Af.shape
    R, P = len(lam), b.shape[1]
    x = np.empty((K * R, P, n))
    for f in range(K):
        AL = Af[f].astype(LD)
        bL = b[f].T.astype(LD)
        for r in range(R):
            c = scipy.linalg.cho_factor(Af[f] + lam[r] * np.eye(n), lower=True)
            xr = scipy.linalg.cho_solve(c, b[f].T)
            prev = np.inf
            for _ in range(30):
                xl = xr.astype(LD)
                res = bL - AL @ xl - LD(lam[r]) * xl
                dx = scipy.linalg.cho_solve(c, res.astype(np.float64))
                xr = xr + dx
                d = np.abs(dx).max() / np.abs(xr).max()
                if d <= 1e-14 or d > 0.5 * prev:
                    break
                prev = d
            assert d <= 1e-12, "reference refinement did not converge (fold %d, lambda %g): %g" % (f, lam[r], d)
            x[f * R + r] = xr.T
    return x


def _err(x, ref):
    """Per-system max |x - ref| / max |ref| (inf where x is not finite)."""
    e = np.abs(x - ref).reshape(len(x), -1).max(axis=1) / np.abs(ref).reshape(len(ref), -1).max(axis=1)
    return np.where(np.isfinite(e), e, np.inf)


def _forced(Af, lam, b, steps):
    """x_1 .. x_steps: the iterates after s corrections, every system running all s of them (tol = -1e-30)."""
    from regenie_b200 import capi
    xs = []
    for s in range(1, steps + 1):
        x, _, _ = capi.mixed_solve(Af, lam, b, steps=s, tol=-1e-30)
        xs.append(x)
    return xs


def _accepted_step(x, xs):
    """Per system: the s (1-based) whose forced iterate x is bit-identical to, or 0 if none is."""
    out = np.zeros(len(x), dtype=int)
    for m in range(len(x)):
        for s, xf in enumerate(xs, start=1):
            if np.array_equal(x[m], xf[m]):
                out[m] = s
                break
    return out


# ------------------------------------------------------------------------------------------------ (a) launch shapes
SHAPES = [  # n, P, R, K
    (1024, 12, 5, 2), (1024, 13, 5, 2), (1024, 25, 5, 2),   # one / two / three chunks, <12> then <10>, odd P
    (2048, 6, 2, 1), (2048, 7, 2, 1), (2048, 13, 2, 1),      # the 6-wide chunks at n = 2048
    (512, 10, 7, 2), (512, 9, 8, 2),                         # per-system residual<10> (R np = 70, 72)
    (256, 11, 6, 2), (256, 12, 6, 2),                        # per-system residual<12> (66, 72)
    (1024, 13, 6, 2),                                        # chunk 1 residual<12>, chunk 2 fused, in one solve
    (128, 3, 8, 16), (256, 3, 8, 16),                        # nmat = 128 systems
]


def test_launch_shapes_cover_every_kernel():
    """The shape matrix runs both substitution kernels and all three residual kernels, a solve that mixes the fused and
    the per-system residual, more than one chunk at n = 2048 and odd P (a padding row in Pp)."""
    seen = {k for n, P, R, _ in SHAPES for c in _launches(n, P, R) for k in c[1:]}
    assert seen == {"trisolve<10>", "trisolve<12>", "fused", "residual<10>", "residual<12>"}, seen
    assert _launches(1024, 13, 6) == [(12, "trisolve<12>", "residual<12>"), (1, "trisolve<10>", "fused")]
    assert [c[0] for c in _launches(2048, 13, 2)] == [6, 6, 1] and [c[0] for c in _launches(1024, 25, 5)] == [12, 12, 1]
    assert any(P % 2 for _, P, _, _ in SHAPES)


@gpu
@pytest.mark.parametrize("n,P,R,K", SHAPES, ids=["n%d-P%d-R%d-K%d" % s for s in SHAPES])
def test_mixed_solve_launch_shapes(n, P, R, K):
    from regenie_b200 import capi
    Af, b, _ = _spectral(n, K, P, seed=n + 31 * P + 7 * R + K, lo=1000.0, hi=50000.0)   # kappa <= 50
    lam = _lam_grid(1000, R)
    ref = _reference(Af, lam, b)
    x, fail, _ = capi.mixed_solve(Af, lam, b, steps=STEPS, tol=1e-9)
    xs, fail_s, _ = capi.mixed_solve(Af, lam, b, steps=STEPS, tol=-1e-9)
    kern = _launches(n, P, R)
    assert fail == 0 and fail_s == 0, (kern, fail, fail_s)
    err, err_s = _err(x, ref), _err(xs, ref)
    assert err.max() < 2e-10, (kern, err)
    assert err_s.max() < 1e-11, (kern, err_s)


@gpu
@pytest.mark.parametrize("steps", range(1, MAX_STEPS + 1))
def test_mixed_solve_every_step_count(steps):
    """n = 256, P = 4, R = 3, K = 2 with 1 .. kMxMaxSteps corrections: a clear flag means within 2 tol; from the
    level-0 step count on the flag is clear and the bounds of the shape matrix hold."""
    from regenie_b200 import capi
    Af, b, _ = _spectral(256, 2, 4, seed=256, lo=1000.0, hi=50000.0)
    lam = _lam_grid(1000, 3)
    ref = _reference(Af, lam, b)
    for tol, bound in ((1e-9, 2e-10), (-1e-9, 1e-11)):
        x, fail, _ = capi.mixed_solve(Af, lam, b, steps=steps, tol=tol)
        err = _err(x, ref)
        assert fail != 0 or err.max() <= 2 * abs(tol), (tol, fail, err)
        if steps >= STEPS:
            assert fail == 0 and err.max() < bound, (tol, fail, err)


@gpu
def test_mixed_solve_refusals_leave_the_next_call_working():
    from regenie_b200 import capi
    Af, b, _ = _spectral(256, 1, 2, seed=5, lo=1000.0, hi=50000.0)
    lam = np.array([10.0, 1000.0])
    ref = _reference(Af, lam, b)
    bad = [(np.zeros((1, 384, 384)), {}), (np.zeros((1, 100, 100)), {}),        # not 128 * 2^k
           (np.zeros((1, 4096, 4096)), {}),                                     # above 2048
           (Af, {"steps": 0}), (Af, {"steps": MAX_STEPS + 1})]                  # steps outside 1 .. kMxMaxSteps
    for A, kw in bad:
        with pytest.raises(capi.RgError):
            capi.mixed_solve(A, lam, np.zeros((1, 2, A.shape[1])), **kw)
        x, fail, _ = capi.mixed_solve(Af, lam, b, steps=STEPS, tol=1e-9)
        assert fail == 0 and _err(x, ref).max() < 2e-10, (A.shape, kw)


# ------------------------------------------------------------------------------------- (b) the stopping-rule contract
TOL = 1e-9


def _sweep_case(tag, Af, b, lam, kappa, steps=STEPS):
    """One batch: the default solve, the reference, the forced iterates.  Rows of (tag, kappa, rho, accepted step,
    error, flag) per system and whether the contract held."""
    from regenie_b200 import capi
    x, fail, _ = capi.mixed_solve(Af, lam, b, steps=steps, tol=TOL)
    ref = _reference(Af, lam, b)
    xs = _forced(Af, lam, b, steps)
    e = np.array([_err(xf, ref) for xf in xs])                      # [steps, nmat]
    with np.errstate(divide="ignore", invalid="ignore"):
        rho = np.where(e[0] > 1e-13, e[1] / e[0], np.nan)           # observed contraction of one correction
    err = _err(x, ref)
    acc = _accepted_step(x, xs)
    rows = [(tag, kappa[m], rho[m], acc[m], err[m], fail) for m in range(len(x))]
    return rows, fail != 0 or err.max() <= 2 * TOL


def _print_rows(rows):
    print("\n%-26s %10s %10s %5s %10s %5s" % ("case", "kappa", "rho", "step", "error", "flag"))
    for tag, k, r, a, e, f in rows:
        print("%-26s %10.3g %10.3g %5d %10.3g %5d" % (tag, k, r, a, e, f))


@gpu
@pytest.mark.parametrize("n", [512, 2048])
def test_stopping_rule_on_log_uniform_spectra(n):
    """kappa(A + lambda_min I) from 1e2 to 1e7 in half decades, spectra log-uniform, lambda from the level-0 grid (the
    other ridge values give smaller kappa).  Fallback flag clear => every system within 2 tol."""
    K, R, P = (2, 5, 4) if n == 512 else (1, 5, 4)
    seeds = (0, 1) if n == 512 else (0,)
    lam = _lam_grid(1000, R)                                        # lambda_min = 10.1
    rows, ok = [], []
    for seed in seeds:
        for e10 in np.arange(2.0, 7.01, 0.5):
            hi = 10.0 ** e10 * (1000.0 + lam.min())
            Af, b, ev = _spectral(n, K, P, seed=1000 * seed + int(10 * e10) + n, lo=1000.0, hi=hi)
            kappa = np.array([(ev[f].max() + l) / (ev[f].min() + l) for f in range(K) for l in lam])
            r, good = _sweep_case("spec n%d s%d 1e%.1f" % (n, seed, e10), Af, b, lam, kappa)
            rows += r
            ok.append(good)
    _print_rows(rows)
    bad = [t for t in rows if t[5] == 0 and t[4] > 2 * TOL]
    assert all(ok), "flag clear with errors above 2 tol: %s" % bad


@gpu
@pytest.mark.parametrize("n", [512, 2048])
def test_stopping_rule_on_ld_grams(n):
    """Fold Grams of genotype blocks with LD clusters of 32 SNPs (a base and copies with a fraction of the calls
    redrawn), rows scaled like 10^6 samples.  kappa ~ 10^6 * (cluster size) / lambda_min: the lambda grid is that of a
    20 000-SNP run (lambda_min = 202) or of a run made of this block alone (lambda_min = 0.0101 n), and the redrawn
    fraction sets the smallest eigenvalues.  Fallback flag clear => every system within 2 tol."""
    K, R, P = (2, 5, 4) if n == 512 else (1, 5, 4)
    rows, ok = [], []
    for seed, M in ((0, 20000), (1, n)):
        lam = _lam_grid(M, R)
        for redraw in (0.5, 0.2, 0.1, 0.05, 0.02, 0.01, 0.005, 0.002) if n == 512 else (0.5, 0.1, 0.02, 0.005, 0.002):
            Af, b, ev = _ld_gram(n, K, P, seed=7 * seed + n, redraw=redraw, n_nominal=1e6, cluster=32, N=4 * n)
            kappa = np.array([(ev[f].max() + l) / (ev[f].min() + l) for f in range(K) for l in lam])
            r, good = _sweep_case("ld n%d M%d %.3f" % (n, M, redraw), Af, b, lam, kappa)
            rows += r
            ok.append(good)
    _print_rows(rows)
    kap = np.array([t[1] for t in rows])
    assert kap.min() < 1e3 and kap.max() > 5e5, (kap.min(), kap.max())
    bad = [t for t in rows if t[5] == 0 and t[4] > 2 * TOL]
    assert all(ok), "flag clear with errors above 2 tol: %s" % bad


# ------------------------------------------------------------------------------------------------- (c) skip logic
@gpu
@pytest.mark.parametrize("n,P,R,K", [(512, 4, 5, 2), (512, 10, 8, 2), (256, 12, 6, 2)],
                         ids=["fused", "residual10", "residual12"])
def test_finished_systems_are_kept_unchanged(n, P, R, K):
    """Systems that finish at different steps: every x of the default solve is bit-identical to the forced iterate x_s of
    the step s it was accepted at, so a finished system is neither lost nor changed by the later launches, including
    folds where only some systems have finished (the fused residual pass still runs for them) and folds that are
    entirely done (it returns early)."""
    from regenie_b200 import capi
    lam = _lam_grid(1000, R)
    steps = MAX_STEPS
    # fold 0: kappa <= 100 for every lambda (all finish early); fold 1: eigenvalues from 1 to 3e5, so kappa runs from
    # ~3 at the largest lambda to ~3e4 at the smallest (finishing at different steps)
    A0, b0, _ = _spectral(n, 1, P, seed=n + P, lo=1000.0, hi=1e5)
    A1, b1, _ = _spectral(n, K - 1, P, seed=n + P + 1, lo=1.0, hi=3e5)
    Af, b = np.concatenate([A0, A1]), np.concatenate([b0, b1])
    x, fail, _ = capi.mixed_solve(Af, lam, b, steps=steps, tol=TOL)
    xs = _forced(Af, lam, b, steps)
    acc = _accepted_step(x, xs)
    print("\n%s: accepted steps per system %s (fold-major, R = %d), flag %d" % (_launches(n, P, R), acc.tolist(), R, fail))
    assert (acc > 0).all(), acc
    per_fold = acc.reshape(K, R)
    assert len(set(acc.tolist())) >= 2, "all systems finished at the same step: the batch does not exercise the skips"
    assert any(len(set(f.tolist())) >= 2 for f in per_fold), "no fold with finished and unfinished systems"
    assert fail == 0
    ref = _reference(Af, lam, b)
    assert _err(x, ref).max() <= 2 * TOL


# --------------------------------------------------------------------------------------------------------- (d) flag
@gpu
def test_flag_on_a_hopeless_system_among_good_ones():
    """Fold 1 has eigenvalues down to 1e-3 and up to 1e9: with lambda = 1e-3 its system has kappa ~ 5e11.  The flag must
    be raised, and the good systems of the same solve must still be right."""
    from regenie_b200 import capi
    A0, b0, _ = _spectral(512, 1, 4, seed=11, lo=1000.0, hi=50000.0)
    A1, b1, _ = _spectral(512, 1, 4, seed=12, lo=1e-3, hi=1e9)
    Af, b = np.concatenate([A0, A1]), np.concatenate([b0, b1])
    lam = np.array([1e-3, 1e9, 1e10])                      # fold 1: kappa 5e11, 2, 1.1
    x, fail, _ = capi.mixed_solve(Af, lam, b, steps=STEPS, tol=TOL)
    assert fail != 0
    ref = _reference(Af[:1], lam, b[:1])
    assert _err(x[:3], ref).max() <= 2 * TOL
    ref1 = _reference(Af[1:], lam[1:], b[1:])
    assert _err(x[4:6], ref1).max() <= 2 * TOL


@gpu
def test_flag_on_a_nan_in_one_fold():
    from regenie_b200 import capi
    Af, b, _ = _spectral(256, 2, 3, seed=13, lo=1000.0, hi=50000.0)
    lam = _lam_grid(1000, 3)
    ref = _reference(Af[:1], lam, b[:1])
    Af[1, 5, 7] = Af[1, 7, 5] = np.nan
    x, fail, _ = capi.mixed_solve(Af, lam, b, steps=STEPS, tol=TOL)
    assert fail != 0
    assert _err(x[:3], ref).max() <= 2 * TOL             # the other fold's systems are untouched by the NaN
    Af[1, 5, 7] = Af[1, 7, 5] = 0.0
    x, fail, _ = capi.mixed_solve(Af, lam, b, steps=STEPS, tol=TOL)
    assert fail == 0 and _err(x, _reference(Af, lam, b)).max() <= 2 * TOL


# ------------------------------------------------------------------------------------------- 2. level 0 end to end
def _fileset(d, g, chrom_sizes, P, C, seed, bsize, R, K=5):
    """PLINK fileset of hard calls g [M, N] whose chromosome c holds chrom_sizes[c - 1] SNPs, a Problem over it with R
    ridge values from the level-0 grid."""
    Y, cov, na = synth.phenotypes(g, P, C, seed=seed, na_frac=0.03)
    N = g.shape[1]
    prefix = helpers.write_fileset(str(d), g, Y, cov, na, drop_pheno={5, 77, N - 3}, drop_cov={11})
    chrom = np.repeat(np.arange(1, len(chrom_sizes) + 1), chrom_sizes)
    with open(prefix + ".bim", "w") as fh:
        for i in range(g.shape[0]):
            fh.write("%d rs%d 0 %d A G\n" % (chrom[i], i, 1000 + i))
    pb = helpers.Problem(prefix, str(d) + "/pheno.txt", str(d) + "/covar.txt", bsize, K=K)
    pb.lam = _lam_grid(pb.M, R)
    return pb


def _fold_kappa(pb, b):
    """kappa(A_f + lambda_min I) of every fold system of block b (the oracle's Gram)."""
    Gt = pb.oracle_l0(b)[3]
    starts = np.concatenate([[0], np.cumsum(pb.fold_sizes)])
    GG = Gt @ Gt.T
    out = []
    for f in range(len(pb.fold_sizes)):
        Gf = Gt[:, starts[f]:starts[f + 1]]
        d = np.linalg.eigvalsh(GG - Gf @ Gf.T)
        out.append((d.max() + pb.lam.min()) / (max(d.min(), 0.0) + pb.lam.min()))
    return np.array(out)


def _run_blocks(pb, st, expect_fallback):
    """Every block through level 0, solver_stats() after each, W against the oracle at 1e-9."""
    for b in range(len(pb.blocks)):
        before = st.solver_stats()
        pb.gpu_l0_block(st, b)
        assert st.status() == 0
        after = st.solver_stats()
        fb = expect_fallback(b)
        if fb is None:
            print("block %d: solver_stats %s -> %s" % (b, before, after))
            assert after[0] == before[0] + 1 and after[1] - before[1] in (0, 1)
        else:
            assert after == (before[0] + 1, before[1] + int(fb)), (b, before, after)
        W_o = pb.oracle_l0(b)[0]
        for ph in range(len(W_o)):
            W = st.fetch_W(b, ph)
            assert np.abs(W - W_o[ph]).max() / np.abs(W_o[ph]).max() < 1e-9, (b, ph)


@gpu
@pytest.mark.parametrize("N,bsize,P,R", [(2000, 500, 10, 8), (3000, 1000, 12, 6), (4000, 1500, 7, 5)],
                         ids=["residual10", "residual12", "n2048-two-chunks"])
def test_level0_blocks_at_the_solver_shapes(tmp_path, monkeypatch, N, bsize, P, R):
    """bsize 500 (n = 512), P = 10, R = 8: residual<10> from the level-0 assembler (first_col_ready);
    bsize 1000 (n = 1024), P = 12, R = 6: residual<12>;  bsize 1500 (n = 2048), P = 7: two chunks of 6 + 1.
    W against the oracle and, for the first shape, against the FP64 Cholesky route on the same handle inputs."""
    from regenie_b200 import capi
    n = 128
    while n < bsize:
        n *= 2
    print(_launches(n, P, R))
    g = synth.genotypes(N, bsize, seed=bsize + P, miss=0.02)
    pb = _fileset(tmp_path, g, [bsize], P, 3, bsize + P, bsize, R)
    assert [blk[2] for blk in pb.blocks] == [bsize] and len(pb.lam) == R
    st = pb.gpu_step1()
    assert st.R == R
    _run_blocks(pb, st, lambda b: False)
    W_mx = [st.fetch_W(0, ph) for ph in range(P)]
    st.close()
    if bsize == 500:
        monkeypatch.setenv("RG_B200_SOLVER", "f64")
        st = pb.gpu_step1()
        pb.gpu_l0_block(st, 0)
        assert st.status() == 0 and st.solver_stats() == (0, 0)
        for ph in range(P):
            W = st.fetch_W(0, ph)
            assert np.abs(W_mx[ph] - W).max() / np.abs(W).max() < 1e-9, ph
        st.close()


@gpu
def test_level0_ld_blocks_fall_back_only_when_they_must(tmp_path):
    """50 000 samples, three 256-SNP blocks as the whole run (M = 768, lambda_min = 7.8): independent SNPs; 16-SNP
    clusters at r^2 ~ 0.9 - 0.99; one base SNP and 255 copies that differ from it in two calls each (kappa > 1e6).
    The near-duplicate block must fall back to FP64, the independent one must not; every W matches the oracle."""
    rng = np.random.default_rng(77)
    N, bs = 50000, 256
    g_ind = synth.genotypes(N, bs, seed=78, miss=0.0)
    g_ld = _ld_genotypes(rng, N, bs, 16, rng.uniform(0.005, 0.05, size=bs))
    maf = 0.3
    base = rng.binomial(2, maf, size=N).astype(np.uint8)
    g_dup = np.repeat(base[None, :], bs, axis=0)
    for i in range(1, bs):
        idx = rng.choice(N, size=2, replace=False)
        g_dup[i, idx] = (g_dup[i, idx] + 1) % 3
    g = np.concatenate([g_ind, g_ld, g_dup])
    pb = _fileset(tmp_path, g, [bs, bs, bs], 2, 3, 79, bs, 5)
    assert [blk[2] for blk in pb.blocks] == [bs] * 3 and abs(pb.lam.min() - 768 * 0.01 / 0.99) < 1e-9
    kap = [_fold_kappa(pb, b).max() for b in range(3)]
    print("\nlargest kappa(A_f + lambda_min I) per block: independent %.3g, 16-SNP clusters %.3g, near-duplicates %.3g" % tuple(kap))
    assert kap[2] > 1e6 and kap[0] < 1e3
    st = pb.gpu_step1()
    _run_blocks(pb, st, lambda b: {0: False, 1: None, 2: True}[b])
    st.close()
