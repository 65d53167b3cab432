"""Level-0 kernel paths that the block size and the fold length select, each against a plain reference.

Level 0 picks its kernels from the shape of the input:
  * ridge solver: the mixed-precision solver of dimension n = 128 * 2^k for bsize <= 2048, the FP64 Cholesky beyond;
  * prediction: the INT8 tensor-core kernel while 2 * rows_p <= 4096, the FP64 CUDA-core kernel beyond (bsize > 2048);
  * statistics: tensor-core digit tiles while 30 * (longest padded fold) < 2^24, FP64 reductions beyond (or with
    RG_B200_STATS=f64), with 1, 2 or 3 groups of 14 (X | Y) columns.
Every test asserts through the "paths" hook and solver_stats() which kernels ran, and compares the level-0 predictors
with the numpy oracle at 1e-9 relative.  The raw predictions and the statistics are also recomputed in long double
from the kernel's own inputs and held to the error bound of the kernel's arithmetic.
"""
import numpy as np
import pytest

import helpers
from oracle import plink, step1
from regenie_b200 import hostprep, synth

pytestmark = pytest.mark.gpu
TOL = 1e-9
U = 2.0 ** -53              # unit round-off of FP64
LD = np.longdouble


def rel(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def _fileset(d, N, chrom_sizes, P, C, miss, seed, bsize, K=5):
    """Synthetic PLINK fileset whose chromosome c holds chrom_sizes[c - 1] consecutive SNPs (so the blocks of a
    chromosome are bsize, ..., remainder), with a few samples lacking a phenotype or a covariate."""
    M = int(sum(chrom_sizes))
    g = synth.genotypes(N, M, seed=seed, miss=miss)
    Y, cov, na = synth.phenotypes(g, P, C, seed=seed, na_frac=0.03)
    prefix = helpers.write_fileset(str(d), g, Y, cov, na, drop_pheno={5, 77, N - 3}, drop_cov={11})
    chrom = np.repeat(np.arange(1, len(chrom_sizes) + 1), chrom_sizes)
    with open(prefix + ".bim", "w") as fh:
        for i in range(M):
            fh.write("%d rs%d 0 %d A G\n" % (chrom[i], i, 1000 + i))
    return helpers.Problem(prefix, str(d) + "/pheno.txt", str(d) + "/covar.txt", bsize, K=K)


def _calls(pb, b):
    """G0 (dosage, 0 where missing) and Miss planes of block b over the kept samples, zero outside the analysis."""
    _, s, bs = pb.blocks[b]
    g = plink.decode_bed(pb.packed[s:s + bs], pb.n_file, keep=pb.keep)
    g = np.where(pb.prep.in_analysis[None, :], g, 0.0)
    mi = g == plink.MISSING_G
    return np.where(mi, 0, g).astype(np.int8), mi.astype(np.int8)


def _hooks(st):
    """The level-0 intermediates of the handle's last block (rg_debug_fetch)."""
    Npad, rp, nC, _, _, K, cpp, _ = [int(x) for x in st.debug("dims", np.int64, 8)]
    P, R, C = st.P, st.R, st.C
    gam = st.debug("gam", np.float64, K * rp * (R * P + 64))
    Qp = gam.size // (K * rp)
    return dict(Npad=Npad, rp=rp, nC=nC, K=K, cpp=cpp,
                paths=tuple(int(x) for x in st.debug("paths", np.int64, 3)),
                gam=gam.reshape(K, rp, Qp), gmu=st.debug("gmu", np.float64, K * rp * Qp).reshape(K, rp, Qp),
                cvec=st.debug("cvec", np.float64, K * Qp * C).reshape(K, Qp, C),
                wraw=st.debug("wraw", np.float64, P * R * Npad).reshape(P, R, Npad),
                pad_of=st.debug("pad_of", np.int32, st.N),
                cnt=st.debug("cnt_fold", np.int32, K * rp * 4).reshape(K, rp, 4),
                sum=st.debug("sum_fold", np.float64, K * rp * 2 * cpp).reshape(K, rp, 2, cpp))


def _ld_matmul(A, B):
    """A [m, n] (small integers) @ B [n, k] in long double, a few rows of A at a time."""
    Bl = B.astype(LD)
    step = max(1, 4_000_000 // max(1, A.shape[1]))
    return np.concatenate([A[r:r + step].astype(LD) @ Bl for r in range(0, A.shape[0], step)], axis=0)


def _limb_value(v, s, nl):
    """gamma rebuilt from the first nl balanced radix-254 digits of v / s * 127 (the INT8 kernel's split)."""
    x = v / s * 127.0
    acc = np.zeros_like(v)
    for l in range(nl):
        d = np.rint(x)
        acc += d * 254.0 ** -l
        x = (x - d) * 254.0
    return s / 127.0 * acc


def _excess(got, ref, bound):
    """Largest |got - ref| / bound (> 1: outside the bound)."""
    err = np.abs(got.astype(LD) - ref).astype(np.float64)
    return float(np.max(np.where(err > 0, err / np.maximum(bound, 1e-300), 0.0)))


def check_raw_predictions(hk, g0, mi, X, mask, fold_sizes, power=False):
    """Raw (unstandardised) predictions of the last block against a long-double recomputation from the kernel's inputs:
        raw[s, q] = (sum_i gam[f,i,q] g0(i,s) + gmu[f,i,q] miss(i,s) - X[s] . cvec[f,q]) * mask[s, p],  q = r P + p,
    f = fold of sample s.  INT8 kernel:  |err| <= s_q 254^-5 sum_i (g0 + miss) + 64 u sum|terms|, s_q = the largest
    |gam|, |gmu| of the column over the fold's rows (five limbs, the last rounded to within 1/2 of (s_q/127) 254^-4).
    FP64 kernel: |err| <= (2 bs + C + 2) u sum|terms| (sequential FMAs).
    power=True also shows that the bound rejects a kernel that dropped its last limb or misplaced a sample or an output."""
    bs = g0.shape[0]
    P, R, Npad = hk["wraw"].shape
    K, C, N, Q = hk["K"], X.shape[1], g0.shape[1], R * P
    i8 = hk["paths"][1] == 1
    pad = np.ones(Npad, dtype=bool)
    pad[hk["pad_of"]] = False
    assert not hk["wraw"][:, :, pad].any(), "layout padding rows of the raw predictions are not zero"
    got = hk["wraw"][:, :, hk["pad_of"]].transpose(2, 1, 0).reshape(N, Q)
    starts = np.concatenate([[0], np.cumsum(fold_sizes)])
    ref = np.zeros((N, Q), dtype=LD)
    bound = np.zeros((N, Q))
    drop = np.zeros((N, Q))
    for f in range(K):
        sl = slice(starts[f], starts[f + 1])
        gam, gmu, cv = hk["gam"][f, :bs, :Q], hk["gmu"][f, :bs, :Q], hk["cvec"][f, :Q]
        A0, Am = g0[:, sl].T.astype(np.float64), mi[:, sl].T.astype(np.float64)
        ref[sl] = _ld_matmul(g0[:, sl].T, gam) + _ld_matmul(mi[:, sl].T, gmu) - X[sl].astype(LD) @ cv.T.astype(LD)
        mag = A0 @ np.abs(gam) + Am @ np.abs(gmu) + np.abs(X[sl]) @ np.abs(cv.T)
        if i8:
            s_q = np.maximum(np.abs(gam).max(axis=0), np.abs(gmu).max(axis=0))
            s_q[s_q == 0] = 1.0
            bound[sl] = s_q[None, :] * 254.0 ** -5 * (A0 + Am).sum(axis=1)[:, None] + 64 * U * mag
            if power:
                drop[sl] = A0 @ (_limb_value(gam, s_q, 4) - gam) + Am @ (_limb_value(gmu, s_q, 4) - gmu)
        else:
            bound[sl] = (2 * bs + C + 2) * U * mag
    m = mask[:, np.arange(Q) % P].astype(np.float64)
    ref *= m
    bound *= m
    ex = _excess(got, ref, bound)
    assert ex <= 1.0, "raw predictions (%s, bs=%d) exceed the error bound %.3g-fold" % ("INT8" if i8 else "FP64", bs, ex)
    if power:
        assert _excess(np.roll(got, 1, axis=0), ref, bound) > 1.0, "a misplaced sample would pass"
        assert _excess(np.roll(got, 1, axis=1), ref, bound) > 1.0, "a misplaced output would pass"
        if i8:
            assert (np.abs(drop * m) > bound).any(), "four limbs instead of five would pass"


def check_statistics(hk, g0, mi, xy, fold_sizes, tc):
    """Per-fold statistics of the last block: counts (n1, n2, n_miss) equal numpy's, and
    sum_fold[f, i] = (sum_s g0(i,s) xy[s, :], sum_s miss(i,s) xy[s, :]) over fold f against long double:
    tensor-core digits (9 radix-30 limbs of xy / s_c * 15): |err| <= s_c 30^-9 sum_s (g0 or miss) + 32 u s_c sum_s(...);
    FP64 reductions: |err| <= (n_f + 2) u sum|terms|, for any order of summation."""
    bs, ncol = g0.shape[0], xy.shape[1]
    starts = np.concatenate([[0], np.cumsum(fold_sizes)])
    s_c = np.abs(xy).max(axis=0)
    for f in range(len(fold_sizes)):
        sl = slice(starts[f], starts[f + 1])
        nf = starts[f + 1] - starts[f]
        cnt = np.stack([(g0[:, sl] == 1).sum(axis=1), (g0[:, sl] == 2).sum(axis=1), mi[:, sl].sum(axis=1)], axis=1)
        assert np.array_equal(hk["cnt"][f, :bs, :3], cnt), "fold %d counts" % f
        for plane, A in enumerate((g0, mi)):
            Af = A[:, sl]
            ref = _ld_matmul(Af, xy[sl])
            w = Af.sum(axis=1, dtype=np.float64)[:, None]
            if tc:
                bound = s_c[None, :] * w * (30.0 ** -9 + 32 * U)
            else:
                bound = (nf + 2) * U * (Af.astype(np.float64) @ np.abs(xy[sl]))
            ex = _excess(hk["sum"][f, :bs, plane, :ncol], ref, bound)
            assert ex <= 1.0, "fold %d, %s plane: statistics exceed the %s bound %.3g-fold" % (
                f, ("G0", "Miss")[plane], "tensor-core" if tc else "FP64", ex)


def _xy(pb):
    return np.hstack([pb.prep.X, pb.prep.Y])


def _run_block(pb, st, b):
    pb.gpu_l0_block(st, b)
    assert st.status() == 0
    return _hooks(st)


def _check_W(pb, st, b):
    W_o = pb.oracle_l0(b)[0]
    for ph in range(len(W_o)):
        assert rel(st.fetch_W(b, ph), W_o[ph]) < TOL, (b, ph)


# ----------------------------------------------------------------------------------------------- (a) block-size switches
def test_block_size_switches_solver_and_prediction(tmp_path, monkeypatch):
    """bsize 2048 (blocks 2048 + 1025): mixed solver at its largest n = 2048, INT8 prediction at 2 rows_p = 4096.
    bsize 2200 (blocks 2200 + 300): FP64 Cholesky at nC = 2240 and FP64 prediction for the first block; the second is
    solved by the mixed solver (n = 512) on a lane that has only ever seen this handle's bsize > 2048."""
    monkeypatch.setenv("RG_B200_LANES", "2")
    N, P, C = 5000, 6, 4                       # Q = 30: both epilogue halves (25 outputs each) of the INT8 kernel
    pa = _fileset(tmp_path, N, [3073, 2500], P, C, 0.02, 21, bsize=2048)
    assert [b[2] for b in pa.blocks[:2]] == [2048, 1025]
    st = pa.gpu_step1()
    for b in (0, 1):
        hk = _run_block(pa, st, b)
        assert hk["paths"] == (1, 1, 2048), hk["paths"]
        check_raw_predictions(hk, *_calls(pa, b), pa.prep.X, pa.prep.mask, pa.fold_sizes)
    assert st.solver_stats() == (2, 0)
    for b in (0, 1):
        _check_W(pa, st, b)
    st.close()

    pb = helpers.Problem(str(tmp_path / "syn"), str(tmp_path / "pheno.txt"), str(tmp_path / "covar.txt"), 2200)
    assert [b[2] for b in pb.blocks[2:4]] == [2200, 300]
    st = pb.gpu_step1()
    hk = _run_block(pb, st, 2)
    assert hk["paths"] == (1, 0, 0) and hk["nC"] == 2240, (hk["paths"], hk["nC"])
    check_raw_predictions(hk, *_calls(pb, 2), pb.prep.X, pb.prep.mask, pb.fold_sizes)
    hk = _run_block(pb, st, 3)                 # the second lane's first block
    assert hk["paths"] == (1, 1, 512), hk["paths"]
    check_raw_predictions(hk, *_calls(pb, 3), pb.prep.X, pb.prep.mask, pb.fold_sizes)
    assert st.solver_stats() == (1, 0)
    for b in (2, 3):
        _check_W(pb, st, b)
    st.close()


# ---------------------------------------------------------------------- (b) prediction kernels vs a long-double reference
@pytest.mark.parametrize("P", [11, 12, 26])
def test_prediction_kernels_within_their_error_bound(tmp_path, monkeypatch, P):
    """Blocks of 2200 (FP64 kernel), 2048 (INT8 at its bound), 129 and 1 SNPs; R = 5 ridge values, so Q = 55, 60, 130
    outputs: 2, 2 and 3 INT8 groups of 50, the last one partial."""
    monkeypatch.setenv("RG_B200_LANES", "2")
    pb = _fileset(tmp_path, 1500, [2200, 2048, 129, 1], P, 3, 0.02, 30 + P, bsize=2200)
    assert [b[2] for b in pb.blocks] == [2200, 2048, 129, 1]
    st = pb.gpu_step1()
    expect = {0: (0, 0), 1: (1, 2048), 2: (1, 256), 3: (1, 128)}
    for b in range(4):
        hk = _run_block(pb, st, b)
        assert hk["paths"] == (1,) + expect[b], (b, hk["paths"])
        check_raw_predictions(hk, *_calls(pb, b), pb.prep.X, pb.prep.mask, pb.fold_sizes, power=pb.blocks[b][2] > 1)
    assert st.solver_stats() == (3, 0)
    for b in range(4):
        _check_W(pb, st, b)
    st.close()


# ------------------------------------------------------------------- (c) tensor-core vs FP64 statistics on the same block
@pytest.mark.parametrize("P", [11, 12, 26])
def test_statistics_tensor_core_and_fp64_agree(tmp_path, monkeypatch, P):
    """C = 3 covariates + P traits = 14, 15, 29 columns: 1, 2, 3 digit groups (128 x 128, 128 x 256, three 128 x 128
    tiles).  1237 samples in four uneven folds, none a multiple of the 256-sample fold padding."""
    pb = _fileset(tmp_path, 1237, [200], P, 3, 0.03, 50 + P, bsize=200, K=4)
    pb.fold_sizes = np.array([517, 131, 300, 289], dtype=np.int64)
    assert pb.fold_sizes.sum() == len(pb.keys)
    g0, mi = _calls(pb, 0)
    monkeypatch.delenv("RG_B200_STATS", raising=False)
    st_tc = pb.gpu_step1()
    monkeypatch.setenv("RG_B200_STATS", "f64")
    st_64 = pb.gpu_step1()
    hks = []
    for st, tc in ((st_tc, 1), (st_64, 0)):
        hk = _run_block(pb, st, 0)
        assert hk["paths"] == (tc, 1, 256) and st.solver_stats() == (1, 0), (hk["paths"], st.solver_stats())
        check_statistics(hk, g0, mi, _xy(pb), pb.fold_sizes, tc=bool(tc))
        _check_W(pb, st, 0)
        hks.append(hk)
        st.close()
    assert np.array_equal(hks[0]["cnt"], hks[1]["cnt"])


# ------------------------------------------------------------------------ (d) the exactness limit of the tensor-core stats
def test_statistics_at_the_tensor_core_exactness_limit():
    """K = 2 folds around the largest fold the tensor-core statistics take: padded to 256 samples, 30 * 559104 < 2^24 but
    559105 pads to 559360 and 30 * 559360 > 2^24.  Only the intercept (a constant column, whose digit is 15) and SNPs with
    dosage 2 in >= 99.9 % of the samples: the intercept's per-fold digit sums come within 0.2 % of 2^24."""
    from regenie_b200 import capi
    F, BS, P = 559104, 64, 2
    assert F % 256 == 0 and 30 * F < 2 ** 24 <= 30 * (F + 256)
    N = 2 * F
    rng = np.random.default_rng(91)
    g = np.full((BS, N), 2, dtype=np.uint8)
    for i in range(BS):
        idx = rng.integers(0, N, size=N // 1500)
        g[i, idx] = rng.choice(np.array([0, 1, 3], dtype=np.uint8), size=idx.size)
    assert (g == 2).mean(axis=1).min() >= 0.999 and (g < 2).any(axis=1).all()
    X, Y, mask, in_an, neff = hostprep.prepare_qt(rng.standard_normal((N, P)), np.zeros((N, 0)))
    assert np.ptp(X[:, 0]) == 0.0
    lam = BS * (1 - hostprep.ridge_grid(5)) / hostprep.ridge_grid(5)
    g0 = np.where(g == 3, 0, g).astype(np.int8)
    mi = (g == 3).astype(np.int8)
    gc = np.where(g == 3, plink.MISSING_G, g.astype(np.float64))
    Gt, _ = step1.residualize_genotypes(plink.mean_impute_block(gc, in_an.astype(bool))[0], X, in_an.astype(bool), N, 1)
    del gc
    packed = synth.pack_bed(g)
    err = {}
    for folds, tc in (([F, F], 1), ([F + 1, F - 1], 0)):
        assert 15 * g0[:, :folds[0]].sum(axis=1, dtype=np.int64).max() > 0.998 * 2 ** 24
        st = capi.Step1(X, Y, mask, in_an, np.array(folds, dtype=np.int64), lam, neff, N, BS, 1)
        st.l0_block_bed(packed, BS, 0)
        assert st.status() == 0
        hk = _hooks(st)
        assert hk["paths"] == (tc, 1, 128) and st.solver_stats() == (1, 0), (hk["paths"], st.solver_stats())
        check_statistics(hk, g0, mi, np.hstack([X, Y]), folds, tc=bool(tc))
        check_raw_predictions(hk, g0, mi, X, mask, folds)
        W_o = step1.level0_kfold(Gt, Y, mask.astype(bool), np.array(folds), lam, neff)
        err["tensor-core" if tc else "FP64"] = max(rel(st.fetch_W(0, ph), W_o[ph]) for ph in range(P))
        st.close()
    assert max(err.values()) < TOL, err
