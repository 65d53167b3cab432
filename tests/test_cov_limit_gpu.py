"""Every Step-1 and Step-2 entry point at the covariate limit: C = 64 columns of X (intercept + 63 covariates), the most
the kernels take (kMaxCov) and what a conditional analysis on many variants reaches.  Each route against the numpy
oracle at the tolerances of its own test at small C: level 0 on 2-bit rows and on dosages (the dense FP64 route), level 1
and LOCO (ridge and logistic), and the Step-2 block routes on 2-bit rows and 8-bit dosages for both trait kinds with
Firth and SPA on the resident block."""
import numpy as np
import pytest

import helpers
from oracle import bgen as obgen
from oracle import plink, prep, step1, step1_bt, step2, step2_bt
from test_s2_paths_gpu import _bt_handle, _bt_problem, _probs, _qt_problem

pytestmark = pytest.mark.gpu
C_MAX = 64


def rel(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def _problem(tmp_path, loocv=False):
    pb = helpers.synthetic_problem(tmp_path, N=1500, M=300, P=2, C=C_MAX, bsize=100, K=5, seed=64, loocv=loocv)
    assert pb.prep.ncov == C_MAX
    return pb


def test_level0_level1_loco_at_64_covariates(tmp_path):
    """rg_l0_block_bed on every block, then rg_l1_fit and rg_loco, against oracle.step1 (test_l0_gpu / test_l1_gpu)."""
    pb = _problem(tmp_path)
    st = pb.gpu_step1()
    for b in range(len(pb.blocks)):
        pb.gpu_l0_block(st, b)
        assert st.status() == 0
        W_o, _, _, _ = pb.oracle_l0(b)
        for ph in range(2):
            assert rel(st.fetch_W(b, ph), W_o[ph]) < 1e-9, (b, ph)
    B = len(pb.blocks) * 5
    h1 = prep.set_ridge_params(5)
    cs, best = st.l1_fit(np.tile(B * (1 - h1) / h1, (2, 1)))
    loco = st.loco([c for c, _, _ in pb.blocks])
    assert st.status() == 0

    def gen():
        for b in range(len(pb.blocks)):
            yield pb.oracle_block(b)[0]
    o = step1.run_step1_qt(gen(), pb.blocks, pb.prep, pb.fold_sizes, pb.M)
    for ph in range(2):
        assert rel(cs[:, ph, :], o["cs"][ph]) < 1e-8
        assert best[ph] == o["best"][ph]
        assert rel(loco[ph], o["loco"][ph]) < 1e-7
    st.close()


@pytest.mark.parametrize("loocv", [False, True])
def test_logistic_level1_and_loco_at_64_covariates(tmp_path, loocv):
    """rg_l1_fit_bt (k-fold IRLS and closed-form LOO) and rg_loco against oracle.step1_bt (test_l1_bt_gpu)."""
    pb = _problem(tmp_path, loocv)
    pr = pb.prep
    rng = np.random.default_rng(5)
    y_raw = (pr.Y + 0.3 * rng.standard_normal(pr.Y.shape) > 0.4).astype(float) * pr.mask
    st = pb.gpu_step1()
    nb = len(pb.blocks)
    for b in range(nb):
        pb.gpu_l0_block(st, b)
    assert st.status() == 0
    B = nb * 5
    h1 = prep.set_ridge_params(5)
    tau = B * (1 - h1) / h1 * 3 / np.pi ** 2
    off = np.stack([step1_bt.null_offset(y_raw[:, p], pr.X, pr.mask[:, p]) for p in range(2)], axis=1)
    cs, best = st.l1_fit_bt(y_raw, off, np.tile(tau, (2, 1)))
    chr_of_block = [c for c, _, _ in pb.blocks]
    loco = st.loco(chr_of_block)
    chr_cols = [(c, chr_of_block.index(c) * 5, chr_of_block.count(c) * 5) for c in sorted(set(chr_of_block))]
    for p in range(2):
        W = np.hstack([st.fetch_W(b, p) for b in range(nb)])
        if loocv:
            cs_o = step1_bt.level1_logistic_loocv(W, y_raw[:, p], off[:, p], pr.mask[:, p], tau)
        else:
            cs_o, betas = step1_bt.level1_logistic_kfold(W, y_raw[:, p], off[:, p], pr.mask[:, p], tau, pb.fold_sizes)
        np.testing.assert_allclose(cs[:, p, :], cs_o, rtol=1e-7, atol=1e-9)
        best_o, _ = step1_bt.output_table(cs_o, pr.neff[p], B, tau)
        assert best[p] == best_o
        if loocv:
            pred = step1_bt.predictions_binary_loocv(W, y_raw[:, p], off[:, p], pr.mask[:, p], tau[best_o], chr_cols)
        else:
            pred = step1_bt.predictions_binary_kfold(W, betas, best_o, pb.fold_sizes, chr_cols)
        np.testing.assert_allclose(loco[p], step1.loco_matrix(pred, chr_cols), rtol=1e-6, atol=1e-8)
    st.close()


def test_level0_dense_fp64_route_at_64_covariates(tmp_path):
    """rg_l0_block_dosage_u8 and rg_l0_block_f64 (the dense FP64 level-0 route) against the oracle (test_l0_dosage_gpu)."""
    pb = helpers.synthetic_problem(tmp_path, N=1100, M=96, P=3, C=C_MAX, bsize=96, seed=4)
    pr = pb.prep
    assert pr.ncov == C_MAX
    rng = np.random.default_rng(11)
    probs, miss = _probs(rng, 96, 1100)
    g = np.stack([obgen.dosage(probs[v, :, 0].astype(np.float64), probs[v, :, 1].astype(np.float64), (miss[v] & 0x80) != 0)[0]
                  for v in range(96)])
    gi, _ = plink.mean_impute_block(g, pr.in_analysis)
    Gt, _ = step1.residualize_genotypes(gi, pr.X, pr.in_analysis, pr.n_analyzed, pr.ncov)
    W_o = step1.level0_kfold(Gt, pr.Y, pr.mask, pb.fold_sizes, pb.lam, pr.neff)
    st = pb.gpu_step1()
    st.l0_block_dosage_u8(probs, miss, 0)
    assert st.status() == 0
    st2 = pb.gpu_step1()
    st2.l0_block_f64(g, 0)
    assert st2.status() == 0
    for ph in range(3):
        assert rel(st.fetch_W(0, ph), W_o[ph]) < 1e-9
        assert rel(st2.fetch_W(0, ph), W_o[ph]) < 1e-9
    st.close()
    st2.close()


def _close_stats(o, i, sc, tol=1e-8):
    """BETA / SE / CHISQ of variant i against the oracle: relative, with the statistic's error taken as absolute near 0
    (a statistic near 0 is a difference of O(1) terms; see test_s2_paths_gpu._same_stats)."""
    se = sc["se"]
    np.testing.assert_allclose(o["se"][i], se, rtol=tol, atol=0)
    assert np.all(np.abs(o["beta"][i] - sc["beta"]) <= tol * (np.abs(sc["beta"]) + np.abs(se))), i
    assert np.all(np.abs(o["chisq"][i] - sc["chisq"]) <= 2 * tol * (1 + sc["chisq"])), i


def test_s2_qt_block_routes_at_64_covariates():
    """rg_s2_block_bed and rg_s2_block_bgen8 against oracle.step2.score_qt."""
    from regenie_b200 import capi, synth
    N, M, P = 3001, 128, 3
    pb = _qt_problem(N, P, C_MAX, seed=64)
    g = synth.genotypes(N, M, seed=64, miss=0.02)
    packed = synth.pack_bed(g)
    graw = plink.decode_bed(packed, N)
    probs, miss = _probs(np.random.default_rng(64), M, N)
    gd = np.stack([obgen.dosage(probs[v, :, 0].astype(np.float64), probs[v, :, 1].astype(np.float64), (miss[v] & 0x80) != 0)[0]
                   for v in range(M)])
    st = capi.Step2(pb["X"], pb["mask"], pb["ia"], pb["n_an"], M)
    st.set_chr(pb["res"], pb["scf"])
    for o, G in ((st.block_bed(packed), graw), (st.block_bgen8(probs, miss), gd)):
        n = 0
        for i in range(M):
            vs = step2.variant_stats(G[i], pb["ia"], pb["mask"])
            if vs["ignored"]:
                assert o["flags"][i] & 1
                continue
            sc = step2.score_qt(vs["g"], pb["X"], pb["res"], pb["mask"], pb["ia"], pb["n_an"], C_MAX, pb["scf"], pb["YtX"], False)
            assert bool(o["flags"][i] & 2) == (sc is None)
            if sc is None:
                continue
            _close_stats(o, i, sc)
            n += 1
        assert n > 100
    st.close()


def test_s2_bt_block_routes_firth_spa_at_64_covariates():
    """rg_s2_block_bgen8_bt with rg_s2_firth / rg_s2_spa on its resident block, then rg_s2_block_bed_bt, against
    oracle.step2_bt.score_bt (test_s2_paths_gpu.test_bt_fractional_dosages_firth_spa at C = 3)."""
    from regenie_b200 import synth
    N, P, bs, z_thr = 3001, 2, 128, 0.5
    b = _bt_problem(N, P, C_MAX, seed=64)
    ia, mask = b["ia"], b["mask"]
    probs, miss = _probs(np.random.default_rng(65), bs, N, miss_frac=0.01)
    st = _bt_handle(b, 256)
    o = st.block_bgen8_bt(probs, miss, min_mac=5.0)
    sel = [(i, j) for i in range(bs) for j in range(P)
           if not (o["flags"][i] & 17) and o["mac"][i, j] >= 5.0 and abs(o["stat"][i, j]) > z_thr]
    assert len(sel) > 50
    fb, fse, flrt, fst = st.firth([a for a, _ in sel], [c for _, c in sel])
    pv, sst = st.spa([a for a, _ in sel], [c for _, c in sel])
    fmap = {k: n for n, k in enumerate(sel)}
    n_firth = n_spa = 0
    m = (miss & 0x80) != 0
    for i in range(bs):
        g, ival = obgen.dosage(probs[i, :, 0].astype(np.float64), probs[i, :, 1].astype(np.float64), m[i])
        for j in range(P):
            s = b["sts"][j]
            r = step2_bt.score_bt(g, ival, ia, mask[:, j], b["Y"][:, j], s, z_thr, N)
            if r is None:
                continue
            assert abs(o["stat"][i, j] - r["stat"]) <= 1e-8 * max(1.0, abs(r["stat"])), (i, j)
            if abs(r["stat"]) <= z_thr:
                continue
            n = fmap[(i, j)]
            assert (fst[n] & 15) == int(r["test_fail"]), (i, j, fst[n])
            if not r["test_fail"]:
                n_firth += 1
                for a, c in zip((fb[n], fse[n], flrt[n]), (r["beta"], r["se"], r["chisq"])):
                    assert abs(a - c) <= 1e-5 * max(abs(c), 1e-8), (i, j, a, c)
            rs = step2_bt.score_bt(g, ival, ia, mask[:, j], b["Y"][:, j], s, z_thr, N, correction="spa")
            assert bool(sst[n] & 15) == rs["test_fail"], (i, j, sst[n])
            if not rs["test_fail"]:
                n_spa += 1
                chisq = step2_bt.chisq1_from_pvalue(max(step2_bt.NL_DBL_DMIN, pv[n]))
                assert abs(chisq - rs["chisq"]) <= 1e-5 * rs["chisq"], (i, j, chisq, rs["chisq"])
    assert n_firth > 50 and n_spa > 50
    # 2-bit rows on the same handle
    gh = synth.genotypes(N, bs, seed=66, miss=0.02)
    packed = synth.pack_bed(gh)
    graw = plink.decode_bed(packed, N)
    ob = st.block_bed_bt(packed, min_mac=5.0)
    n = 0
    for i in range(bs):
        for j in range(P):
            r = step2_bt.score_bt(graw[i], np.zeros(N), ia, mask[:, j], b["Y"][:, j], b["sts"][j], np.inf, N)
            if r is None:
                continue
            assert abs(ob["stat"][i, j] - r["stat"]) <= 1e-8 * max(1.0, abs(r["stat"])), (i, j)
            for k in ("beta", "se", "chisq"):
                assert abs(ob[k][i, j] - r[k]) <= 1e-8 * max(abs(r[k]), 1e-8), (i, j, k)
            n += 1
    assert n > 150
    st.close()
