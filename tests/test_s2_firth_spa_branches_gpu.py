"""s2_firth_kernel and s2_spa_kernel on the branches that decide a TEST_FAIL row, and the binary-trait routes at a
biobank sample count.

1. The constructed block of firth_spa_cases (P = 2, half the rows flipped, z_thr = 0 so that every pair that is not
   ignored is selected) through rg_s2_block_bgen8_bt and rg_s2_block_bed_bt.  For every selection the status must
   equal the oracle's bit for bit: Firth st & 15 (Newton-Raphson failed), (st >> 4) & 15 (pseudo-Firth state) and
   st & 256 (carriers only); SPA st & 15 (reason) and st & 256 (fast).  Values agree to 1e-5 where both succeed.
   Branches with an asserted count (firth_spa_cases.check_floors): pseudo states 0, 1, 2; Newton-Raphson converged
   and stopped at its iteration cap; carriers only; SPA success, K'' = 0 in the search and at the root, p1 + p2 > 1,
   and p1 + p2 NaN because K(r) overflowed (see oracle.step2_bt.spa_test: status 5 where the reference ends the run).
   Branches not reached by these inputs:
     * pseudo state 3 (w == 0): impossible, get_pvec clamps eta;
     * pseudo state 4 and Newton-Raphson LRT < 0: the penalised likelihood of one coefficient is maximised at the
       root of the modified score, so a converged LRT is negative only through a rounding tie at LRT ~ 0 (the
       smallest converged LRT in the block is about 1e-4);
     * SPA limits: the score sits inside [lim_lo, lim_hi] unless it is at the edge to rounding;
     * SPA iteration cap: K'' = 0 ends the bisection from +-DBL_MAX first.
2. N = 300 000 (> 2^18 samples, two tensor-core chunks) with P = 2 and 160 variants: counts bit-exact against numpy,
   block_bed_bt against block_bgen8_bt, the statistics and > 256 Firth / SPA selections against the oracle.
"""
import math

import numpy as np
import pytest

import firth_spa_cases as fc
from oracle import step2_bt

pytestmark = pytest.mark.gpu
PATH_KEYS = ("tc", "nchunk", "chunk_len", "drows", "nchunks", "Npad", "dp", "bt_dp")


def _paths(st):
    return dict(zip(PATH_KEYS, (int(x) for x in st.debug("s2_paths", np.int64, 8))))


def _handle(pb, max_bs):
    from regenie_b200 import capi
    sts = pb["sts"]
    st = capi.Step2(pb["X"], pb["mask"], pb["ia"], pb["n_an"], max_bs)
    st.set_chr_bt(np.stack([s.gamma_sqrt_mask for s in sts], 1), np.stack([s.gamma_sqrt for s in sts], 1),
                  np.stack([s.yres for s in sts], 1), [s.Xg for s in sts], pb["Y"],
                  np.stack([s.cov_blup_offset for s in sts], 1), np.stack([s.phat for s in sts], 1))
    return st


def _probs(g):
    probs = np.zeros(g.shape + (2,), dtype=np.uint8)
    probs[..., 0] = (g == 2) * 255
    probs[..., 1] = (g == 1) * 255
    return probs, np.where(g == 3, 0x82, 0x02).astype(np.uint8)


def _route(st, g, route, min_mac):
    from regenie_b200 import synth
    if route == "bed":
        return st.block_bed_bt(synth.pack_bed(g), min_mac=min_mac)
    probs, miss = _probs(g)
    return st.block_bgen8_bt(probs, miss, min_mac=min_mac)


def _close(a, c, floor):
    return abs(a - c) <= 1e-5 * max(abs(c), floor)


@pytest.fixture(scope="module")
def branch_block():
    pb = fc.problem()
    return pb, fc.oracle_rows(pb)


@pytest.mark.parametrize("route", ["bgen8", "bed"])
def test_firth_spa_status_on_every_branch(branch_block, route):
    pb, rows = branch_block
    st = _handle(pb, fc.BS)
    o = _route(st, pb["g"], route, fc.MIN_MAC)
    sel = [(i, j) for i in range(fc.BS) for j in range(fc.P)
           if not (o["flags"][i] & 17) and o["mac"][i, j] >= fc.MIN_MAC and abs(o["stat"][i, j]) > 0.0]
    assert sorted(sel) == sorted(rows), set(sel) ^ set(rows)
    vi, ti = [a for a, _ in sel], [c for _, c in sel]
    fb, fse, flrt, fst = st.firth(vi, ti)
    pv, sst = st.spa(vi, ti)
    st.close()
    seen = dict(pseudo=np.zeros(5, int), nr=np.zeros(3, int), spa=np.zeros(6, int), carriers=0, nan_tail=0)
    for n, (i, j) in enumerate(sel):
        rf, rs = rows[(i, j)]
        assert abs(o["stat"][i, j] - rf["stat"]) <= 1e-8 * max(1.0, abs(rf["stat"])), (i, j)
        nr_failed = rf["nr"] is not None and rf["nr"] != step2_bt.NR_CONVERGED
        got = (fst[n] & 15, (fst[n] >> 4) & 15, bool(fst[n] & 256))
        assert got == (int(nr_failed), rf["firth_state"], rf["carriers_only"]), (i, j, got, rf["firth_state"], rf["nr"])
        seen["pseudo"][rf["firth_state"]] += 1
        if rf["nr"] is not None:
            seen["nr"][rf["nr"]] += 1
        seen["carriers"] += rf["carriers_only"]
        if not rf["test_fail"]:
            assert _close(fb[n], rf["beta"], 1e-6) and _close(fse[n], rf["se"], 1e-6), (i, j, fb[n], fse[n], rf)
            assert abs(flrt[n] - rf["chisq"]) <= 1e-5 * abs(rf["chisq"]) + 1e-8, (i, j, flrt[n], rf["chisq"])
        got = (sst[n] & 15, bool(sst[n] & 256))
        assert got == (rs["spa_reason"], rs["is_sparse"]), (i, j, got, rs["spa_reason"])
        seen["spa"][rs["spa_reason"]] += 1
        seen["nan_tail"] += rs["spa_nan_tail"]
        if rs["spa_nan_tail"]:                         # the kernel's tail is NaN too, and fails the test
            assert math.isnan(pv[n]), (i, j, pv[n])
        if rs["spa_reason"] == step2_bt.SPA_OK:
            logp = -math.log10(max(step2_bt.NL_DBL_DMIN, pv[n]))
            assert _close(logp, rs["logp"], 1e-3), (i, j, logp, rs["logp"])
    fc.check_floors(seen)                              # the same floors as the CPU test of the oracle


# ------------------------------------------------------------------------------------- 2. biobank sample count
def _big_problem(N, seed):
    rng = np.random.default_rng(seed)
    P, C = 2, 3
    ia = np.ones(N, dtype=bool)
    cov = rng.standard_normal((N, C - 1))
    X = np.hstack([np.ones((N, 1)), cov]) * ia[:, None]
    mask = np.ones((N, P), dtype=bool)
    eta = np.stack([-3.0 + 0.3 * cov[:, 0], -0.2 + 0.3 * cov[:, 1]], 1)
    Y = ((rng.random((N, P)) < 1 / (1 + np.exp(-eta))) & mask).astype(np.float64)
    blup = np.zeros((N, P))                   # (the branch block above carries the LOCO offsets)
    sts = [step2_bt.BtChrom(Y[:, j], X, blup[:, j], mask[:, j]) for j in range(P)]
    bs = 160
    g = np.zeros((bs, N), dtype=np.uint8)
    maf = rng.uniform(0.05, 0.5, 48)
    g[:48] = rng.binomial(2, maf[:, None], size=(48, N))                        # common
    for r in range(48, 96):                                                   # rare, MAC < 50
        idx = rng.choice(N, 3 + r % 40, replace=False)
        g[r, idx] = np.where(Y[idx, r % 2] == 1, 1, rng.integers(0, 2, len(idx)))
        g[r, idx[0]] = 1
    g[96:] = rng.binomial(2, rng.uniform(0.01, 0.2, bs - 96)[:, None], size=(bs - 96, N))
    g[::3] = np.where(g[::3] == 3, 3, 2 - g[::3])                             # flipped (major allele coded)
    miss = rng.random((bs, N)) < np.where(np.arange(bs) % 4 == 0, 0.01, 0.0)[:, None]
    g[miss] = 3                                                               # missing calls on every 4th row
    return dict(N=N, P=P, C=C, ia=ia, X=X, mask=mask, Y=Y, sts=sts, g=g, n_an=int(ia.sum()), bs=bs)


def test_bt_routes_at_300k_samples():
    N = 300_000
    pb = _big_problem(N, seed=77)
    g, ia, mask, P, bs = pb["g"], pb["ia"], pb["mask"], pb["P"], pb["bs"]
    st = _handle(pb, bs)
    ob = _route(st, g, "bed", 5.0)
    pa = _paths(st)
    Npad = (N + 127) // 128 * 128
    assert pa["tc"] == 1 and pa["Npad"] == Npad and pa["nchunk"] >= 2, pa
    assert pa["chunk_len"] * (pa["nchunk"] - 1) < Npad, pa
    # counts against numpy integer sums
    obs = (g != 3) & ia[None, :]
    gz = np.where(obs, g, 0).astype(np.int64)
    ns1 = obs.sum(axis=1)
    tot1 = gz.sum(axis=1)
    assert np.array_equal(ob["ns_all"], ns1)
    np.testing.assert_array_equal(ob["af_all"], tot1 / (2.0 * ns1))
    m = mask.astype(np.int64)
    nsp = obs.astype(np.int64) @ m
    totp = (gz @ m).astype(np.float64)
    assert np.array_equal(ob["ns"], nsp)
    np.testing.assert_array_equal(ob["af"], totp / (2.0 * nsp))
    np.testing.assert_array_equal(ob["mac"], np.minimum(totp, 2.0 * nsp - totp))
    assert np.array_equal(ob["flags"] & 1, (np.minimum(tot1, 2 * ns1 - tot1) < 5.0).astype(np.int32))
    assert np.array_equal((ob["flags"] & 8) != 0, tot1 / ns1 > 1)
    mu = np.where(tot1 / ns1 > 1, 2 - tot1 / ns1, tot1 / ns1)
    gf = np.where(tot1[:, None] / ns1[:, None] > 1, 2 - gz, gz) * obs
    nnz = (gf != 0).sum(axis=1) + np.where(mu != 0, (~obs & ia[None, :]).sum(axis=1), 0)
    assert np.array_equal((ob["flags"] & 4) != 0, nnz <= N * 0.5)
    # Firth and SPA on the 2-bit block: > 256 selections (two launches), the same bits when split in two calls
    sel = [(i, j) for i in range(bs) for j in range(P)
           if not (ob["flags"][i] & 17) and ob["mac"][i, j] >= 5.0 and abs(ob["stat"][i, j]) > 0.0]
    assert len(sel) > 256
    vi, ti = [a for a, _ in sel], [c for _, c in sel]
    fb, fse, flrt, fst = st.firth(vi, ti)
    pv, sst = st.spa(vi, ti)
    h = len(sel) // 3
    for lo, hi in ((0, h), (h, len(sel))):
        for a, c in zip(st.firth(vi[lo:hi], ti[lo:hi]), (fb, fse, flrt, fst)):
            assert np.array_equal(a, c[lo:hi], equal_nan=a.dtype.kind == "f")
        for a, c in zip(st.spa(vi[lo:hi], ti[lo:hi]), (pv, sst)):
            assert np.array_equal(a, c[lo:hi], equal_nan=a.dtype.kind == "f")
    # the dosage route on the same hard calls
    od = _route(st, g, "bgen8", 5.0)
    st.close()
    for k in ("ns", "flags"):
        assert np.array_equal(ob[k], od[k]), k
    assert np.array_equal(ob["af"], od["af"])
    ok = np.isfinite(od["stat"])
    assert np.all(np.abs(ob["stat"] - od["stat"])[ok] <= 1e-9 * np.maximum(1.0, np.abs(od["stat"][ok])))
    # the oracle on a sample of selections: carriers-only fits among them
    rng = np.random.default_rng(7)
    pick = sorted(set(rng.choice(len(sel), 40, replace=False)) | {n for n, (i, _) in enumerate(sel) if 48 <= i < 60})
    n_fast = 0
    for n in pick:
        i, j = sel[n]
        gd = np.where(g[i] == 3, -3.0, g[i].astype(np.float64))
        args = (gd, np.zeros(N), ia, mask[:, j], pb["Y"][:, j], pb["sts"][j], 0.0, N)
        rf = step2_bt.score_bt(*args)
        assert abs(ob["stat"][i, j] - rf["stat"]) <= 1e-8 * max(1.0, abs(rf["stat"])), (i, j)
        got = (fst[n] & 15, (fst[n] >> 4) & 15, bool(fst[n] & 256))
        nr_failed = rf["nr"] is not None and rf["nr"] != step2_bt.NR_CONVERGED
        assert got == (int(nr_failed), rf["firth_state"], rf["carriers_only"]), (i, j, got)
        n_fast += rf["carriers_only"]
        if not rf["test_fail"]:
            assert _close(fb[n], rf["beta"], 1e-6) and _close(fse[n], rf["se"], 1e-6), (i, j)
            assert abs(flrt[n] - rf["chisq"]) <= 1e-5 * abs(rf["chisq"]) + 1e-8, (i, j)
        rs = step2_bt.score_bt(*args, correction="spa")
        assert (sst[n] & 15, bool(sst[n] & 256)) == (rs["spa_reason"], rs["is_sparse"]), (i, j, sst[n])
        if rs["spa_reason"] == step2_bt.SPA_OK:
            assert _close(-math.log10(max(step2_bt.NL_DBL_DMIN, pv[n])), rs["logp"], 1e-3), (i, j)
    assert len(pick) >= 40 and n_fast >= 5
