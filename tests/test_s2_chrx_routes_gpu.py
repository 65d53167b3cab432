"""Step 2 on the non-PAR part of chromosome X, on every block route, against an exact integer reference.

With sex information (rg_s2_set_sex before rg_s2_set_chr / rg_s2_set_chr_bt) the chromosome's feature row F gains 1 + P
columns: the analysed males, then the males among each trait's samples.  A variant flagged by rg_s2_set_non_par (for the
next block call only) counts its males, coded 0/2, half towards the allele count (src/Geno.cpp:2447-2462):

    macr = sum d - 1/2 sum_males d,     MAC = min(macr, 2 ns - (males with a call) - macr),

while N and A1FREQ keep the autosomal formulas (A1FREQ divides by 2 ns: --skip-dosage-comp is not used here).  The
reference below forms these from the codes in Python integers and fractions.Fraction (d = g for hard calls, d = 255 x
dosage for 8-bit probabilities), never from floats.

Hard calls: every sum is an exact integer and the halves are exact in binary, so N, MAC and A1FREQ must be bit-exact.
8-bit dosages: the kernels scale the integer sums by the double nearest 1/255 before the male half is taken off, so
MAC is not the rounded rational; it is held to the error bound of that arithmetic (see _mac_bound), a few ulp.  The
statistics do not depend on sex: they equal those of a handle without it, bit for bit on the 2-bit tensor routes (exact
integer sums) and within 1e-12 on the dosage routes, and the numpy oracle at the tolerances of test_s2_paths_gpu.py.
"""
import math
from fractions import Fraction

import numpy as np
import pytest

import interaction_bt_oracle as ibo
import interaction_oracle as io
from oracle import bgen as obgen
from oracle import plink, step2, step2_bt
from oracle.prep import get_basis

pytestmark = pytest.mark.gpu
U = 2.0 ** -53
LD = np.longdouble
K255 = 1.0 / 255.0
PATH_KEYS = ("tc", "nchunk", "chunk_len", "drows", "nchunks", "Npad", "dp", "bt_dp")
DROP = [2, 2501, 5003]                     # samples of the file that the handle does not hold (sample_idx)


def _paths(st):
    return dict(zip(PATH_KEYS, (int(x) for x in st.debug("s2_paths", np.int64, 8))))


def _codes(probs, miss, keep, ref_first):
    """Integer dosage x 255, INFO term x 255 and the missing flag of every kept sample (parseSnpfromBGEN in integers)."""
    p0 = probs[:, keep, 0].astype(np.int64)
    p1 = probs[:, keep, 1].astype(np.int64)
    hom = np.maximum(255 - p0 - p1, 0) if ref_first else p0
    m = np.zeros(p0.shape, dtype=bool) if miss is None else (miss[:, keep] & 0x80) != 0
    d = np.where(m, 0, p1 + 2 * hom)
    e = np.where(m, 0, 4 * hom + p1)
    return d, e, m


def _check_sums(got, planes, F, rows, exact_cols, n_terms):
    """got [rows][planes][dp] FP64 sums of plane * F: exact on the 0/1 columns, within gamma_n sum |plane F| elsewhere."""
    FL = F.astype(LD)
    for k, z in enumerate(planes):
        zr = z[rows]
        ref = zr.astype(LD) @ FL
        bound = (n_terms * U) * (np.abs(zr).astype(np.float64) @ np.abs(F)) * 1.01
        err = np.abs(got[rows, k, :F.shape[1]].astype(LD) - ref).astype(np.float64)
        bad = np.argwhere(err > bound)
        assert bad.size == 0, ("sum plane %d, row %d, column %d off by %g (bound %g)" %
                               (k, rows[bad[0][0]], bad[0][1], err[tuple(bad[0])], bound[tuple(bad[0])]))
        assert np.array_equal(got[rows, k][:, exact_cols], ref[:, exact_cols].astype(np.float64)), ("0/1 column", k)


# ------------------------------------------------------------------------------------------------------ the data
def _samples(n_file, P, seed, drop):
    """Kept samples, sex, analysed set and trait masks.  About 2 % of the samples lie outside the analysis, both sexes
    among them; trait 1 also drops 15 % of the males, so the per-trait male totals differ."""
    rng = np.random.default_rng(seed)
    keep = np.ones(n_file, dtype=bool)
    if drop:
        keep[DROP] = False
    male_f = rng.random(n_file) < 0.45
    N = int(keep.sum())
    male = male_f[keep]
    ia = np.ones(N, dtype=bool)
    ia[rng.choice(N, N // 50, replace=False)] = False
    assert (~ia & male).any() and (~ia & ~male).any()
    mask = ia[:, None] & (rng.random((N, P)) > 0.05)
    if P > 1:
        mask[:, 1] &= ~(male & (rng.random(N) < 0.15))
    assert P == 1 or (mask[:, 0] & male).sum() > (mask[:, 1] & male).sum() + N // 50
    return dict(n_file=n_file, keep=keep, sidx=np.nonzero(keep)[0].astype(np.int32) if drop else None, N=N,
                male_f=male_f, male=male, ia=ia, mask=mask, P=P, rng=rng)


def _alt_counts(rng, bs, male_f):
    """ALT allele counts [bs, n_file] (3 = missing): females binomial, males 0/2 with a few coded 1 (the reference warns
    and counts them 0.5), 3 % missing.  Three quarters of the rows are rare, with an autosomal MAC of about 35-55 at
    5000 samples, which the male rule lowers by about a fifth, so that many of them cross a MAC threshold; the rest are
    common, some with the ALT allele the major one."""
    n = len(male_f)
    af = np.concatenate([rng.uniform(0.0035, 0.0055, bs - bs // 4), rng.uniform(0.03, 0.97, bs // 4)])
    rng.shuffle(af)
    g = rng.binomial(2, af[:, None], size=(bs, n))
    g = np.where(male_f[None, :], 2 * rng.binomial(1, af[:, None], size=(bs, n)), g)
    g = np.where(male_f[None, :] & (rng.random((bs, n)) < 0.002), 1, g)
    return np.where(rng.random((bs, n)) < 0.03, 3, g)


def _bed_rows(a, ref_first):
    """.bed rows whose decoded calls (with or without --ref-first) are the ALT counts a."""
    from regenie_b200 import synth
    return synth.pack_bed(np.where(a == 3, 3, a if not ref_first else 2 - a))


def _probs(rng, a, ref_first):
    """8-bit probability pairs of the ALT counts a, in the file's allele order: 30 % of the carriers (males too) and 2 %
    of the non-carriers get a fractional call."""
    bs, n = a.shape
    hom = np.where(a == 2, 255, 0)
    het = np.where(a == 1, 255, 0)
    r = rng.random((bs, n))
    f2 = (a == 2) & (r < 0.3)
    hom = np.where(f2, rng.integers(170, 255, (bs, n)), hom)
    het = np.where(f2, ((255 - hom) * rng.random((bs, n))).astype(np.int64), het)
    f1 = (a == 1) & (r < 0.3)
    het = np.where(f1, rng.integers(120, 255, (bs, n)), het)
    hom = np.where(f1, ((255 - het) * rng.random((bs, n)) * 0.3).astype(np.int64), hom)
    f0 = (a == 0) & (r < 0.02)
    het = np.where(f0, rng.integers(1, 90, (bs, n)), het)
    miss = np.where(a == 3, 0x82, 0x02).astype(np.uint8)
    hom, het = np.where(a == 3, 0, hom), np.where(a == 3, 0, het)
    p0 = 255 - hom - het if ref_first else hom
    return np.stack([p0, het], axis=-1).astype(np.uint8), miss


def _calls(sm, a, kind, probs=None, miss=None, ref_first=False):
    """(d, unit, missing) of the kept samples: d integer ALT dosage x unit."""
    keep = sm["keep"]
    if kind == "hard":
        ak = a[:, keep]
        return np.where(ak == 3, 0, ak).astype(np.int64), 1, ak == 3
    d, _, m = _codes(probs, miss, keep, ref_first)
    return d, 255, m


# ------------------------------------------------------------------------------------------- the exact reference
def _exact(sm, d, m, unit, non_par):
    """Integer sums and the exact MAC of every variant, over all analysed samples (column 0) and per trait."""
    ia, mask, male = sm["ia"], sm["mask"].astype(np.int64), sm["male"]
    ok = ~m & ia[None, :]
    dz = np.where(ok, d, 0)
    dm = dz * male[None, :]
    okm = (ok & male[None, :]).astype(np.int64)
    tot = np.column_stack([dz.sum(1), dz @ mask])                 # [bs, 1 + P]
    mtot = np.column_stack([dm.sum(1), dm @ mask])
    ns = np.column_stack([ok.sum(1), ok.astype(np.int64) @ mask])
    nmale = np.column_stack([okm.sum(1), okm @ mask])
    mac = np.empty(tot.shape, dtype=object)
    for i in range(tot.shape[0]):
        for c in range(tot.shape[1]):
            t, n2 = int(tot[i, c]), 2 * int(ns[i, c])
            if non_par[i]:
                r = Fraction(2 * t - int(mtot[i, c]), 2 * unit)
                mac[i, c] = min(r, n2 - int(nmale[i, c]) - r)
            else:
                r = Fraction(t, unit)
                mac[i, c] = min(r, n2 - r)
    return dict(tot=tot, mtot=mtot, ns=ns, nmale=nmale, mac=mac, ok=ok)


def _mac_bound(ex, i, c, unit, non_par):
    """Error bound of a dosage MAC: sum d and sum_males d are exact integers, each scaled by fl(1/255) (two roundings),
    the half is exact, then one subtraction for macr and one for 2 ns - males - macr."""
    if unit == 1:
        return 0.0
    t, mt = int(ex["tot"][i, c]), int(ex["mtot"][i, c])
    macr = (t - (mt / 2 if non_par else 0)) / unit
    other = 2 * int(ex["ns"][i, c]) - (int(ex["nmale"][i, c]) if non_par else 0) - macr
    err = 1.01 * U * (2 * (t + mt / 2) / unit + abs(macr))
    return err + (1.01 * U * abs(other) if other < macr else 0.0)


def _check_counts(route, o, ex, sm, unit, non_par, min_mac):
    """N, MAC, A1FREQ and the MAC decisions of one block call against the exact reference."""
    bs, P = o["mac"].shape
    assert np.array_equal(o["ns_all"], ex["ns"][:, 0]), (route, "N_all")
    assert np.array_equal(o["ns"], ex["ns"][:, 1:]), (route, "N")
    tot = ex["tot"].astype(np.float64) * (K255 if unit == 255 else 1.0)
    af = tot / (2.0 * ex["ns"])
    assert np.array_equal(o["af_all"], af[:, 0], equal_nan=True), (route, "A1FREQ_all")
    assert np.array_equal(o["af"], af[:, 1:], equal_nan=True), (route, "A1FREQ")
    got = np.column_stack([o["mac_all"], o["mac"]])
    for i in range(bs):
        for c in range(1 + P):
            want = ex["mac"][i, c]
            if unit == 1 or not non_par[i]:
                w = float(want) if unit == 1 else min(tot[i, c], 2.0 * ex["ns"][i, c] - tot[i, c])
                assert got[i, c] == w, (route, "MAC", i, "trait %d" % (c - 1), got[i, c], w)
            else:
                b = _mac_bound(ex, i, c, unit, True)
                assert abs(Fraction(got[i, c]) - want) <= b, (route, "MAC", i, "trait %d" % (c - 1), got[i, c], float(want), b)
    assert np.array_equal((o["flags"] & 1) != 0, np.array([x < min_mac for x in ex["mac"][:, 0]])), (route, "flag bit 0")
    ign = np.array([[x < min_mac for x in row] for row in ex["mac"][:, 1:]])
    assert np.array_equal(o["mac"] < min_mac, ign), (route, "per-trait ignore")


def _check_oracle_mac(route, ex, graw, sm, non_par):
    """Hard calls: the exact MAC equals the oracle's variant_stats(male=, non_par=) bit for bit."""
    for i in range(graw.shape[0]):
        vs = step2.variant_stats(graw[i], sm["ia"], sm["mask"], male=sm["male"], non_par=bool(non_par[i]))
        assert Fraction(vs["mac1"]) == ex["mac"][i, 0], (route, i, vs["mac1"], float(ex["mac"][i, 0]))
        for p in range(sm["P"]):
            assert Fraction(float(vs["mac"][p])) == ex["mac"][i, 1 + p], (route, i, p, vs["mac"][p], float(ex["mac"][i, 1 + p]))


def _min_mac(exs, lo=20.0, hi=60.0):
    """A MAC threshold that more than 50 variants cross under the male rule, no exact MAC within 4 ulp of it."""
    best = None
    for t in np.arange(lo, hi) + 0.25:                                # hard-call MACs are halves, dosage ones k / 510
        moved = sum(int((x < t) != (y < t)) for ex_x, ex_a in exs for x, y in zip(ex_x["mac"][:, 0], ex_a["mac"][:, 0]))
        if best is None or moved > best[1]:
            best = (float(t), moved)
    t = best[0]
    for ex_x, ex_a in exs:
        for e in (ex_x, ex_a):
            for x in e["mac"].ravel():
                assert abs(float(x) - t) > 4 * 2 * U * t
    assert best[1] > 50, best
    return t


def _same_stats(route, a, b, exact):
    """Statistics of the chrX handle against those of the handle without sex."""
    if exact:
        for k in ("stat", "beta", "se"):
            bad = np.argwhere(~((a[k] == b[k]) | (np.isnan(a[k]) & np.isnan(b[k]))))
            assert bad.size == 0, (route, k, "variant %d trait %d" % tuple(bad[0]), a[k][tuple(bad[0])], b[k][tuple(bad[0])])
        return
    fin = np.isfinite(b["stat"])
    assert np.array_equal(fin, np.isfinite(a["stat"])), route
    tol = 1e-12
    d = np.abs(a["stat"] - b["stat"])[fin] > tol * np.maximum(1.0, np.abs(b["stat"][fin]))
    assert not d.any(), (route, "stat", np.argwhere(fin)[np.argmax(d)])
    d = np.abs(a["beta"] - b["beta"])[fin] > tol * (np.abs(b["beta"]) + np.abs(b["se"]))[fin]
    assert not d.any(), (route, "beta", np.argwhere(fin)[np.argmax(d)])
    d = np.abs(a["se"] - b["se"])[fin] > tol * np.abs(b["se"][fin])
    assert not d.any(), (route, "se", np.argwhere(fin)[np.argmax(d)])


# -------------------------------------------------------------------------------------------------- the handles
def _qt_state(sm, C, seed):
    rng = np.random.default_rng(seed)
    ia, mask, N, P = sm["ia"], sm["mask"], sm["N"], sm["P"]
    X = np.zeros((N, C))
    X[ia], _ = np.linalg.qr(np.hstack([np.ones((int(ia.sum()), 1)), rng.standard_normal((int(ia.sum()), C - 1))]))
    X = np.asfortranarray(X)
    n_an = int(ia.sum())
    res = rng.standard_normal((N, P)) * mask
    res = np.asfortranarray(res / (np.linalg.norm(res, axis=0) / np.sqrt(n_an - C)))
    return dict(X=X, n_an=n_an, res=res, scf=rng.uniform(0.5, 2.0, P), YtX=res.T @ X, C=C)


def _bt_state(sm, C, seed):
    rng = np.random.default_rng(seed)
    ia, mask, N, P = sm["ia"], sm["mask"], sm["N"], sm["P"]
    cov = rng.standard_normal((N, C - 1))
    X = np.hstack([np.ones((N, 1)), cov]) * ia[:, None]
    eta = -0.8 + cov @ rng.normal(0, 0.4, size=(C - 1, P))
    Y = ((rng.random((N, P)) < 1 / (1 + np.exp(-eta))) & mask).astype(np.float64)
    blup = 0.3 * rng.standard_normal((N, P)) * mask
    sts = [step2_bt.BtChrom(Y[:, j], X, blup[:, j], mask[:, j]) for j in range(P)]
    return dict(X=X, Y=Y, sts=sts, n_an=int(ia.sum()), C=C)


def _qt_handle(sm, q, bs_max, sex):
    from regenie_b200 import capi
    st = capi.Step2(q["X"], sm["mask"], sm["ia"], q["n_an"], bs_max)
    if sex:
        st.set_sex(sm["male"])
    st.set_chr(q["res"], q["scf"])
    return st


def _bt_handle(sm, b, bs_max, sex):
    from regenie_b200 import capi
    sts = b["sts"]
    st = capi.Step2(b["X"], sm["mask"], sm["ia"], b["n_an"], bs_max)
    if sex:
        st.set_sex(sm["male"])
    st.set_chr_bt(np.stack([s.gamma_sqrt_mask for s in sts], 1), np.stack([s.gamma_sqrt for s in sts], 1),
                  np.stack([s.yres for s in sts], 1), [s.Xg for s in sts], b["Y"],
                  np.stack([s.cov_blup_offset for s in sts], 1), np.stack([s.phat for s in sts], 1))
    return st


def _run(st, route, blk, sm, ref_first, min_mac):
    if route in ("bed", "bed_f64"):
        return st.block_bed(blk, sample_idx=sm["sidx"], ref_first=ref_first, min_mac=min_mac)
    if route == "bed_bt":
        return st.block_bed_bt(blk, sample_idx=sm["sidx"], ref_first=ref_first, min_mac=min_mac)
    fn = st.block_bgen8 if route == "bgen8" else st.block_bgen8_bt
    return fn(blk[0], blk[1], sample_idx=sm["sidx"], ref_first=ref_first, min_mac=min_mac)


def _qt_F(sm, q, dp):
    """rg_s2_set_chr's feature row with sex: [a | x | res | m | m_p x_c | male | male m_p]."""
    N, C, P, ia, mask = sm["N"], q["C"], sm["P"], sm["ia"], sm["mask"]
    F = np.zeros((N, dp))
    F[:, 0] = ia
    F[:, 1:1 + C] = q["X"]
    F[:, 1 + C:1 + C + P] = q["res"]
    F[:, 1 + C + P:1 + C + 2 * P] = mask
    for p in range(P):
        F[:, 1 + C + 2 * P + p * C:1 + C + 2 * P + (p + 1) * C] = mask[:, p:p + 1] * q["X"]
    base = 1 + C + 2 * P + P * C
    F[:, base] = ia & sm["male"]
    F[:, base + 1:base + 1 + P] = (ia & sm["male"])[:, None] & mask
    return F, [0] + list(range(1 + C + P, 1 + C + 2 * P)) + list(range(base, base + 1 + P))


def _bt_F(sm, b, dp):
    """rg_s2_set_chr_bt's feature row with sex: [a | per trait: m | w^2 | w yres | w XGamma_c | male | male m_p]."""
    N, P, C, ia, mask = sm["N"], sm["P"], b["C"], sm["ia"], sm["mask"]
    F = np.zeros((N, dp))
    F[:, 0] = ia
    for p, s in enumerate(b["sts"]):
        c0 = 1 + p * (3 + C)
        w = np.where(ia, s.gamma_sqrt_mask, 0.0)
        F[:, c0] = mask[:, p] & ia
        F[:, c0 + 1] = w * w
        F[:, c0 + 2] = w * s.yres
        F[:, c0 + 3:c0 + 3 + C] = w[:, None] * s.Xg
    base = 1 + P * (3 + C)
    F[:, base] = ia & sm["male"]
    F[:, base + 1:base + 1 + P] = (ia & sm["male"])[:, None] & mask
    return F, [0] + [1 + p * (3 + C) for p in range(P)] + list(range(base, base + 1 + P))


# ---------------------------------------------------------------------------------- 1. every route, exact counts
ROUTES = [("bed", True, False), ("bed_f64", False, True), ("bgen8", True, True), ("bed_bt", True, True),
          ("bgen8_bt", False, False)]


@pytest.mark.parametrize("route,drop,ref_first", ROUTES)
def test_chrx_route_counts_and_statistics(monkeypatch, route, drop, ref_first):
    """N = 5001 kept samples (Npad 5120: three 2048-sample dosage chunks), P = 3, C = 3 (23 feature columns with sex).
    A block of 256 variants with alternating non-PAR flags, a partial block of 77 with every flag set, then both blocks
    again: with every flag clear, and without rg_s2_set_non_par (the flags of a call do not reach the next one).  Each
    call against the exact reference, the statistics against the oracle and against a handle without sex."""
    P, C = 3, 3
    bt = route.endswith("_bt")
    hard = route.startswith("bed")
    sm = _samples(5004 if drop else 5001, P, seed=7 + len(route), drop=drop)
    rng = sm["rng"]
    if route == "bed_f64":
        monkeypatch.setenv("RG_B200_S2_STATS", "f64")
    else:
        monkeypatch.delenv("RG_B200_S2_STATS", raising=False)
    state = _bt_state(sm, C, seed=11) if bt else _qt_state(sm, C, seed=11)
    mk = _bt_handle if bt else _qt_handle
    sx, ns = mk(sm, state, 256, True), mk(sm, state, 256, False)
    blocks, refs = [], []
    for bs in (256, 77):
        a = _alt_counts(rng, bs, sm["male_f"])
        if hard:
            blk = _bed_rows(a, ref_first)
            d, unit, m = _calls(sm, a, "hard")
            graw = plink.decode_bed(blk, sm["n_file"], keep=sm["keep"], ref_first=ref_first)
            ival = np.zeros_like(graw)
        else:
            blk = _probs(rng, a, ref_first)
            d, unit, m = _calls(sm, a, "dose", *blk, ref_first=ref_first)
            graw, ival = obgen.dosage(blk[0][:, sm["keep"], 0].astype(np.float64), blk[0][:, sm["keep"], 1].astype(np.float64),
                                      m, ref_first=ref_first)
        blocks.append(blk)
        refs.append((d, unit, m, graw, ival))
    flags = [(np.arange(256) % 2 == 1).astype(np.uint8), np.ones(77, dtype=np.uint8)]
    ex_x = [_exact(sm, r[0], r[2], r[1], f) for r, f in zip(refs, flags)]
    ex_a = [_exact(sm, r[0], r[2], r[1], np.zeros_like(f)) for r, f in zip(refs, flags)]
    min_mac = _min_mac(list(zip(ex_x, ex_a)))
    out_x, out_a = [], []
    for blk, f in zip(blocks, flags):
        sx.set_non_par(f)
        out_x.append(_run(sx, route, blk, sm, ref_first, min_mac))
        pa = _paths(sx)
        assert pa["nchunks"] == 3 and pa["Npad"] == 5120
        assert (pa["bt_dp"] if bt else pa["dp"]) == 32
        assert pa["tc"] == (0 if route == "bed_f64" else 1)
        if not hard:                                                   # the sums, male columns exact
            rp = (len(f) + 127) // 128 * 128
            S4 = sx.debug("bt_sums", np.float64, rp * 4 * 32).reshape(rp, 4, 32)
            d, _, m = refs[len(out_x) - 1][:3]
            _, e, _ = _codes(blk[0], blk[1], sm["keep"], ref_first)
            F, cols01 = (_bt_F(sm, state, 32) if bt else _qt_F(sm, state, 32))
            _check_sums(S4, (d, d * d, m.astype(np.int64), e), F, list(range(0, len(f), 5)), cols01, 5120 + 3)
        out_a.append(_run(ns, route, blk, sm, ref_first, min_mac))
    # the same blocks with every flag clear, then without flags: the autosomal rule
    sx.set_non_par(np.zeros(256, dtype=np.uint8))
    clear = _run(sx, route, blocks[0], sm, ref_first, min_mac)
    after = _run(sx, route, blocks[1], sm, ref_first, min_mac)
    for k in ("ns", "ns_all", "af", "af_all", "mac", "mac_all", "flags"):
        assert np.array_equal(clear[k], out_a[0][k], equal_nan=k.startswith("af")), (route, "flags clear", k)
        assert np.array_equal(after[k], out_a[1][k], equal_nan=k.startswith("af")), (route, "after the flagged call", k)
    n_checked = 0
    for b in range(2):
        d, unit, m, graw, ival = refs[b]
        _check_counts(route, out_x[b], ex_x[b], sm, unit, flags[b], min_mac)
        _check_counts(route, out_a[b], ex_a[b], sm, unit, np.zeros_like(flags[b]), min_mac)
        if hard:
            _check_oracle_mac(route, ex_x[b], graw, sm, flags[b])
        ox, oa = out_x[b], out_a[b]
        assert np.array_equal(ox["flags"] & ~1, oa["flags"] & ~1), route
        _same_stats(route, ox, oa, exact=hard)
        if not hard:                                                   # INFO: the autosomal formula, sex plays no part
            ok = ex_x[b]["ok"]
            maskp = sm["mask"].astype(np.int64)
            _, e, _ = _codes(blocks[b][0], blocks[b][1], sm["keep"], ref_first)
            num = (255 * (np.where(ok, e, 0) @ maskp) - (np.where(ok, d * d, 0) @ maskp)) / 65025.0
            af = ox["af"]
            info = np.where((af == 0) | (af == 1), 1.0, 1.0 - num / (2 * ex_x[b]["ns"][:, 1:] * af * (1 - af)))
            bad = np.argwhere(np.abs(ox["info"] - info) > 1e-12)
            assert bad.size == 0, (route, "INFO", tuple(bad[0]), ox["info"][tuple(bad[0])], info[tuple(bad[0])])
            assert np.abs(ox["info"] - oa["info"]).max() <= 1e-12, route
        # the oracle, chrX rule
        for i in range(len(flags[b])):
            npar = bool(flags[b][i])
            if bt:
                for j in range(P):
                    r = step2_bt.score_bt(graw[i], ival[i], sm["ia"], sm["mask"][:, j], state["Y"][:, j], state["sts"][j],
                                          1e9, sm["N"], male=sm["male"], non_par=npar, min_mac=min_mac)
                    ignored = bool(ox["flags"][i] & 17) or ox["mac"][i, j] < min_mac
                    assert (r is None) == ignored, (route, i, j, ox["flags"][i], ox["mac"][i, j])
                    if r is None:
                        continue
                    assert abs(ox["stat"][i, j] - r["stat"]) <= 1e-8 * max(1.0, abs(r["stat"])), (route, i, j, ox["stat"][i, j], r["stat"])
                    n_checked += 1
                continue
            vs = step2.variant_stats(graw[i], sm["ia"], sm["mask"], male=sm["male"], non_par=npar)
            if vs["mac1"] < min_mac:
                assert ox["flags"][i] & 1, (route, i)
                continue
            sc = step2.score_qt(vs["g"], state["X"], state["res"], sm["mask"], sm["ia"], state["n_an"], C, state["scf"],
                                state["YtX"], False)
            assert bool(ox["flags"][i] & 2) == (sc is None), (route, i)
            if sc is None:
                continue
            for k, kk in (("beta", "beta"), ("se", "se"), ("chisq", "chisq")):
                for j in range(P):
                    assert abs(ox[k][i, j] - sc[kk][j]) <= 1e-8 * abs(sc[kk][j]), (route, k, i, j, ox[k][i, j], sc[kk][j])
            n_checked += 1
    sx.close()
    ns.close()
    assert n_checked > (300 if bt else 100), n_checked


# ------------------------------------------------------------------ 2. shapes where the male columns change the layout
@pytest.mark.parametrize("kind,C,P,before,after", [
    ("qt", 2, 3, dict(dp=16, drows=256), dict(dp=32, drows=256)),       # 15 -> 19 columns
    ("qt", 5, 3, dict(dp=32, drows=256), dict(dp=32, drows=512)),       # 27 -> 31: a third digit group of 14 columns
    ("bt", 2, 3, dict(bt_dp=16, drows=256), dict(bt_dp=32, drows=256)),  # 16 -> 20
])
def test_chrx_male_columns_change_the_layout(monkeypatch, kind, C, P, before, after):
    """The male columns alone push F over a 16-column tile or a 14-column digit group.  On hard calls (every 2-bit route
    sums exactly) the counts equal the exact reference, the 0/1 columns of the sums, the male ones included, equal the
    integer sums, and the statistics equal the handle without sex bit for bit."""
    monkeypatch.delenv("RG_B200_S2_STATS", raising=False)
    sm = _samples(1501, P, seed=40 + C, drop=False)
    rng = sm["rng"]
    bt = kind == "bt"
    state = _bt_state(sm, C, seed=12) if bt else _qt_state(sm, C, seed=12)
    mk = _bt_handle if bt else _qt_handle
    route = "bed_bt" if bt else "bed"
    sx, ns = mk(sm, state, 128, True), mk(sm, state, 128, False)
    a = _alt_counts(rng, 128, sm["male_f"])
    blk = _bed_rows(a, False)
    d, unit, m = _calls(sm, a, "hard")
    flags = (rng.random(128) < 0.6).astype(np.uint8)
    sx.set_non_par(flags)
    ox = _run(sx, route, blk, sm, False, 5.0)
    px = _paths(sx)
    oa = _run(ns, route, blk, sm, False, 5.0)
    pn = _paths(ns)
    for k, v in before.items():
        assert pn[k] == v, (kind, C, P, "without sex", k, pn[k])
    for k, v in after.items():
        assert px[k] == v, (kind, C, P, "with sex", k, px[k])
    ex = _exact(sm, d, m, unit, flags)
    _check_counts(route, ox, ex, sm, unit, flags, 5.0)
    _same_stats(route, ox, oa, exact=True)
    dp = px["bt_dp" if bt else "dp"]
    planes = 4 if bt else 3
    S = sx.debug("bt_sums" if bt else "s2_sums", np.float64, 128 * planes * dp).reshape(128, planes, dp)
    F, cols01 = (_bt_F(sm, state, dp) if bt else _qt_F(sm, state, dp))
    F01 = F[:, cols01].astype(np.int64)
    for k, z in enumerate((d, d * d, m.astype(np.int64))):
        assert np.array_equal(S[:, k][:, cols01], (z @ F01).astype(np.float64)), (kind, "0/1 column sums", k)
    sx.close()
    ns.close()


# ----------------------------------------------------------------------------------------- 3. the call protocol
def _small(seed=60, P=2):
    sm = _samples(1501, P, seed=seed, drop=False)
    a = _alt_counts(sm["rng"], 96, sm["male_f"])
    d, _, m = _calls(sm, a, "hard")
    return sm, _bed_rows(a, False), d, m


def test_chrx_flags_cross_trait_kinds():
    """A handle that holds both kinds: the flags apply to the next call whatever its kind, then are gone."""
    sm, blk, d, m = _small()
    q, b = _qt_state(sm, 3, seed=1), _bt_state(sm, 3, seed=1)
    st = _bt_handle(sm, b, 96, True)
    st.set_chr(q["res"], q["scf"])
    flags = np.ones(96, dtype=np.uint8)
    ex_x, ex_a = _exact(sm, d, m, 1, flags), _exact(sm, d, m, 1, 0 * flags)
    st.set_non_par(flags)
    o1 = st.block_bed_bt(blk, min_mac=5.0)
    _check_counts("bed_bt then bed", o1, ex_x, sm, 1, flags, 5.0)
    o2 = st.block_bed(blk, min_mac=5.0)
    _check_counts("bed after bed_bt", o2, ex_a, sm, 1, 0 * flags, 5.0)
    st.set_non_par(flags)
    o3 = st.block_bed(blk, min_mac=5.0)
    _check_counts("bed", o3, ex_x, sm, 1, flags, 5.0)
    o4 = st.block_bed_bt(blk, min_mac=5.0)
    _check_counts("bed_bt after bed", o4, ex_a, sm, 1, 0 * flags, 5.0)
    assert sum(int(x != y) for x, y in zip(ex_x["mac"][:, 0], ex_a["mac"][:, 0])) > 40
    st.close()


def test_chrx_flags_without_sex_and_set_sex_timing():
    """Flags without sex information follow the autosomal rule.  rg_s2_set_sex takes effect at the next
    rg_s2_set_chr: set after it, the flags still follow the autosomal rule; cleared after it, the males still count half."""
    sm, blk, d, m = _small(seed=61)
    q = _qt_state(sm, 3, seed=2)
    flags = np.ones(96, dtype=np.uint8)
    ex_x, ex_a = _exact(sm, d, m, 1, flags), _exact(sm, d, m, 1, 0 * flags)
    st = _qt_handle(sm, q, 96, False)
    st.set_non_par(flags)
    _check_counts("no sex", st.block_bed(blk), ex_a, sm, 1, 0 * flags, 5.0)
    st.set_sex(None)
    st.set_chr(q["res"], q["scf"])
    st.set_non_par(flags)
    _check_counts("set_sex(None)", st.block_bed(blk), ex_a, sm, 1, 0 * flags, 5.0)
    st.set_sex(sm["male"])                                           # after rg_s2_set_chr: not yet
    st.set_non_par(flags)
    _check_counts("set_sex after set_chr", st.block_bed(blk), ex_a, sm, 1, 0 * flags, 5.0)
    assert _paths(st)["dp"] == 16                                    # 14 columns: no male columns yet
    st.set_chr(q["res"], q["scf"])
    st.set_non_par(flags)
    _check_counts("next set_chr", st.block_bed(blk), ex_x, sm, 1, flags, 5.0)
    assert _paths(st)["dp"] == 32                                    # 14 + 1 + P
    st.set_sex(None)                                                 # cleared after rg_s2_set_chr: still in effect
    st.set_non_par(flags)
    _check_counts("set_sex(None) after set_chr", st.block_bed(blk), ex_x, sm, 1, flags, 5.0)
    st.set_chr(q["res"], q["scf"])
    st.set_non_par(flags)
    _check_counts("cleared at set_chr", st.block_bed(blk), ex_a, sm, 1, 0 * flags, 5.0)
    st.close()


@pytest.mark.parametrize("route", ["bed", "bgen8", "bed_bt", "bgen8_bt"])
def test_chrx_short_flags_refused(route):
    """rg_s2_set_non_par with fewer flags than the block has variants: the call is refused with its message, the flags
    are dropped, and the next call on the handle works under the autosomal rule."""
    from regenie_b200 import capi
    sm = _samples(1501, 2, seed=62, drop=False)
    a = _alt_counts(sm["rng"], 96, sm["male_f"])
    bt = route.endswith("_bt")
    state = _bt_state(sm, 3, seed=3) if bt else _qt_state(sm, 3, seed=3)
    st = (_bt_handle if bt else _qt_handle)(sm, state, 96, True)
    if route.startswith("bed"):
        blk = _bed_rows(a, False)
        d, unit, m = _calls(sm, a, "hard")
    else:
        blk = _probs(sm["rng"], a, False)
        d, unit, m = _calls(sm, a, "dose", *blk)
    st.set_non_par(np.ones(95, dtype=np.uint8))
    with pytest.raises(capi.RgError, match="fewer flags than the block has variants"):
        _run(st, route, blk, sm, False, 5.0)
    o = _run(st, route, blk, sm, False, 5.0)
    _check_counts(route, o, _exact(sm, d, m, unit, np.zeros(96, dtype=bool)), sm, unit, np.zeros(96, dtype=bool), 5.0)
    st.set_non_par(np.ones(96, dtype=np.uint8))
    o = _run(st, route, blk, sm, False, 5.0)
    _check_counts(route, o, _exact(sm, d, m, unit, np.ones(96, dtype=bool)), sm, unit, np.ones(96, dtype=bool), 5.0)
    st.close()


# ---------------------------------------------------------------------------- 4. Firth and SPA on a chrX block
def test_chrx_firth_spa():
    """rg_s2_block_bgen8_bt on chrX, C = 2, P = 3 (16 feature columns, 20 with sex: dp 16 -> 32), N = 4501: Firth and SPA
    on every (variant, trait) with |z| > 0.5 whose chrX MAC passes.  Equal bit for bit to the same selections on a handle
    without sex, except Firth where the chrX MAC and the autosomal one lie on either side of 50 (the carriers-only
    iterations of a sparse variant): there, and everywhere, within the oracle's tolerances of the chrX rule."""
    P, C, bs, z_thr, min_mac = 3, 2, 192, 0.5, 5.25
    sm = _samples(4501, P, seed=70, drop=False)
    rng = sm["rng"]
    b = _bt_state(sm, C, seed=70)
    a = _alt_counts(rng, bs, sm["male_f"])
    lo = bs // 2                                                      # rare rows: carriers with fractional dosages
    car = rng.random((bs - lo, sm["n_file"])) < 0.008
    a[lo:] = np.where(car, np.where(sm["male_f"][None, :], 2, 1), 0)
    probs, miss = _probs(rng, a, False)
    d, unit, m = _calls(sm, a, "dose", probs, miss)
    sx, ns = _bt_handle(sm, b, 256, True), _bt_handle(sm, b, 256, False)
    flags = np.ones(bs, dtype=np.uint8)
    sx.set_non_par(flags)
    ox = sx.block_bgen8_bt(probs, miss, min_mac=min_mac)
    assert _paths(sx)["bt_dp"] == 32
    oa = ns.block_bgen8_bt(probs, miss, min_mac=min_mac)
    assert _paths(ns)["bt_dp"] == 16
    ex_x = _exact(sm, d, m, unit, flags)
    sel = [(i, j) for i in range(bs) for j in range(P)
           if not (ox["flags"][i] & 17) and ox["mac"][i, j] >= min_mac and abs(ox["stat"][i, j]) > z_thr]
    assert sel == [(i, j) for i in range(bs) for j in range(P)
                   if ex_x["mac"][i, 0] >= min_mac and not (ox["flags"][i] & 16) and ex_x["mac"][i, 1 + j] >= min_mac
                   and abs(ox["stat"][i, j]) > z_thr]
    vi, ti = [v for v, _ in sel], [t for _, t in sel]
    fx, fa = sx.firth(vi, ti), ns.firth(vi, ti)
    px, pa = sx.spa(vi, ti), ns.spa(vi, ti)
    for u, w in zip(px, pa):
        assert np.array_equal(u, w, equal_nan=u.dtype.kind == "f"), "SPA"
    n_straddle = n_firth = 0
    g, ival = obgen.dosage(probs[:, :, 0].astype(np.float64), probs[:, :, 1].astype(np.float64), m)
    for n, (i, j) in enumerate(sel):
        straddle = (ox["mac"][i, j] < 50) != (oa["mac"][i, j] < 50) and bool(ox["flags"][i] & 4)
        n_straddle += straddle
        if not straddle:
            for u, w in zip(fx, fa):
                assert u[n] == w[n] or (np.isnan(u[n]) and np.isnan(w[n])), ("Firth", i, j, u[n], w[n])
        r = step2_bt.score_bt(g[i], ival[i], sm["ia"], sm["mask"][:, j], b["Y"][:, j], b["sts"][j], z_thr, sm["N"],
                              male=sm["male"], non_par=True)
        assert r is not None and (fx[3][n] & 15) == int(r["test_fail"]), ("Firth", i, j, fx[3][n])
        if not r["test_fail"]:
            n_firth += 1
            for u, w in zip((fx[0][n], fx[1][n], fx[2][n]), (r["beta"], r["se"], r["chisq"])):
                assert abs(u - w) <= 1e-5 * max(abs(w), 1e-8), ("Firth", i, j, u, w)
        rs = step2_bt.score_bt(g[i], ival[i], sm["ia"], sm["mask"][:, j], b["Y"][:, j], b["sts"][j], z_thr, sm["N"],
                               male=sm["male"], non_par=True, correction="spa")
        assert bool(px[1][n] & 15) == rs["test_fail"], ("SPA", i, j, px[1][n])
        if not rs["test_fail"]:
            chisq = step2_bt.chisq1_from_pvalue(max(step2_bt.NL_DBL_DMIN, px[0][n]))
            assert abs(chisq - rs["chisq"]) <= 1e-5 * rs["chisq"], ("SPA", i, j, chisq, rs["chisq"])
    assert len(sel) > 150 and n_firth > 100 and n_straddle > 0, (len(sel), n_firth, n_straddle)
    sx.close()
    ns.close()


# -------------------------------------------------------------------------------------------- 5. GxE on a chrX block
def _thresholds(mx, ma, lo_q, hi_q):
    """A min_mac and a rare_mac between quantiles of the chrX MACs at which some pairs change side only under the male
    rule (MACs are halves, so a threshold at a quarter is never hit)."""
    def pick(q, le):
        best = None
        for t in np.quantile(mx, np.linspace(q - 0.1, q + 0.1, 21)):
            t = math.floor(t) + 0.25
            moved = int(((mx <= t) != (ma <= t)).sum() if le else ((mx < t) != (ma < t)).sum())
            if best is None or moved > best[1]:
                best = (t, moved)
        assert best[1] > 0
        return best[0]
    return pick(lo_q, False), pick(hi_q, True)


def test_chrx_interaction_qt():
    """rg_s2_interaction on a chrX block: robust route with HC4 forced below rare_mac.  The skip (min_mac) and the HC4
    switch (MAC <= rare_mac) read the chrX MAC of the resident block; the oracle gets the exact chrX MAC."""
    P, C, bs = 2, 3, 120
    sm = _samples(1501, P, seed=80, drop=False)
    rng = sm["rng"]
    q = _qt_state(sm, C, seed=80)
    st = _qt_handle(sm, q, bs, True)
    E = np.where(sm["ia"], rng.normal(size=sm["N"]) * 1.5 + 0.3, 0.0)
    st.set_interaction(E)
    a = _alt_counts(rng, bs, sm["male_f"])
    blk = _bed_rows(a, False)
    d, _, m = _calls(sm, a, "hard")
    flags = np.ones(bs, dtype=np.uint8)
    ex_x, ex_a = _exact(sm, d, m, 1, flags), _exact(sm, d, m, 1, 0 * flags)
    mx = np.array([[float(x) for x in r] for r in ex_x["mac"][:, 1:]])
    ma = np.array([[float(x) for x in r] for r in ex_a["mac"][:, 1:]])
    min_mac, rare_mac = _thresholds(mx, ma, 0.2, 0.6)
    st.set_non_par(flags)
    o = st.block_bed(blk, min_mac=0.5)
    assert np.array_equal(o["mac"], mx)
    status, coef, vcov = st.interaction(bs, rare_mac=rare_mac, min_mac=min_mac, force_robust=True, force_hc4=True)
    graw = plink.decode_bed(blk, sm["n_file"])
    gimp, _ = plink.mean_impute_block(graw, sm["ia"])
    n_skip = n_hc4 = n_ok = 0
    for v in range(bs):
        if o["flags"][v] & 3:
            assert (status[v] == 0).all()
            continue
        r = io.robust(gimp[v], E, q["X"], q["res"], sm["mask"], q["scf"], q["n_an"], mx[v], rare_mac, True, False)
        for i in range(P):
            if mx[v, i] < min_mac:
                assert status[v, i] == 0, ("skip", v, i, mx[v, i])
                n_skip += ma[v, i] >= min_mac
                continue
            if r is None:
                assert status[v, i] in (0, -1)
                continue
            assert status[v, i] == 1, (v, i, status[v, i])
            se = np.sqrt(np.diag(vcov[v, i]))
            want_se = np.sqrt(np.diag(r[1][i]))
            assert np.allclose(coef[v, i], r[0][i], rtol=1e-5, atol=0) and np.allclose(se, want_se, rtol=1e-5, atol=0), \
                (v, i, "MAC %g rare_mac %g" % (mx[v, i], rare_mac), coef[v, i], r[0][i], se, want_se)
            n_hc4 += (mx[v, i] <= rare_mac) != (ma[v, i] <= rare_mac)
            n_ok += 1
    assert n_skip > 0 and n_hc4 > 0 and n_ok > 100, (n_skip, n_hc4, n_ok)
    st.close()


def test_chrx_interaction_bt():
    """rg_s2_interaction_bt on a chrX block: the robust / model-based choice MAC > rare_mac and the min_mac skip read the
    chrX MAC; the oracle gets the exact chrX MAC."""
    P, C, bs = 2, 3, 120
    sm = _samples(1501, P, seed=90, drop=False)
    rng = sm["rng"]
    ia, mask, N = sm["ia"], sm["mask"], sm["N"]
    E = np.where(ia, rng.normal(size=N) * 1.5 + 0.3, 0.0)
    X, _ = get_basis(np.column_stack([np.ones(N), rng.standard_normal((N, C - 1)), E, E * E]) * ia[:, None])
    Y = ((rng.random((N, P)) < 0.35) & mask).astype(np.float64)
    blup = 0.2 * rng.standard_normal((N, P))
    sts = [step2_bt.BtChrom(Y[:, j], X, blup[:, j], mask[:, j]) for j in range(P)]
    off = np.stack([blup[:, j] * mask[:, j] + X @ sts[j].beta0 for j in range(P)], 1)
    b = dict(X=X, Y=Y, sts=sts, n_an=int(ia.sum()), C=X.shape[1])
    st = _bt_handle(sm, b, bs, True)
    st.set_interaction_bt(E, off)
    a = _alt_counts(rng, bs, sm["male_f"])
    blk = _bed_rows(a, False)
    d, _, m = _calls(sm, a, "hard")
    flags = np.ones(bs, dtype=np.uint8)
    ex_x, ex_a = _exact(sm, d, m, 1, flags), _exact(sm, d, m, 1, 0 * flags)
    mx = np.array([[float(x) for x in r] for r in ex_x["mac"][:, 1:]])
    ma = np.array([[float(x) for x in r] for r in ex_a["mac"][:, 1:]])
    min_mac, rare_mac = _thresholds(mx, ma, 0.2, 0.6)
    st.set_non_par(flags)
    o = st.block_bed_bt(blk, min_mac=0.5)
    assert np.array_equal(o["mac"], mx)
    status, coef, vcov = st.interaction_bt(rare_mac=rare_mac, min_mac=min_mac)
    graw = plink.decode_bed(blk, sm["n_file"])
    gimp, _ = plink.mean_impute_block(graw, ia)
    n_skip = n_route = n_ok = 0
    for v in range(bs):
        if o["flags"][v] & 1:
            assert (status[v] == 0).all()
            continue
        flipped = bool(o["flags"][v] & 8)
        g = np.where(ia, 2.0 - gimp[v], 0.0) if flipped else gimp[v]
        dsg = ibo.design(g, E, X, b["n_an"])
        for i in range(P):
            if mx[v, i] < min_mac or dsg is None:
                assert status[v, i] == 0, ("skip", v, i, mx[v, i])
                n_skip += dsg is not None and ma[v, i] >= min_mac
                continue
            so, beta, V = ibo.wald(dsg[0], Y[:, i], off[:, i], mask[:, i], mx[v, i], rare_mac)
            assert status[v, i] == so, (v, i, "MAC %g rare_mac %g" % (mx[v, i], rare_mac), status[v, i], so)
            if so < 0:
                continue
            n_route += (mx[v, i] > rare_mac) != (ma[v, i] > rare_mac)
            cw, Vw = ibo.printed(beta, V, dsg[1], dsg[2], flipped)
            se, want_se = np.sqrt(np.diag(vcov[v, i])), np.sqrt(np.diag(Vw))
            assert np.allclose(coef[v, i], cw, rtol=1e-5, atol=1e-10) and np.allclose(se, want_se, rtol=1e-5, atol=1e-10), \
                (v, i, coef[v, i], cw, se, want_se)
            n_ok += 1
    assert n_skip > 0 and n_route > 0 and n_ok > 60, (n_skip, n_route, n_ok)
    st.close()
