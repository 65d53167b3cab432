"""Step-2 kernel paths that the input's shape selects, each against a plain reference.

Step 2 forms every statistic from code-wise sums  S1 = sum g F,  S2 = sum g^2 F,  Sm = sum miss F  (and Se = sum e F for
dosages, e = 4 p_hom + p_het) of one per-sample feature row F, and picks the kernels that form them from the input:
  * 2-bit rows (.bed / .pgen): three int8 planes (g, g^2, missing), built from the 2-bit rows inside the Gram kernel,
    against radix-30 digit rows of F on the tensor cores, over sample chunks that keep 60 * chunk < 2^24
    (ceil(Npad / 2^18) chunks, more when the tiles would not fill the SMs), every digit sum an exact integer, FP64
    Horner after.  RG_B200_S2_STATS=f64, read at every rg_s2_set_chr, selects the FP64 CUDA-core kernel over chunks of
    2048 samples instead;
  * 8-bit dosages: dosage_relayout_kernel (one 8-byte load per four samples when they are consecutive and the address is
    8-byte aligned, per-sample loads otherwise: odd file rows mix both) and dosage_stats_kernel over chunks of 2048
    samples and tiles of 16 feature columns, the last tile partly live, then a fixed-order sum of the chunks and of
    the non-zero / hom-alt counts;
  * binary traits add the Firth and SPA kernels on the resident block, 256 selections per launch.
Every test asserts through the "s2_paths" hook which path ran and how many chunks it used.  N, A1FREQ, MAC and the flags
are checked bit for bit against numpy integer sums, the statistics against the numpy oracle at 1e-8 relative (Firth and
SPA at 1e-5), and the sums themselves (hooks "s2_sums", "bt_sums") against a long-double recomputation from F, held to
the error bound of the kernel's arithmetic; the 0/1 columns of F must come out exact.
"""
import math

import numpy as np
import pytest

import helpers
from oracle import bgen as obgen
from oracle import plink, prep, step2, step2_bt

pytestmark = pytest.mark.gpu
U = 2.0 ** -53
LD = np.longdouble
K255 = 1.0 / 255.0
PATH_KEYS = ("tc", "nchunk", "chunk_len", "drows", "nchunks", "Npad", "dp", "bt_dp")


def _paths(st):
    return dict(zip(PATH_KEYS, (int(x) for x in st.debug("s2_paths", np.int64, 8))))


def _probs(rng, bs, n, miss_frac=0.02):
    p0 = rng.integers(0, 256, size=(bs, n))
    p1 = (rng.random((bs, n)) * (256 - p0)).astype(np.int64)
    certain = rng.random((bs, n)) < 0.7                      # most calls are (nearly) hard calls
    g = rng.integers(0, 3, size=(bs, n))
    p0 = np.where(certain, (g == 2) * 255, p0)
    p1 = np.where(certain, (g == 1) * 255, p1)
    probs = np.stack([p0, p1], axis=2).astype(np.uint8)
    miss = np.where(rng.random((bs, n)) < miss_frac, 0x82, 0x02).astype(np.uint8)
    return probs, miss


def _hard(g, ref_first):
    """Probability pair of hard dosage g (ALT allele count) in the file's allele order."""
    hom = 0 if ref_first else 2
    return np.stack([(g == hom) * 255, (g == 1) * 255], axis=-1).astype(np.uint8)


def _basis(ia, cov):
    """Orthonormal basis of [1 | cov] over the analysed samples, zero rows elsewhere."""
    X = np.zeros((len(ia), cov.shape[1] + 1))
    X[ia], _ = np.linalg.qr(np.hstack([np.ones((int(ia.sum()), 1)), cov[ia]]))
    return np.asfortranarray(X)


def _qt_problem(N, P, C, seed, all_analysed=False):
    rng = np.random.default_rng(seed)
    ia = np.ones(N, dtype=bool)
    if not all_analysed:
        ia[rng.choice(N, N // 50, replace=False)] = False
    X = _basis(ia, rng.standard_normal((N, C - 1)))
    mask = ia[:, None] & (rng.random((N, P)) > 0.05)
    n_an = int(ia.sum())
    res = rng.standard_normal((N, P)) * mask
    res = np.asfortranarray(res / (np.linalg.norm(res, axis=0) / np.sqrt(n_an - C)))
    return dict(N=N, P=P, C=C, ia=ia, X=X, mask=mask, n_an=n_an, res=res, scf=rng.uniform(0.5, 2.0, P), YtX=res.T @ X)


def _qt_F(pb, dp):
    """The feature row of rg_s2_set_chr: [a | x | res | m | m_p x_c], zero-padded to dp columns."""
    N, C, P = pb["N"], pb["C"], pb["P"]
    F = np.zeros((N, dp))
    F[:, 0] = pb["ia"]
    F[:, 1:1 + C] = pb["X"]
    F[:, 1 + C:1 + C + P] = pb["res"]
    F[:, 1 + C + P:1 + C + 2 * P] = pb["mask"]
    for p in range(P):
        F[:, 1 + C + 2 * P + p * C:1 + C + 2 * P + (p + 1) * C] = pb["mask"][:, p:p + 1] * pb["X"]
    return F


def _qt_01_cols(C, P):
    return [0] + list(range(1 + C + P, 1 + C + 2 * P))


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


def _same_stats(a, b, tol=1e-9):
    """Two statistics paths on the same calls: stat within tol * max(1, |stat|) (a statistic near 0 is a difference of
    O(1) terms, so its error is absolute), BETA = stat * SE within the same error times SE, SE within tol relative."""
    assert np.all(np.abs(a["stat"] - b["stat"]) <= tol * np.maximum(1.0, np.abs(b["stat"]))), "stat"
    assert np.all(np.abs(a["beta"] - b["beta"]) <= tol * (np.abs(b["beta"]) + np.abs(b["se"]))), "beta"
    np.testing.assert_allclose(a["se"], b["se"], rtol=tol, atol=0, err_msg="se")


def _edge_rows(rng, n_file, ref_first, with_missing):
    """Seven rows that sit on the branches of the finish: all missing, monomorphic 0, all dosage 2, all heterozygous,
    one carrier, a rare (sparse) row and one fractional call among hard calls."""
    g = np.zeros((7, n_file), dtype=np.int64)
    g[2] = 2
    g[3] = 1
    g[4, n_file // 3] = 2
    g[5, rng.choice(n_file, n_file // 100, replace=False)] = 1
    g[6] = rng.integers(0, 3, size=n_file)
    probs = _hard(g, ref_first)
    probs[6, n_file // 2] = (100, 80)
    miss = np.where(rng.random((7, n_file)) < 0.02, 0x82, 0x02).astype(np.uint8)
    miss[0] = 0x82
    if not with_missing:
        g[0] = rng.integers(0, 3, size=n_file)
        probs[0] = _hard(g[0], ref_first)
    return probs, miss


# ------------------------------------------------------------------------------------------ 1. QT on fractional dosages
@pytest.mark.parametrize("n_file,P,ref_first,with_missing", [
    (5004, 1, 0, True), (5001, 3, 1, True), (5001, 20, 0, True), (5004, 20, 1, True), (5001, 3, 0, False)])
def test_qt_fractional_dosages(n_file, P, ref_first, with_missing):
    """rg_s2_block_bgen8 on ~30 % fractional calls: N = 5001 kept samples (Npad 5120: three FP64 chunks, the last one
    partial), odd rows (misaligned every other row) or three removed samples; P = 20 gives 104 feature columns, seven
    column tiles with half of the last one live.  A full block of 256 variants and a partial one of 77."""
    from regenie_b200 import capi
    C = 3
    rng = np.random.default_rng(100 + n_file + P + 7 * ref_first)
    keep = np.ones(n_file, dtype=bool)
    if n_file == 5004:
        keep[[2, 2501, 5003]] = False
    sample_idx = np.nonzero(keep)[0].astype(np.int32) if not keep.all() else None
    N = int(keep.sum())
    pb = _qt_problem(N, P, C, seed=n_file + P)
    strict = P == 1
    st = capi.Step2(pb["X"], pb["mask"], pb["ia"], pb["n_an"], 256, strict=strict)
    st.set_chr(pb["res"], pb["scf"])
    n_checked = n_sparse = n_flag2 = 0
    for bs in (256, 77):
        probs, miss = _probs(rng, bs, n_file)
        ep, em = _edge_rows(rng, n_file, ref_first, with_missing)
        probs[:7], miss[:7] = ep, em
        miss = miss if with_missing else None
        o = st.block_bgen8(probs, miss, sample_idx=sample_idx, ref_first=bool(ref_first))
        pa = _paths(st)
        assert (pa["nchunks"], pa["Npad"]) == (3, 5120)
        dp = pa["dp"]
        assert dp == ((1 + C + 2 * P + P * C + 15) // 16) * 16
        d, e, m = _codes(probs, miss, keep, ref_first)
        # sums of the dosage statistics kernel (integer units) and their scaling
        rp = (bs + 127) // 128 * 128
        S4 = st.debug("bt_sums", np.float64, rp * 4 * dp).reshape(rp, 4, dp)
        S3 = st.debug("s2_sums", np.float64, rp * 3 * dp).reshape(rp, 3, dp)
        assert np.array_equal(S3[:, 0], S4[:, 0] * K255) and np.array_equal(S3[:, 1], S4[:, 1] * K255 * K255)
        assert np.array_equal(S3[:, 2], S4[:, 2])
        F = _qt_F(pb, dp)
        rows = list(range(7)) + list(range(7, bs, 9))
        _check_sums(S4, (d, d * d, m.astype(np.int64), e), F, rows, _qt_01_cols(C, P), 5120 + 3)
        assert not S4[bs:].any()                                       # padding rows stay empty
        nnz = st.debug("bt_nnz", np.float64, rp)[:bs]
        ia, mask = pb["ia"], pb["mask"]
        ok = ~m & ia[None, :]
        assert np.array_equal(nnz, ((d != 0) & ok).sum(axis=1).astype(float))
        assert np.array_equal(st.debug("bt_n510", np.float64, rp)[:bs], ((d == 510) & ok).sum(axis=1).astype(float))
        # counts, A1FREQ, MAC, flags: bit for bit from the integer sums
        ns1 = ok.sum(axis=1)
        tot1 = np.where(ok, d, 0).sum(axis=1).astype(np.float64) * K255
        assert np.array_equal(o["ns_all"], ns1)
        np.testing.assert_array_equal(o["af_all"], tot1 / (2.0 * ns1))
        mac1 = np.minimum(tot1, 2.0 * ns1 - tot1)
        assert np.array_equal(o["mac_all"], mac1)
        okp = ok[:, :, None] & mask[None, :, :]                        # [variant, sample, trait]
        nsp = okp.sum(axis=1)
        totp = np.einsum("vs,vsp->vp", np.where(ok, d, 0), okp).astype(np.float64) * K255
        assert np.array_equal(o["ns"], nsp)
        np.testing.assert_array_equal(o["af"], totp / (2.0 * nsp))
        np.testing.assert_array_equal(o["mac"], np.minimum(totp, 2.0 * nsp - totp))
        assert np.array_equal(o["flags"] & 1, (mac1 < 5.0).astype(np.int32))
        mu = tot1 / ns1
        sparse = (nnz + np.where(mu != 0.0, (m & ia[None, :]).sum(axis=1), 0)) <= N * 0.5
        assert np.array_equal((o["flags"] & 4) != 0, sparse)
        for i in range(bs):
            g, ival = obgen.dosage(probs[i, keep, 0].astype(np.float64), probs[i, keep, 1].astype(np.float64),
                                   m[i], ref_first=bool(ref_first))
            vs = step2.variant_stats(g, ia, mask)
            assert o["ns_all"][i] == vs["ns1"] and np.array_equal(o["ns"][i], vs["ns"])
            if vs["ignored"]:
                assert o["flags"][i] & 1, i
                continue
            # the oracle sums N rounded dosages p / 255 (and 1 - a - b for ref-first): its own error is below (N + 3) U
            np.testing.assert_allclose(o["af"][i], vs["af"], rtol=(N + 3) * U, atol=0)
            info_p = np.array([ival[ok[i] & mask[:, p]].sum() for p in range(P)])
            af = vs["af"]
            info = np.where((af == 0) | (af == 1), 1.0, 1.0 - info_p / (2 * vs["ns"] * af * (1 - af)))
            assert np.abs(o["info"][i] - info).max() <= 1e-12, (i, o["info"][i], info)
            sc = step2.score_qt(vs["g"], pb["X"], pb["res"], mask, ia, pb["n_an"], C, pb["scf"], pb["YtX"], strict)
            assert bool(o["flags"][i] & 2) == (sc is None), i
            if sc is None:
                n_flag2 += 1
                continue
            assert bool(o["flags"][i] & 4) == sc["is_sparse"]
            n_sparse += sc["is_sparse"]
            for k in ("beta", "se", "chisq"):
                np.testing.assert_allclose(o[k][i], sc[k], rtol=1e-8, atol=0, err_msg="%s row %d" % (k, i))
            n_checked += 1
    st.close()
    assert n_checked > 250 and n_sparse >= 2 and n_flag2 == 2


# ----------------------------------------------------------------- 2. QT: dosage path and 2-bit path on the same hard calls
def test_qt_dosage_and_2bit_paths_agree_on_hard_calls():
    from regenie_b200 import capi, synth
    N, M, P, C = 3001, 256, 3, 3
    pb = _qt_problem(N, P, C, seed=21)
    g = synth.genotypes(N, M, seed=21, miss=0.02)
    g[7] = np.where(g[7] == 3, 3, 0)
    g[7, 5:12] = 1                                                    # rare: sparse branch
    packed = synth.pack_bed(g)
    graw = plink.decode_bed(packed, N)
    probs = np.zeros((M, N, 2), dtype=np.uint8)
    probs[:, :, 0] = (graw == 2) * 255
    probs[:, :, 1] = (graw == 1) * 255
    miss = np.where(graw == plink.MISSING_G, 0x82, 0x02).astype(np.uint8)
    st = capi.Step2(pb["X"], pb["mask"], pb["ia"], pb["n_an"], M)
    st.set_chr(pb["res"], pb["scf"])
    ob = st.block_bed(packed)
    assert _paths(st)["tc"] == 1
    od = st.block_bgen8(probs, miss)
    for k in ("ns", "ns_all", "af", "af_all", "mac", "mac_all", "flags"):
        assert np.array_equal(ob[k], od[k]), k
    assert (ob["flags"] & 4).any() and not (ob["flags"] & 4).all()
    _same_stats(od, ob)
    st.close()


# ------------------------------------------------------- 3. BT on fractional dosages, two column tiles, Firth and SPA
def _bt_problem(N, P, C, seed):
    rng = np.random.default_rng(seed)
    ia = np.ones(N, dtype=bool)
    ia[rng.choice(N, N // 60, replace=False)] = False
    cov = rng.standard_normal((N, C - 1))
    X = np.hstack([np.ones((N, 1)), cov]) * ia[:, None]
    mask = ia[:, None] & (rng.random((N, P)) > 0.04)
    eta = -0.8 + cov @ rng.normal(0, 0.4, size=(C - 1, P))
    Y = ((rng.random((N, P)) < 1 / (1 + np.exp(-eta))) & mask).astype(np.float64)
    blup = 0.3 * rng.standard_normal((N, P)) * mask
    sts = [step2_bt.BtChrom(Y[:, j], X, blup[:, j], mask[:, j]) for j in range(P)]
    return dict(N=N, P=P, C=C, ia=ia, X=X, mask=mask, Y=Y, sts=sts, n_an=int(ia.sum()))


def _bt_F(b, dp):
    """The feature row of rg_s2_set_chr_bt: [a | per trait: m | w^2 | w yres | w XGamma_c]."""
    N, P, C, ia = b["N"], b["P"], b["C"], b["ia"]
    F = np.zeros((N, dp))
    F[:, 0] = ia
    for p, s in enumerate(b["sts"]):
        c0 = 1 + p * (3 + C)
        w = np.where(ia, s.gamma_sqrt_mask, 0.0)
        F[:, c0] = b["mask"][:, p] & ia
        F[:, c0 + 1] = w * w
        F[:, c0 + 2] = w * s.yres
        F[:, c0 + 3:c0 + 3 + C] = w[:, None] * s.Xg
    return F


def _bt_handle(b, max_bs):
    from regenie_b200 import capi
    sts = b["sts"]
    st = capi.Step2(b["X"], b["mask"], b["ia"], b["n_an"], max_bs)
    st.set_chr_bt(np.stack([s.gamma_sqrt_mask for s in sts], 1), np.stack([s.gamma_sqrt for s in sts], 1),
                  np.stack([s.yres for s in sts], 1), [s.Xg for s in sts], b["Y"],
                  np.stack([s.cov_blup_offset for s in sts], 1), np.stack([s.phat for s in sts], 1))
    return st


def test_bt_fractional_dosages_firth_spa():
    """N = 4501 (Npad 4608: three chunks), P = 3, C = 3: 19 feature columns, two column tiles.  Common fractional
    variants (half of them flipped), rare variants whose carriers hold fractional dosages below 0.5 (the carriers-only
    Firth iterations) and their flipped mirror images; Firth and SPA on every (variant, trait) with |z| > 0.5, more
    than 256 selections in one call, and the same selections in two smaller calls give the same bits."""
    N, P, C, bs, z_thr = 4501, 3, 3, 192, 0.5
    rng = np.random.default_rng(41)
    b = _bt_problem(N, P, C, seed=41)
    probs, miss = _probs(rng, bs, N, miss_frac=0.01)
    for lo, hi, flip in ((64, 128, False), (128, 192, True)):       # rare: ~0.6 % carriers with dosage in (0, 0.8]
        car = rng.random((hi - lo, N)) < 0.006
        x = np.where(car, rng.integers(1, 205, size=(hi - lo, N)), 0)
        probs[lo:hi, :, 1] = x                                         # dosage x / 255, or 2 - x / 255 when flipped
        probs[lo:hi, :, 0] = 255 - x if flip else 0
    probs[0] = _hard(np.ones(N, dtype=np.int64), False)             # every sample heterozygous: den = 0, flag 16
    st = _bt_handle(b, 256)
    o = st.block_bgen8_bt(probs, miss, min_mac=5.0)
    pa = _paths(st)
    assert (pa["nchunks"], pa["Npad"], pa["bt_dp"]) == (3, 4608, 32)
    keep = np.ones(N, dtype=bool)
    d, e, m = _codes(probs, miss, keep, False)
    S4 = st.debug("bt_sums", np.float64, 256 * 4 * 32).reshape(256, 4, 32)
    F = _bt_F(b, 32)
    _check_sums(S4, (d, d * d, m.astype(np.int64), e), F, list(range(0, bs, 5)),
                [0] + [1 + p * (3 + C) for p in range(P)], 4608 + 3)
    ia, mask = b["ia"], b["mask"]
    ok = ~m & ia[None, :]
    ns1 = ok.sum(axis=1)
    tot1 = np.where(ok, d, 0).sum(axis=1).astype(np.float64) * K255
    np.testing.assert_array_equal(o["af_all"], tot1 / (2.0 * ns1))
    okp = ok[:, :, None] & mask[None, :, :]
    nsp = okp.sum(axis=1)
    totp = np.einsum("vs,vsp->vp", np.where(ok, d, 0), okp).astype(np.float64) * K255
    assert np.array_equal(o["ns"], nsp)
    np.testing.assert_array_equal(o["af"], totp / (2.0 * nsp))
    np.testing.assert_array_equal(o["mac"], np.minimum(totp, 2.0 * nsp - totp))
    assert np.array_equal(o["flags"] & 1, (np.minimum(tot1, 2.0 * ns1 - tot1) < 5.0).astype(np.int32))
    sel = [(i, j) for i in range(bs) for j in range(P)
           if not (o["flags"][i] & 17) and o["mac"][i, j] >= 5.0 and abs(o["stat"][i, j]) > z_thr]
    vi, ti = [a for a, _ in sel], [c for _, c in sel]
    assert len(sel) > 256
    fb, fse, flrt, fst = st.firth(vi, ti)
    pv, sst = st.spa(vi, ti)
    h = len(sel) // 3
    for part in ((0, h), (h, len(sel))):                             # the same selections in two calls: same bits
        f2 = st.firth(vi[part[0]:part[1]], ti[part[0]:part[1]])
        for a, c in zip(f2, (fb, fse, flrt, fst)):
            assert np.array_equal(a, c[part[0]:part[1]], equal_nan=a.dtype.kind == "f")
        p2 = st.spa(vi[part[0]:part[1]], ti[part[0]:part[1]])
        for a, c in zip(p2, (pv, sst)):
            assert np.array_equal(a, c[part[0]:part[1]], equal_nan=a.dtype.kind == "f")
    fmap = {k: n for n, k in enumerate(sel)}
    n_rows = n_firth = n_fast = n_spa = 0
    for i in range(bs):
        g, ival = obgen.dosage(probs[i, :, 0].astype(np.float64), probs[i, :, 1].astype(np.float64), m[i])
        for j in range(P):
            s = b["sts"][j]
            r = step2_bt.score_bt(g, ival, ia, mask[:, j], b["Y"][:, j], s, z_thr, N)
            ignored = bool(o["flags"][i] & 1) or o["mac"][i, j] < 5.0 or bool(o["flags"][i] & 16)
            assert (r is None) == ignored, (i, j, o["flags"][i])
            if r is None:
                continue
            n_rows += 1
            assert bool(o["flags"][i] & 8) == r["flipped"], i
            np.testing.assert_allclose(o["af"][i, j], r["af"], rtol=(N + 3) * U, atol=0)   # the oracle's float sum
            assert abs(o["info"][i, j] - r["info"]) <= 1e-12, (i, j, o["info"][i, j], r["info"])
            assert abs(o["stat"][i, j] - r["stat"]) <= 1e-8 * abs(r["stat"]), (i, j, o["stat"][i, j], r["stat"])
            if abs(r["stat"]) <= z_thr:
                for k in ("beta", "se", "chisq"):
                    assert abs(o[k][i, j] - r[k]) <= 1e-8 * abs(r[k]), (i, j, k)
                continue
            n = fmap[(i, j)]
            n_firth += 1
            n_fast += bool(fst[n] & 256)
            assert (fst[n] & 15) == int(r["test_fail"]), (i, j, fst[n])
            if not r["test_fail"]:
                for a, c in zip((fb[n], fse[n], flrt[n]), (r["beta"], r["se"], r["chisq"])):
                    assert abs(a - c) <= 1e-5 * max(abs(c), 1e-8), (i, j, a, c)
            rs = step2_bt.score_bt(g, ival, ia, mask[:, j], b["Y"][:, j], s, z_thr, N, correction="spa")
            assert bool(sst[n] & 15) == rs["test_fail"], (i, j, sst[n])
            if not rs["test_fail"]:
                n_spa += 1
                chisq = step2_bt.chisq1_from_pvalue(max(step2_bt.NL_DBL_DMIN, pv[n]))
                assert abs(chisq - rs["chisq"]) <= 1e-5 * rs["chisq"], (i, j, chisq, rs["chisq"])
    st.close()
    assert (o["flags"][0] & 16) and (o["flags"] & 8).sum() > 40 and n_rows > 400
    assert n_firth == len(sel) and n_fast > 20 and n_spa > 200


# ---------------------------------------------------------------------------- 4. the FP64 2-bit statistics (fallback)
def _run_case_f64(tmp_path, monkeypatch, N, M, P, miss):
    """test_s2_gpu.run_case on the FP64 statistics, then the tensor-core statistics on the same handle inputs."""
    from regenie_b200 import capi, synth
    g = synth.genotypes(N, M, seed=11, miss=miss)
    Y, cov, na = synth.phenotypes(g, P, 3, seed=11, na_frac=0.04)
    prefix = helpers.write_fileset(str(tmp_path), g, Y, cov, na, drop_pheno={7}, drop_cov={13})
    bim = plink.read_bim(prefix + ".bim")
    keys, _ = plink.read_fam(prefix + ".fam")
    pr = prep.prepare(keys, str(tmp_path) + "/pheno.txt", str(tmp_path) + "/covar.txt", step=2)
    rng = np.random.default_rng(5)
    blups = rng.normal(size=pr.Y.shape) * 0.3 * pr.mask          # stand-in LOCO predictions
    res, p_sd, scf = step2.compute_res(pr.Y, blups, pr.mask, pr.neff, pr.ncov, pr.scale_Y)
    YtX = res.T @ pr.X
    strict = P == 1
    st = capi.Step2(pr.X, pr.mask, pr.in_analysis, pr.n_analyzed, M, strict=strict)
    monkeypatch.setenv("RG_B200_S2_STATS", "f64")
    st.set_chr(res, scf)
    packed = plink.read_bed_rows(prefix + ".bed", len(keys), bim.offset)
    o = st.block_bed(packed)
    pa = _paths(st)
    assert pa["tc"] == 0 and pa["nchunks"] == (pa["Npad"] + 2047) // 2048 == 2
    dp = pa["dp"]
    rows = list(range(0, M, 7))
    graw = plink.decode_bed(packed, len(keys))
    ia = pr.in_analysis.astype(bool)
    gz = np.where(graw == plink.MISSING_G, 0, graw).astype(np.int64)
    planes = (gz, gz * gz, (graw == plink.MISSING_G).astype(np.int64))
    Fq = _qt_F(dict(N=len(keys), C=pr.X.shape[1], P=P, ia=ia, X=pr.X, res=res, mask=pr.mask.astype(bool)), dp)
    s_f64 = st.debug("s2_sums", np.float64, M * 3 * dp).reshape(M, 3, dp)
    _check_sums(s_f64, planes, Fq, rows, _qt_01_cols(pr.X.shape[1], P), pa["Npad"] + 2)
    n_checked = 0
    for i in range(M):
        vs = step2.variant_stats(graw[i], pr.in_analysis, pr.mask)
        assert bool(o["flags"][i] & 1) == bool(vs["ignored"])
        assert o["ns_all"][i] == vs["ns1"] and np.array_equal(o["ns"][i], vs["ns"])
        if vs["ignored"]:
            continue
        assert np.array_equal(o["af"][i], vs["af"])
        sc = step2.score_qt(vs["g"], pr.X, res, pr.mask, pr.in_analysis, pr.n_analyzed, pr.ncov, scf, YtX, strict)
        assert sc is not None and bool(o["flags"][i] & 4) == sc["is_sparse"]
        for k in ("beta", "se", "chisq"):
            assert np.allclose(o[k][i], sc[k], rtol=1e-8, atol=0), (k, i, o[k][i], sc[k])
        n_checked += 1
    # rg_s2_block_bed_bt needs the tensor-core sums: it refuses under the fallback
    one = np.ones((len(keys), P))
    st.set_chr_bt(one * pr.mask, one, np.zeros((len(keys), P)), [pr.X] * P, np.zeros((len(keys), P)))
    with pytest.raises(capi.RgError, match="tensor-core"):
        st.block_bed_bt(packed[:8])
    # the tensor-core path on the same handle inputs
    monkeypatch.delenv("RG_B200_S2_STATS")
    st.set_chr(res, scf)
    ot = st.block_bed(packed)
    pt = _paths(st)
    assert pt["tc"] == 1 and pt["nchunk"] >= 1 and pt["chunk_len"] * (pt["nchunk"] - 1) < pt["Npad"]
    for k in ("ns", "ns_all", "af", "af_all", "mac", "mac_all", "flags"):
        assert np.array_equal(o[k], ot[k]), k
    _same_stats(ot, o)
    s_tc = st.debug("s2_sums", np.float64, M * 3 * dp).reshape(M, 3, dp)
    _check_tensor_sums(s_tc, planes, Fq, rows, _qt_01_cols(pr.X.shape[1], P))
    st.close()
    return n_checked


def _check_tensor_sums(got, planes, F, rows, exact_cols):
    """Sums of the tensor-core path: F is represented to s_c * 0.5 / 15 * 30^-8 per sample (nine radix-30 digits of
    F / s_c * 15, s_c = max |F_c|), the digit sums are exact, the Horner and the scaling add a few FP64 roundings."""
    FL = F.astype(LD)
    s = np.abs(F).max(axis=0)
    s = np.where(s > 0, s, 1.0)
    for k, z in enumerate(planes):
        zr = z[rows]
        ref = zr.astype(LD) @ FL
        az = np.abs(zr).sum(axis=1).astype(np.float64)[:, None]
        bound = az * s[None, :] * (0.5 / 15 * 30.0 ** -8 + 32 * U)
        err = np.abs(got[rows, k, :F.shape[1]].astype(LD) - ref).astype(np.float64)
        bad = np.argwhere(err > bound)
        assert bad.size == 0, ("tensor sum plane %d, row %d, column %d off by %g (bound %g)" %
                               (k, rows[bad[0][0]], bad[0][1], err[tuple(bad[0])], bound[tuple(bad[0])]))
        assert np.array_equal(got[rows, k][:, exact_cols], ref[:, exact_cols].astype(np.float64)), ("0/1 column", k)


@pytest.mark.parametrize("P", [3, 50])
def test_qt_f64_statistics_fallback(tmp_path, monkeypatch, P):
    """RG_B200_S2_STATS=f64 at N = 3000 (Npad 3072: two FP64 chunks): s2_stats_kernel + partial_sum_kernel against the
    oracle, then against the tensor-core path on the same inputs."""
    assert _run_case_f64(tmp_path, monkeypatch, N=3000, M=256, P=P, miss=0.02) > 200


# ------------------------------------------------------------------------------- 5. the tensor-core chunk limit
@pytest.mark.parametrize("N,nchunk", [(262144, 1), (262145, 2)])
def test_qt_tensor_chunk_limit(N, nchunk):
    """max_block_size 2048, C = 3, P = 33: D = 169 feature columns = 7 digit-row tiles x 48 row tiles = 336 >= 296, so
    the chunk count comes from the 2^18 rule alone.  A row of g = 2 everywhere puts 60 * 262 144 = 15 728 640 < 2^24 in
    the S2 digit sum of column 0; nearly fixed rows and rows with a few missing calls sit beside it."""
    from regenie_b200 import capi, synth
    P, C, bs = 33, 3, 128
    pb = _qt_problem(N, P, C, seed=55, all_analysed=True)
    rng = np.random.default_rng(55)
    maf = rng.uniform(0.02, 0.5, size=bs)
    g = rng.binomial(2, maf[:, None], size=(bs, N)).astype(np.uint8)
    g[0] = 2
    g[1:4] = 0
    g[1, 17] = g[2, N - 1] = g[3, N // 2] = 1                        # one heterozygote
    for r in range(4, 12):
        g[r, rng.choice(N, 3 + r, replace=False)] = 3                  # a few missing calls
    g[12] = np.where(rng.random(N) < 0.5, 3, 2)                       # half missing, the rest hom-alt
    st = capi.Step2(pb["X"], pb["mask"], pb["ia"], pb["n_an"], 2048)
    st.set_chr(pb["res"], pb["scf"])
    o = st.block_bed(synth.pack_bed(g))
    pa = _paths(st)
    Npad = (N + 127) // 128 * 128
    assert pa["tc"] == 1 and pa["Npad"] == Npad and pa["nchunk"] == nchunk, pa
    assert pa["drows"] == 1792 and pa["chunk_len"] == (262144 if nchunk == 1 else 131200)
    obs = g != 3
    gz = np.where(obs, g, 0).astype(np.float64)
    mask = pb["mask"].astype(np.float64)
    ns1 = obs.sum(axis=1)
    assert np.array_equal(o["ns_all"], ns1)
    np.testing.assert_array_equal(o["af_all"], gz.sum(axis=1) / (2.0 * ns1))
    ns = obs.astype(np.float64) @ mask
    assert np.array_equal(o["ns"], ns)
    np.testing.assert_array_equal(o["af"], (gz @ mask) / (2.0 * ns))
    mu = gz.sum(axis=1) / ns1
    nnz = (gz != 0).sum(axis=1) + np.where(mu != 0, N - ns1, 0)
    assert np.array_equal((o["flags"] & 4) != 0, nnz <= N * 0.5)
    # the 0/1 columns of the sums: exact integers (float64 products of small integers, summed exactly by BLAS)
    dp = pa["dp"]
    S = st.debug("s2_sums", np.float64, bs * 3 * dp).reshape(bs, 3, dp)
    cols = _qt_01_cols(C, P)
    F01 = np.hstack([pb["ia"][:, None].astype(np.float64), mask])
    for k, z in enumerate((gz, gz * gz, (~obs).astype(np.float64))):
        assert np.array_equal(S[:, k][:, cols], z @ F01), k
    assert S[0, 1, 0] == 4.0 * N
    X, res = pb["X"], pb["res"]
    YtX = res.T @ X
    for i in (0, 1, 5, 12, 20, 64, 100, 127):
        gi = np.where(obs[i], g[i], mu[i]).astype(np.float64)
        sparse = (gi != 0).sum() <= N * 0.5                            # check_sparse_G, src/Geno.cpp:3165
        xtg = X.T @ gi
        gr = gi - X @ xtg
        if not sparse and np.linalg.norm(gr) / math.sqrt(N - C) < 1e-6:
            assert o["flags"][i] & 2, i
            continue
        for j in range(P):
            if sparse:                                                 # src/Step2_Models.cpp:404, :410
                gm = gi * mask[:, j]
                num = res[:, j] @ gi - YtX[j] @ xtg
                den = gm @ gm - 2 * (X.T @ gm) @ xtg + xtg @ xtg
            else:                                                      # :415-416
                num = res[:, j] @ gr
                den = (mask[:, j] * gr * gr).sum()
            ref = num / np.sqrt(den)
            assert abs(o["stat"][i, j] - ref) <= 1e-8 * max(1.0, abs(ref)), (i, j, o["stat"][i, j], ref)
            np.testing.assert_allclose(o["beta"][i, j], ref * pb["scf"][j] / np.sqrt(den), rtol=1e-8)
            np.testing.assert_allclose(o["se"][i, j], pb["scf"][j] / np.sqrt(den), rtol=1e-8)
    st.close()
