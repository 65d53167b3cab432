"""GPU parity: Step-2 QT score test through the C ABI vs the numpy oracle.

CHR/POS/ID/A1FREQ/N must be bit-exact (integer sums); BETA/SE/CHISQ/LOG10P within 1e-5 relative
(north_star) -- here held to 1e-8 on the unrounded values and exactly on the printed 6-digit row.
"""
import numpy as np
import pytest

import helpers
from oracle import plink, prep, step2

pytestmark = pytest.mark.gpu


def run_case(tmp_path, N, M, P, miss, strict=False, maf_hi=0.5):
    from regenie_b200 import capi, synth
    g = synth.genotypes(N, M, seed=11, miss=miss, maf_hi=maf_hi)
    Y, cov, na = synth.phenotypes(g, P, 3, seed=11, na_frac=0.04)
    prefix = helpers.write_fileset(str(tmp_path), g, Y, cov, na, drop_pheno={7}, drop_cov={13})
    bim = plink.read_bim(prefix + ".bim")
    keys, _ = plink.read_fam(prefix + ".fam")
    pr = prep.prepare(keys, str(tmp_path) + "/pheno.txt", str(tmp_path) + "/covar.txt", step=2, strict=strict)
    rng = np.random.default_rng(5)
    blups = rng.normal(size=pr.Y.shape) * 0.3 * pr.mask          # stand-in LOCO predictions
    res, p_sd, scf = step2.compute_res(pr.Y, blups, pr.mask, pr.neff, pr.ncov, pr.scale_Y)
    YtX = res.T @ pr.X
    st = capi.Step2(pr.X, pr.mask, pr.in_analysis, pr.n_analyzed, 256, strict=strict or P == 1)
    st.set_chr(res, scf)
    packed = plink.read_bed_rows(prefix + ".bed", len(keys), bim.offset)
    n_checked = n_sparse = 0
    for s in range(0, M, 256):
        rows = packed[s:s + 256]
        o = st.block_bed(rows)
        graw = plink.decode_bed(rows, len(keys))
        for i in range(rows.shape[0]):
            vs = step2.variant_stats(graw[i], pr.in_analysis, pr.mask)
            assert bool(o["flags"][i] & 1) == bool(vs["ignored"])
            assert o["ns_all"][i] == vs["ns1"]
            assert np.array_equal(o["ns"][i], vs["ns"])              # N: bit-exact
            if vs["ignored"]:
                continue
            assert np.array_equal(o["af"][i], vs["af"])              # A1FREQ: bit-exact
            sc = step2.score_qt(vs["g"], pr.X, res, pr.mask, pr.in_analysis, pr.n_analyzed, pr.ncov, scf, YtX,
                                strict or P == 1)
            assert sc is not None
            assert bool(o["flags"][i] & 4) == sc["is_sparse"]
            n_sparse += sc["is_sparse"]
            for k in ("beta", "se", "chisq"):
                assert np.allclose(o[k][i], sc[k], rtol=1e-8, atol=0), (k, i, o[k][i], sc[k])
            for ph in range(P):
                a = step2.sumstats_row(1, 1, "x", "A", "G", o["af"][i, ph], o["ns"][i, ph], o["beta"][i, ph],
                                       o["se"][i, ph], o["chisq"][i, ph], step2.get_logp(o["chisq"][i, ph]))
                b = step2.sumstats_row(1, 1, "x", "A", "G", vs["af"][ph], vs["ns"][ph], sc["beta"][ph], sc["se"][ph],
                                       sc["chisq"][ph], sc["logp"][ph])
                ta, tb = a.split(), b.split()
                assert ta[:8] == tb[:8]          # CHROM..A1FREQ N TEST: exact
                for x, y in zip(ta[8:12], tb[8:12]):
                    assert abs(float(x) - float(y)) <= 1e-5 * abs(float(y))
            n_checked += 1
    return n_checked, n_sparse


def test_s2_qt_multitrait_dense_and_sparse(tmp_path):
    n, ns = run_case(tmp_path, N=1500, M=400, P=3, miss=0.02)
    assert n > 300 and 0 < ns < n          # both genotype branches exercised


def test_s2_qt_strict_single_trait(tmp_path):
    n, ns = run_case(tmp_path, N=900, M=300, P=1, miss=0.01)
    assert n > 200


def test_s2_qt_rare_variants_and_mac_filter(tmp_path):
    n, ns = run_case(tmp_path, N=1200, M=300, P=2, miss=0.0, maf_hi=0.02)
    assert ns > 0


def test_s2_qt_fifty_traits(tmp_path):
    """BASELINE configs[4] trait count: 254 feature columns = 19 digit groups = 10 column tiles on the tensor-core path."""
    n, ns = run_case(tmp_path, N=700, M=256, P=50, miss=0.02)
    assert n > 200


def test_staged_input_gives_the_same_rows(tmp_path):
    """rg_s2_stage: the rows of block b+1 copied on the copy stream while block b is tested (pinned memory from
    rg_host_alloc) - every output equal, bit for bit, to the call that copies its own rows."""
    import ctypes as C
    from regenie_b200 import capi, synth
    N, M, P, bs = 3000, 768, 3, 256
    g = synth.genotypes(N, M, seed=3, miss=0.02)
    Y, cov, na = synth.phenotypes(g, P, 3, seed=3, na_frac=0.03)
    prefix = helpers.write_fileset(str(tmp_path), g, Y, cov, na)
    bim = plink.read_bim(prefix + ".bim")
    keys, _ = plink.read_fam(prefix + ".fam")
    pr = prep.prepare(keys, str(tmp_path) + "/pheno.txt", str(tmp_path) + "/covar.txt", step=2)
    res, p_sd, scf = step2.compute_res(pr.Y, np.zeros_like(pr.Y), pr.mask, pr.neff, pr.ncov, pr.scale_Y)
    st = capi.Step2(pr.X, pr.mask, pr.in_analysis, pr.n_analyzed, bs)
    st.set_chr(res, scf)
    packed = np.ascontiguousarray(plink.read_bed_rows(prefix + ".bed", len(keys), bim.offset))
    stride = packed.shape[1]
    plain = [st.block_bed(packed[s:s + bs]) for s in range(0, M, bs)]
    L = capi.lib()
    L.rg_host_alloc.argtypes = [C.c_void_p, C.c_int64]
    L.rg_host_free.argtypes = [C.c_void_p]
    hp = C.c_void_p()
    capi.check(L.rg_host_alloc(C.byref(hp), packed.nbytes))
    try:
        C.memmove(hp, packed.ctypes.data, packed.nbytes)
        nb = M // bs
        nxt = st.stage(0, hp.value, bs * stride)
        for b in range(nb):
            cur = nxt
            if b + 1 < nb:
                nxt = st.stage((b + 1) & 1, hp.value + (b + 1) * bs * stride, bs * stride)
            o = st.block_bed_raw(cur, bs, stride)
            for k in ("af", "ns", "mac", "af_all", "ns_all", "flags", "stat", "beta", "se", "chisq"):
                assert np.array_equal(o[k], plain[b][k]), (k, b)
    finally:
        capi.check(L.rg_host_free(hp))
    st.close()


def test_block_routes_need_their_chromosome_call_and_count_the_kernels_they_launch():
    """The quantitative-trait block routes refuse to run before rg_s2_set_chr, which fills the feature rows, YtX and the
    scale factors they read; each of the four routes adds the number of kernels it launches to rg_launch_count."""
    from regenie_b200 import capi
    rng = np.random.default_rng(3)
    N, P, C, bs = 1000, 2, 3, 32
    X = np.asfortranarray(np.linalg.qr(np.hstack([np.ones((N, 1)), rng.standard_normal((N, C - 1))]))[0])
    g = rng.integers(0, 3, (bs, N))
    probs = np.stack([(g == 2) * 255, (g == 1) * 255], axis=2).astype(np.uint8)
    packed = rng.integers(0, 256, (bs, (N + 3) // 4), dtype=np.uint8)
    st = capi.Step2(X, np.ones((N, P), dtype=np.uint8), np.ones(N, dtype=np.uint8), N, bs)
    for call in (lambda: st.block_bed(packed), lambda: st.block_bgen8(probs)):
        with pytest.raises(capi.RgError, match="rg_s2_set_chr has not been called"):
            call()

    def launches(call):
        n0 = capi.lib().rg_launch_count(st.h)
        call()
        return capi.lib().rg_launch_count(st.h) - n0

    st.set_chr(rng.standard_normal((N, P)), np.ones(P))
    assert launches(lambda: st.block_bed(packed)) == 4
    assert launches(lambda: st.block_bgen8(probs)) == 6
    p = rng.uniform(0.2, 0.8, (N, P))
    gs = np.sqrt(p * (1 - p))
    y = (rng.random((N, P)) < p).astype(float)
    st.set_chr_bt(gs, gs, (y - p) / gs, [X * gs[:, [j]] for j in range(P)], y)
    assert launches(lambda: st.block_bgen8_bt(probs)) == 5
    assert launches(lambda: st.block_bed_bt(packed)) == 5
    st.close()
