"""GPU parity of the GxE interaction tests (rg_s2_interaction) with the numpy restatement in interaction_oracle.py.

Both routes on .bed rows and 8-bit dosages with missing calls, a sample subset, N not a multiple of 16, a block size
that is not a multiple of the row pad, two traits with different masks, HC3 / HC4 / model-based standard errors and the
HLM route with the null state the oracle fitted.  BETA, SE, the Wald statistics and the 2-DF statistic within 1e-5
relative.
"""
import numpy as np
import pytest

import helpers
import interaction_oracle as io
from oracle import bgen, plink, prep, step2

pytestmark = pytest.mark.gpu

RTOL = 1e-5


def stats(coef, vcov):
    """BETA / SE / CHISQ of the two rows and the 2-DF statistic (src/Interaction.cpp:206-273)."""
    se = np.sqrt(np.diag(vcov))
    return np.concatenate([coef, se, coef ** 2 / np.diag(vcov), [coef @ np.linalg.solve(vcov, coef)]])


def setup(tmp_path, N, M, bs, kind, seed=3, hlm_k=None):
    """kind: "bed", "bed_rf" (.bed rows with --ref-first, i.e. flipped alleles) or "bgen8".  hlm_k: pad the HLM X
    (covariates, E^2, LOCO) with random columns up to hlm_k columns."""
    from regenie_b200 import capi, synth
    g = synth.genotypes(N, M, seed=seed, miss=0.02, maf_hi=0.5)
    Y, cov, na = synth.phenotypes(g, 2, 3, seed=seed, na_frac=0.05)
    prefix = helpers.write_fileset(str(tmp_path), g, Y, cov, na, drop_pheno={7}, drop_cov={13})
    keys, _ = plink.read_fam(prefix + ".fam")
    pr = prep.prepare(keys, str(tmp_path) + "/pheno.txt", str(tmp_path) + "/covar.txt", step=2, strict=False)
    assert pr.mask[:, 0].sum() != pr.mask[:, 1].sum()               # different masks
    ia = pr.in_analysis.astype(bool)
    rng = np.random.default_rng(seed)
    blups = rng.normal(size=pr.Y.shape) * 0.3 * pr.mask
    res, _, scf = step2.compute_res(pr.Y, blups, pr.mask, pr.neff, pr.ncov, pr.scale_Y)
    E = np.where(ia, rng.normal(size=len(ia)) * 1.5 + 0.3, 0.0)
    st = capi.Step2(pr.X, pr.mask, pr.in_analysis, pr.n_analyzed, bs)
    st.set_chr(res, scf)
    # HLM null state of each trait, fitted by the oracle
    V, _ = io.hlm_design(E, pr.X, blups[:, 0])
    dl, pl, yl = [], [], []
    for i in range(2):
        _, Xh = io.hlm_design(E, pr.X, blups[:, i])
        if hlm_k:
            Xh = np.column_stack([Xh, rng.normal(size=(len(ia), hlm_k - Xh.shape[1])) * ia[:, None]])
        y = (pr.Y[:, i] + 0.2 * E * pr.Y[:, i]) * pr.mask[:, i]
        b, _ = io.hlm_fit(y, pr.mask[:, i], Xh, V)
        d, Px, yres = io.hlm_state(y, pr.mask[:, i], Xh, V, b)
        dl.append(d); pl.append(Px); yl.append(yres)
    st.set_interaction(E, np.stack(dl, 1), pl, np.stack(yl, 1))
    # genotypes
    if kind in ("bed", "bed_rf"):
        bim = plink.read_bim(prefix + ".bim")
        rows = plink.read_bed_rows(prefix + ".bed", len(keys), bim.offset)
        gi = [plink.decode_bed(rows[s:s + bs], len(keys), ref_first=kind == "bed_rf") for s in range(0, M, bs)]
        blocks = [rows[s:s + bs] for s in range(0, M, bs)]
    else:
        probs, miss = helpers.synthetic_dosage_probs(M, len(keys), seed=seed)
        dos, _ = bgen.dosage(probs[..., 0].astype(float), probs[..., 1].astype(float), miss)
        gi = [dos[s:s + bs] for s in range(0, M, bs)]
        blocks = [(probs[s:s + bs], (miss[s:s + bs] * 0x80).astype(np.uint8)) for s in range(0, M, bs)]
    return st, pr, res, scf, E, (dl, pl, yl), blocks, gi


def run_block(st, kind, blk, min_mac):
    if kind in ("bed", "bed_rf"):
        return st.block_bed(blk, min_mac=min_mac, ref_first=kind == "bed_rf")
    return st.block_bgen8(blk[0], blk[1], min_mac=min_mac)


@pytest.mark.parametrize("kind", ["bed", "bed_rf", "bgen8"])
@pytest.mark.parametrize("mode", ["hlm", "hlm_k64", "split", "hc3", "hc4", "model", "no_hlm_state"])
def test_interaction_matches_oracle(tmp_path, kind, mode):
    """no_hlm_state: rg_s2_set_interaction without the HLM state, so every variant takes the robust route at the default
    rare_mac.  hlm_k64: 64 columns in the HLM X (the covariate limit)."""
    N, M, bs = 1001, 150, 72
    st, pr, res, scf, E, (dl, pl, yl), blocks, gi = setup(tmp_path, N, M, bs, kind, hlm_k=64 if mode == "hlm_k64" else None)
    assert mode != "hlm_k64" or pl[0].shape[1] == 64
    if mode == "no_hlm_state":
        st.set_interaction(E)
    ia = pr.in_analysis.astype(bool)
    opts = dict(rare_mac=1000.0, min_mac=5.0)
    if mode in ("hc3", "hc4", "model"):
        opts.update(force_robust=True, force_hc4=mode == "hc4", no_robust=mode == "model")
    counts = {1: 0, 2: 0, -1: 0}
    for blk, graw in zip(blocks, gi):
        o = run_block(st, kind, blk, opts["min_mac"])
        b = o["flags"].shape[0]
        if mode == "split":                                         # traits of one variant on both sides of rare_mac
            lo, hi = o["mac"].min(axis=1), o["mac"].max(axis=1)
            k = int(np.argmax(hi - lo))
            opts["rare_mac"] = 0.5 * (lo[k] + hi[k])
        if mode == "hc4":
            opts["rare_mac"] = float(np.median(o["mac"]))           # HC4 for the traits with MAC <= rare_mac
        status, coef, vcov = st.interaction(b, **opts)
        gimp, _ = plink.mean_impute_block(graw, ia)
        for v in range(b):
            if o["flags"][v] & 3:
                assert (status[v] == 0).all()
                continue
            mac = o["mac"][v]
            hlm = mode in ("hlm", "hlm_k64", "split") and (mac < opts["rare_mac"]).any()
            for i in range(2):
                if mac[i] < opts["min_mac"]:
                    assert status[v, i] == 0
                    continue
                if hlm:
                    want = io.hlm_test(gimp[v], E, dl[i], pl[i], yl[i])
                else:
                    r = io.robust(gimp[v], E, pr.X, res, pr.mask, scf, pr.n_analyzed, mac, opts["rare_mac"],
                                  opts.get("force_hc4", False), opts.get("no_robust", False))
                    want = None if r is None else (r[0][i], r[1][i])
                if want is None:
                    assert status[v, i] in (0, -1)
                    continue
                assert status[v, i] == (2 if hlm else 1), (v, i, status[v, i])
                counts[int(status[v, i])] += 1
                got, ref = stats(coef[v, i], vcov[v, i]), stats(*want)
                assert np.allclose(got, ref, rtol=RTOL, atol=0), (mode, v, i, got, ref)
    if mode in ("hlm", "hlm_k64"):
        assert counts[2] > 50
    elif mode == "split":
        assert counts[2] > 0
    else:
        assert counts[1] > 50


def test_interaction_skips_singular(tmp_path):
    """E constant over the analysed samples: E o G is a multiple of G, so H^T H is near-singular: status -1 (no rows)
    for every pair that is not ignored, 0 for the ignored ones."""
    N, M, bs = 1001, 40, 40
    st, pr, res, scf, E, _, blocks, _ = setup(tmp_path, N, M, bs, "bed")
    st.set_interaction(pr.in_analysis.astype(float) * 2.0)
    o = st.block_bed(blocks[0])
    status, _, _ = st.interaction(bs, force_robust=True, min_mac=5.0)
    live = ((o["flags"] & 3) == 0)[:, None] & (o["mac"] >= 5.0)
    assert live.sum() > 20
    assert (status[live] == -1).all() and (status[~live] == 0).all()


def test_interaction_needs_words_of_current_block(tmp_path):
    """A .bed block run before rg_s2_set_interaction left no genotype words: the call is refused, not run on stale or
    missing data.  Running the block again after the state is set makes it work."""
    from regenie_b200 import capi
    N, M, bs = 1001, 40, 40
    st, pr, res, scf, E, _, blocks, _ = setup(tmp_path, N, M, bs, "bed")
    st.set_chr(res, scf)                                            # clears the interaction state
    st.block_bed(blocks[0])
    st.set_interaction(E)
    with pytest.raises(capi.RgError, match="rg_s2_set_interaction"):
        st.interaction(bs)
    st.block_bed(blocks[0])
    status, _, _ = st.interaction(bs)
    assert (status == 1).sum() > 20
    st.set_chr(res, scf)                                            # a new chromosome: the block's words are stale
    st.set_interaction(E)
    with pytest.raises(capi.RgError):
        st.interaction(bs)
