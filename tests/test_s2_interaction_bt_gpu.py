"""GPU parity of the binary-trait GxE interaction tests (rg_s2_interaction_bt, rg_s2_interaction_firth) with the numpy
restatement in interaction_bt_oracle.py.

.bed rows, .bed rows with --ref-first (flipped alleles) and 8-bit dosages with missing calls; N = 1001 with samples
outside the analysis (and a shuffled subset of them through sample_idx), a block size that is not a multiple of the row pad, two traits with different masks (one with
about 5 % cases), and the covariate basis spanning E and E^2.  BETA, SE, the Wald statistics and the 2-DF statistic of
the Wald route, and the coefficients, SEs and LRTs of the Firth route, within 1e-5 relative.
"""
import numpy as np
import pytest
from scipy.stats import chi2

import helpers
import interaction_bt_oracle as ibo
from oracle import bgen, plink, prep, step2_bt
from oracle.prep import get_basis

pytestmark = pytest.mark.gpu

RTOL = 1e-5


def stats(coef, vcov):
    """BETA / SE / CHISQ of the two rows and the 2-DF statistic."""
    se = np.sqrt(np.diag(vcov))
    return np.concatenate([coef, se, coef ** 2 / np.diag(vcov), [coef @ np.linalg.solve(vcov, coef)]])


def close(got, ref):
    return np.allclose(got, ref, rtol=RTOL, atol=1e-10)


class Case:
    """A binary-trait Step-2 handle with its interaction state, the blocks of one genotype input and what the oracle
    needs.  kind: "bed", "bed_rf" or "bgen8".  extra_cov: random covariate columns added to the basis."""

    def __init__(self, tmp_path, kind, N=1001, M=150, bs=72, P=2, seed=3, extra_cov=0, E_const=False, bs_max=None,
                 subset=False):
        from regenie_b200 import capi, synth
        g = synth.genotypes(N, M, seed=seed, miss=0.02, maf_hi=0.5)
        Yq, cov, na = synth.phenotypes(g, P, 3, seed=seed, na_frac=0.05)
        Yb = np.zeros_like(Yq)
        for j in range(P):
            q = 0.95 if j == 1 else 0.6                               # trait 1: about 5 % cases
            Yb[:, j] = Yq[:, j] > np.quantile(Yq[:, j], q)
        prefix = helpers.write_fileset(str(tmp_path), g, Yb, cov, na, drop_pheno={7}, drop_cov={13})
        file_keys, _ = plink.read_fam(prefix + ".fam")
        # subset: the handle's samples are a shuffled subset of the file's (sample_idx)
        self.sidx = np.random.default_rng(seed + 5).permutation(N)[:N - 60].astype(np.int32) if subset else None
        keys = file_keys if not subset else [file_keys[i] for i in self.sidx]
        N = len(keys)
        pr = prep.prepare(keys, str(tmp_path) + "/pheno.txt", str(tmp_path) + "/covar.txt", bt=True, step=2)
        self.ia = ia = pr.in_analysis.astype(bool)
        self.mask, self.Y = pr.mask.astype(bool), pr.Y_raw
        if P >= 2:
            assert self.mask[:, 0].sum() != self.mask[:, 1].sum()
        rng = np.random.default_rng(seed)
        self.E = np.where(ia, 2.0 if E_const else rng.normal(size=N) * 1.5 + 0.3, 0.0)
        cols = [pr.X, self.E, self.E * self.E] + ([rng.normal(size=(N, extra_cov))] if extra_cov else [])
        self.X, _ = get_basis(np.column_stack(cols) * ia[:, None])
        self.n_analyzed = pr.n_analyzed
        blup = 0.2 * rng.standard_normal((N, P))
        sts = [step2_bt.BtChrom(self.Y[:, j], self.X, blup[:, j], self.mask[:, j]) for j in range(P)]
        self.off = np.stack([blup[:, j] * self.mask[:, j] + self.X @ sts[j].beta0 for j in range(P)], 1)
        self.firth_off = np.stack([s.cov_blup_offset for s in sts], 1)
        self.bt_state = (np.stack([s.gamma_sqrt_mask for s in sts], 1), np.stack([s.gamma_sqrt for s in sts], 1),
                         np.stack([s.yres for s in sts], 1), [s.Xg for s in sts], self.Y)
        self.kind, self.P, self.bs, self.bs_max = kind, P, bs, bs_max or bs
        if kind in ("bed", "bed_rf"):
            bim = plink.read_bim(prefix + ".bim")
            self.rows = plink.read_bed_rows(prefix + ".bed", len(file_keys), bim.offset)
            self.graw = plink.decode_bed(self.rows, len(file_keys), ref_first=kind == "bed_rf")
        else:
            self.probs, miss = helpers.synthetic_dosage_probs(M, len(file_keys), seed=seed)
            self.graw, _ = bgen.dosage(self.probs[..., 0].astype(float), self.probs[..., 1].astype(float), miss)
            self.miss = (miss * 0x80).astype(np.uint8)
        if subset:
            self.graw = self.graw[:, self.sidx]
        self.gimp, _ = plink.mean_impute_block(self.graw, ia)
        self.M = M

    def handle(self, traits=None, firth=True):
        from regenie_b200 import capi
        t = list(range(self.P)) if traits is None else list(traits)
        st = capi.Step2(self.X, self.mask[:, t], self.ia.astype(np.uint8), self.n_analyzed, self.bs_max)
        a, b, c, xg, y = self.bt_state
        st.set_chr_bt(a[:, t], b[:, t], c[:, t], [xg[j] for j in t], y[:, t],
                      self.firth_off[:, t] if firth else None)
        st.set_interaction_bt(self.E, self.off[:, t])
        return st

    def block(self, st, s0, s1):
        if self.kind in ("bed", "bed_rf"):
            return st.block_bed_bt(self.rows[s0:s1], sample_idx=self.sidx, ref_first=self.kind == "bed_rf")
        return st.block_bgen8_bt(self.probs[s0:s1], self.miss[s0:s1], sample_idx=self.sidx)

    def design(self, v, flipped):
        g = np.where(self.ia, 2.0 - self.gimp[v], 0.0) if flipped else self.gimp[v]
        return ibo.design(g, self.E, self.X, self.n_analyzed)


def check_wald(case, st, s0, o, status, coef, vcov, opts, traits=None):
    """Every pair of the block against the oracle; returns the counts of statuses 1 and 3."""
    t = list(range(case.P)) if traits is None else list(traits)
    counts = {1: 0, 3: 0}
    for v in range(o["flags"].shape[0]):
        gv = s0 + v
        if o["flags"][v] & 1:
            assert (status[v] == 0).all()
            continue
        mean = case.graw[gv][case.ia & (case.graw[gv] != -3)].mean()
        flipped = bool(o["flags"][v] & 8)
        assert flipped == (mean > 1)
        d = case.design(gv, flipped)
        for k, i in enumerate(t):
            if o["mac"][v, k] < opts["min_mac"] or d is None:
                assert status[v, k] == 0, (v, k)
                continue
            so, b, V = ibo.wald(d[0], case.Y[:, i], case.off[:, i], case.mask[:, i], o["mac"][v, k], opts["rare_mac"],
                                opts.get("force_robust", False), opts.get("no_robust", False))
            assert status[v, k] == so, (v, k, status[v, k], so)
            if so < 0:
                continue
            counts[so] += 1
            want = ibo.printed(b, V, d[1], d[2], flipped)
            got, ref = stats(coef[v, k], vcov[v, k]), stats(*want)
            assert close(got, ref), (v, k, got, ref)
    return counts


@pytest.mark.parametrize("kind", ["bed", "bed_rf", "bgen8"])
@pytest.mark.parametrize("mode", ["default", "force_robust", "no_robust"])
def test_interaction_bt_matches_oracle(tmp_path, kind, mode):
    """default: rare_mac at the block's median MAC, so both routes occur; force_robust: HC3 everywhere; no_robust:
    model-based everywhere.  The handle reads a shuffled subset of the file's samples."""
    case = Case(tmp_path, kind, subset=True)
    st = case.handle()
    tot = {1: 0, 3: 0}
    for s0 in range(0, case.M, case.bs):
        s1 = min(case.M, s0 + case.bs)
        o = case.block(st, s0, s1)
        opts = dict(rare_mac=float(np.median(o["mac"])) if mode == "default" else 1000.0, min_mac=5.0,
                    force_robust=mode == "force_robust", no_robust=mode == "no_robust")
        status, coef, vcov = st.interaction_bt(**opts)
        c = check_wald(case, st, s0, o, status, coef, vcov, opts)
        tot[1] += c[1]; tot[3] += c[3]
    if mode == "default":
        assert tot[1] > 5 and tot[3] > 50, tot
    elif mode == "force_robust":
        assert tot[1] > 100 and tot[3] == 0, tot
    else:
        assert tot[3] > 100 and tot[1] == 0, tot


@pytest.mark.parametrize("kind", ["bed", "bed_rf", "bgen8"])
def test_interaction_firth_matches_oracle(tmp_path, kind):
    """pThresh 0.95: most pairs take the Firth route, more than kIntBtBatch (128) of them, so the pairs are run in several
    batches; their status, coefficients, SEs and LRTs against the oracle.  The first 20 pairs are selected again at the
    end (in the last batch) and give the same bits."""
    case = Case(tmp_path, kind, M=150, bs=150)
    st = case.handle()
    o = case.block(st, 0, case.M)
    status, coef, vcov = st.interaction_bt(min_mac=5.0)
    thr = chi2.isf(0.95, 1)
    sel = [(v, i) for v in range(case.M) for i in range(case.P)
           if status[v, i] in (1, 3) and coef[v, i, 1] ** 2 / vcov[v, i, 1, 1] >= thr]
    assert len(sel) > 2 * 128 - 50                                  # three batches, the last one partly filled
    n = len(sel)
    sel = sel + sel[:20]
    fc, fse, flrt, fst = st.interaction_firth([v for v, _ in sel], [i for _, i in sel])
    for out in (fc, fse, flrt, fst):
        assert np.array_equal(out[n:], out[:20])
    sel = sel[:n]
    n_ok = 0
    for k, (v, i) in enumerate(sel):
        flipped = bool(o["flags"][v] & 8)
        H, sf, scf = case.design(v, flipped)
        so, b, se, lrt = ibo.firth(H, case.Y[:, i], case.firth_off[:, i], case.mask[:, i])
        assert fst[k] == so, (v, i, fst[k], so)
        if so:
            continue
        n_ok += 1
        sg = -1.0 if flipped else 1.0
        s = np.array([1 / sf, 1 / scf])
        assert close(fc[k], sg * b * s), (v, i, fc[k], sg * b * s)
        assert close(fse[k], se * s), (v, i, fse[k], se * s)
        assert close(flrt[k], lrt), (v, i, flrt[k], lrt)
        assert (flrt[k] >= 0).all()
    assert n_ok > 150


def test_interaction_bt_constant_e_is_singular(tmp_path):
    """E constant over the analysed samples: E o G is collinear with G after the covariates (which span E) are projected
    out, so every live pair gets no rows (-1 or 0), never a result."""
    case = Case(tmp_path, "bed", M=40, bs=40, E_const=True)
    st = case.handle()
    o = case.block(st, 0, 40)
    status, _, _ = st.interaction_bt(force_robust=True, min_mac=5.0)
    live = ((o["flags"] & 1) == 0)[:, None] & (o["mac"] >= 5.0)
    assert live.sum() > 20
    assert np.isin(status[live], (-1, 0)).all() and (status[~live] == 0).all()


def test_interaction_bt_call_order_is_refused(tmp_path):
    from regenie_b200 import capi
    case = Case(tmp_path, "bed", M=40, bs=40)
    st = case.handle(firth=False)
    # Firth before any Wald call on the block, and without the null-Firth offsets
    o = case.block(st, 0, 40)
    with pytest.raises(capi.RgError, match="rg_s2_interaction_bt"):
        st.interaction_firth([0], [0])
    st.interaction_bt()
    with pytest.raises(capi.RgError, match="firth_offset"):
        st.interaction_firth([0], [0])
    # a new chromosome clears the interaction state and ends the block
    a, b, c, xg, y = case.bt_state
    st.set_chr_bt(a, b, c, xg, y, case.firth_off)
    with pytest.raises(capi.RgError, match="rg_s2_set_interaction_bt"):
        st.interaction_bt()
    st.set_interaction_bt(case.E, case.off)
    with pytest.raises(capi.RgError, match="resident|block"):
        st.interaction_bt()
    case.block(st, 0, 40)
    status, _, _ = st.interaction_bt()
    assert (status != 0).sum() > 20
    # a new block after the Wald call: Firth needs the Wald call on that block
    case.block(st, 0, 40)
    with pytest.raises(capi.RgError, match="rg_s2_interaction_bt"):
        st.interaction_firth([0], [0])
    # a resident quantitative-trait block
    rng = np.random.default_rng(0)
    res = rng.normal(size=(len(case.ia), case.P)) * case.mask
    st.set_chr(res, np.ones(case.P))
    st.block_bed(case.rows[:40])
    with pytest.raises(capi.RgError, match="rg_s2_block_bed_bt"):
        st.interaction_bt()


def test_interaction_bt_bit_identical_across_traits_and_partitions(tmp_path):
    """One trait of a P = 3 handle against a P = 1 handle, and blocks of 72 against blocks of 40: the same bits."""
    case = Case(tmp_path, "bed", M=120, bs=72, P=3, bs_max=72)
    full = case.handle()
    one = case.handle(traits=[2])
    for s0 in range(0, 120, 72):
        s1 = min(120, s0 + 72)
        case.block(full, s0, s1); case.block(one, s0, s1)
        a = full.interaction_bt(min_mac=5.0)
        b = one.interaction_bt(min_mac=5.0)
        for x, y in zip(a, b):
            assert np.array_equal(x[:, 2:3], y), "P = 3 vs P = 1"
        assert (a[0][:, 2] != 0).sum() > 20
    ref = {}
    for s0 in range(0, 120, 72):
        case.block(full, s0, min(120, s0 + 72))
        st_, c_, v_ = full.interaction_bt(min_mac=5.0)
        for v in range(st_.shape[0]):
            ref[s0 + v] = (st_[v], c_[v], v_[v])
    for s0 in range(0, 120, 40):
        case.block(full, s0, s0 + 40)
        st_, c_, v_ = full.interaction_bt(min_mac=5.0)
        for v in range(40):
            r = ref[s0 + v]
            assert np.array_equal(st_[v], r[0]) and np.array_equal(c_[v], r[1]) and np.array_equal(v_[v], r[2])


@pytest.mark.parametrize("N,P,bs,extra", [(1001, 4, 128, 0), (2100, 5, 129, 59), (2047, 1, 17, 0), (2049, 8, 16, 0)])
def test_interaction_bt_shapes(tmp_path, N, P, bs, extra):
    """Each side of the kernels' boundaries: kIntBtBatch (128) variants per batch, kIntBtTG (4) traits per CTA, 16 H
    slots per CTA of the H kernel, the 2048-sample chunks of the sums, and C = 64 (E and E^2 counted in it)."""
    case = Case(tmp_path, "bed", N=N, M=bs, bs=bs, P=P, extra_cov=extra)
    if extra:
        assert case.X.shape[1] == 64
    st = case.handle()
    o = case.block(st, 0, bs)
    opts = dict(rare_mac=float(np.median(o["mac"])), min_mac=5.0)
    status, coef, vcov = st.interaction_bt(**opts)
    c = check_wald(case, st, 0, o, status, coef, vcov, opts)
    assert c[1] + c[3] > bs * P // 3


def test_interaction_qt_and_bt_interleaved_match_fresh_handles(tmp_path):
    """One handle with both trait kinds' chromosome and interaction state, the quantitative-trait and binary-trait
    interaction calls (and Firth) interleaved block by block, against a fresh handle of each kind: the same bits."""
    from regenie_b200 import capi
    case = Case(tmp_path, "bed", M=150, bs=72)
    rng = np.random.default_rng(11)
    res = rng.normal(size=case.mask.shape) * case.mask
    scf = np.array([1.3, 0.7])

    def qt_state(st):
        st.set_chr(res, scf)
        st.set_interaction(case.E)

    both = case.handle()
    qt_state(both)
    qt = capi.Step2(case.X, case.mask, case.ia.astype(np.uint8), case.n_analyzed, case.bs_max)
    qt_state(qt)
    bt = case.handle()
    n_qt = n_bt = n_f = 0
    for s0 in range(0, case.M, case.bs):
        s1 = min(case.M, s0 + case.bs)
        rows = case.rows[s0:s1]
        got, want = [], []
        for st, out in ((both, got), (qt, want)):
            st.block_bed(rows, min_mac=5.0)
            out.append(st.interaction(min_mac=5.0, force_robust=True))
        for st, out in ((both, got), (bt, want)):
            case.block(st, s0, s1)
            r = st.interaction_bt(min_mac=5.0)
            out.append(r)
            sel = np.argwhere(np.isin(r[0], (1, 3)))[:40]
            out.append(st.interaction_firth(sel[:, 0], sel[:, 1]))
        for g, w in zip(got, want):
            for a, b in zip(g, w):
                assert np.array_equal(a, b)
        n_qt += int((got[0][0] == 1).sum())
        n_bt += int(np.isin(got[1][0], (1, 3)).sum())
        n_f += int((got[2][3] == 0).sum())
    assert n_qt > 100 and n_bt > 100 and n_f > 40
