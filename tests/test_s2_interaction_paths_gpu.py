"""GxE interaction tests (rg_s2_set_interaction / rg_s2_interaction) at the shapes that select their chunking: several
sample chunks of kStatChunk = 2048 with a partly filled last one, host slabs of kIntSlab = 16 384 feature rows with a
partial last slab, more than kIntTG = 8 traits (a second and third trait group of the meat kernel), 64 covariates (the
robust columns straddle two 128-column CTAs of the sums kernel) and N = 300 000.

Every case asserts through the "int_paths" debug view which shape ran.  The feature rows are rebuilt bit for bit in
numpy, the routes follow the rule of s2_int_route_kernel, the chunk-reduced sums stay within the error bound of their
fixed summation order against a long-double reference, and the statistics match interaction_oracle.py within 1e-5
relative.  Invariants that hold bit for bit: one trait of a P = 17 handle against a P = 1 handle, the block partition,
option and block-size changes on one handle, a chromosome change, and a sample subset of a shuffled file.  Status edges:
skip_int, a constant E, and the HLM trait order (a near-singular trait ends the rows of the traits after it).
"""
import numpy as np
import pytest

import helpers
import interaction_oracle as io
from oracle import bgen, plink, step2

pytestmark = pytest.mark.gpu

RTOL = 1e-5
CHUNK, SLAB = 2048, 16384
INF = 1e15                                     # rare_mac above every MAC: every variant on the HLM route

# name: N, P, C, K (columns of the HLM X), and the shape it selects: Npad, sample chunks, host slabs, trait groups
CASES = {
    "chunk_full": (2048, 8, 4, 3, (2048, 1, 1, 1)),
    "chunk_part": (2049, 9, 4, 3, (2176, 2, 1, 2)),
    "chunks3": (5001, 17, 4, 64, (5120, 3, 1, 3)),
    "slab_full": (16384, 2, 4, 3, (16384, 8, 1, 1)),
    "slab_part": (16385, 2, 4, 3, (16512, 9, 2, 1)),
    "many": (40001, 3, 4, 8, (40064, 20, 3, 1)),
    "wide": (5001, 9, 64, 64, (5120, 3, 1, 2)),
    "large": (300000, 2, 4, 6, (300032, 147, 19, 1)),
}
MODES = {
    "hlm": dict(rare_mac=INF),
    "split": dict(),                           # rare_mac between the variants' MACs: both routes in one call
    "hc3": dict(force_robust=True),
    "hc4": dict(force_robust=True, force_hc4=True),
    "model": dict(force_robust=True, no_robust=True),
}


class Data:
    pass


def _make(name, e_in_x=False, seed=11):
    """Samples, covariates, traits, E, the oracle's HLM null state per trait and the genotypes of one case.  The analysis
    has --remove-style holes on both sides of every chunk and slab boundary; a few variants have MAC below 5."""
    N, P, C, K, _ = CASES[name]
    rng = np.random.default_rng(seed + N + P + C)
    d = Data()
    d.name, d.N, d.P, d.C, d.K, d.npad = name, N, P, C, K, CASES[name][4][0]
    d.M = 64 if N > 20000 else 96
    ia = rng.random(N) > 0.03
    for b in list(range(CHUNK, N, CHUNK)) + list(range(SLAB, N, SLAB)):
        ia[b - 3:b - 1] = False
        ia[b + 1:b + 3] = False
    ia[N - 2] = False
    d.ia = ia
    d.E = np.where(ia, rng.normal(size=N) * 1.5 + 0.3, 0.0)
    A = np.column_stack([np.ones(N), d.E, rng.normal(size=(N, C))] if e_in_x else
                        [np.ones(N), rng.normal(size=(N, C))])[:, :C]
    d.X = np.zeros((N, C))
    d.X[ia] = np.linalg.qr(A[ia])[0]            # orthonormal basis of the covariates on the analysed samples
    d.mask = ia[:, None] & (rng.random((N, P)) > 0.05)
    d.n_analyzed = int(ia.sum())
    Y = rng.normal(size=(N, P))
    Y = (Y - d.X @ (d.X.T @ Y)) * d.mask
    blups = rng.normal(size=(N, P)) * 0.3 * d.mask
    d.res, _, d.scf = step2.compute_res(Y, blups, d.mask, d.mask.sum(axis=0), C, np.ones(P))
    # HLM null state: X_hlm = (covariates, E^2, blup) cut or padded with random columns to K columns
    V, _ = io.hlm_design(d.E, d.X, blups[:, 0])
    d.dinv, d.px, d.yres = np.zeros((N, P)), [], np.zeros((N, P))
    for p in range(P):
        _, Xh = io.hlm_design(d.E, d.X, blups[:, p])
        if K < Xh.shape[1]:
            Xh = np.column_stack([Xh[:, :K - 2], Xh[:, C:]])
        if Xh.shape[1] < K:
            Xh = np.column_stack([Xh, rng.normal(size=(N, K - Xh.shape[1])) * ia[:, None]])
        y = (Y[:, p] + 0.2 * d.E * Y[:, p]) * d.mask[:, p]
        b, _ = io.hlm_fit(y, d.mask[:, p], Xh, V)
        d.dinv[:, p], Px, d.yres[:, p] = io.hlm_state(y, d.mask[:, p], Xh, V, b)
        d.px.append(Px)
    from regenie_b200 import synth
    g = synth.genotypes(N, d.M, seed=seed, miss=0.02, maf_lo=0.005)
    for v in range(3):                         # MAC below min_mac: ignored traits
        g[v] = np.where(g[v] == 3, 3, 0)
        g[v, rng.choice(np.where(ia)[0], v + 1, replace=False)] = 1
    d.bed = synth.pack_bed(g)
    d.probs, d.pmiss = helpers.synthetic_dosage_probs(d.M, N, seed=seed)
    return d


@pytest.fixture(scope="module")
def data():
    """One Data per case and covariate layout, built (HLM null fits included) once for the module."""
    cache = {}

    def get(name, e_in_x=False):
        if (name, e_in_x) not in cache:
            cache[(name, e_in_x)] = _make(name, e_in_x)
        return cache[(name, e_in_x)]
    return get


def handle(d, bs_max, traits=None, hlm=True, res=None, E=None):
    from regenie_b200 import capi
    t = list(range(d.P)) if traits is None else list(traits)
    st = capi.Step2(d.X, d.mask[:, t], d.ia.astype(np.uint8), d.n_analyzed, bs_max)
    st.set_chr((d.res if res is None else res)[:, t], d.scf[t])
    E = d.E if E is None else E
    if hlm:
        st.set_interaction(E, d.dinv[:, t], [d.px[p] for p in t], d.yres[:, t])
    else:
        st.set_interaction(E)
    return st


def genotypes(d, kind):
    """(code [M, N]: the integer dosage x 255 the kernels read, -1 = missing; g [M, N]: the oracle's genotypes, -3 =
    missing) of the case's variants for kind "bed", "bed_rf" (.bed rows with --ref-first) or "bgen8"."""
    if kind == "bgen8":
        p = d.probs.astype(np.int64)
        code = np.where(d.pmiss, -1, p[..., 1] + 2 * p[..., 0])
        g, _ = bgen.dosage(d.probs[..., 0].astype(float), d.probs[..., 1].astype(float), d.pmiss)
        return code, g
    g = plink.decode_bed(d.bed, d.N, ref_first=kind == "bed_rf")
    return np.where(g < 0, -1, np.rint(g * 255)).astype(np.int64), g


def run_block(st, d, kind, s, e, min_mac=5.0, sample_idx=None, src=None):
    """Variants [s, e) of the case (or of `src`, the rows of a file with sample_idx) as one block."""
    if kind in ("bed", "bed_rf"):
        rows = (d.bed if src is None else src)[s:e]
        return st.block_bed(rows, min_mac=min_mac, ref_first=kind == "bed_rf", sample_idx=sample_idx)
    probs, miss = (d.probs, d.pmiss) if src is None else src
    return st.block_bgen8(probs[s:e], (miss[s:e] * 0x80).astype(np.uint8), min_mac=min_mac, sample_idx=sample_idx)


def paths(st):
    return st.debug("int_paths", np.int64, 8)


def check_paths(st, name, bs, K):
    """The chunk, slab and trait-group counts of the case's table row, the feature widths, K and the block size."""
    N, P, C, _, (npad, nchunks, nslabs, ngroups) = CASES[name]
    nr = 2 * C + 2 * P + 3
    want = [nchunks, npad, nr + (P * (2 * K + 5) if K else 0), nr, K, ngroups, nslabs, bs]
    assert paths(st).tolist() == want


def split_mac(o):
    """rare_mac between the variants' smallest trait MACs: about half the variants on each route."""
    return float(np.median(o["mac"].min(axis=1)))


def opts_for(mode, o):
    opts = dict(min_mac=5.0, **MODES[mode])
    if mode == "split":
        opts["rare_mac"] = split_mac(o)
    if mode == "hc4":
        opts["rare_mac"] = float(np.median(o["mac"]))   # HC4 for the traits with MAC <= rare_mac
    return opts


def want_route(o, K, opts):
    rare = (o["mac"] < opts.get("rare_mac", 1000.0)).any(axis=1)
    robust_only = K == 0 or opts.get("force_robust", False) or opts.get("no_robust", False)
    return np.where(o["flags"] & 3, 0, np.where(rare & (not robust_only), 2, 1)).astype(np.int8)


def feature_rows(d, hlm):
    """int_F rebuilt with the products rg_s2_set_interaction forms, in its order: [Npad][nf]."""
    N, P, C, K, npad = d.N, d.P, d.C, d.K if hlm else 0, d.npad
    nr = 2 * C + 2 * P + 3
    nf = nr + (P * (2 * K + 5) if K else 0)
    F = np.zeros((npad, nf))
    ia = d.ia
    e = np.where(ia, d.E, 0.0)[:, None]
    X, R = d.X, d.res
    F[:N, :C] = X
    F[:N, C:2 * C] = e * X
    F[:N, 2 * C:2 * C + P] = R
    F[:N, 2 * C + P:2 * C + 2 * P] = e * R
    F[:N, 2 * C + 2 * P] = 1.0
    F[:N, 2 * C + 2 * P + 1] = e[:, 0]
    F[:N, 2 * C + 2 * P + 2] = e[:, 0] * e[:, 0]
    for p in range(P if K else 0):
        t = nr + p * (2 * K + 5)
        dd, y = d.dinv[:, p][:, None], d.yres[:, p]
        x = dd * d.px[p]
        F[:N, t:t + K] = x
        F[:N, t + K:t + 2 * K] = e * x
        F[:N, t + 2 * K] = dd[:, 0] * y
        F[:N, t + 2 * K + 1] = (dd[:, 0] * e[:, 0]) * y
        d2 = dd[:, 0] * dd[:, 0]
        F[:N, t + 2 * K + 2] = d2
        F[:N, t + 2 * K + 3] = d2 * e[:, 0]
        F[:N, t + 2 * K + 4] = (d2 * e[:, 0]) * e[:, 0]
    F[:N][~ia] = 0.0
    pow2 = np.zeros(nf, dtype=bool)
    pow2[2 * C + 2 * P:nr] = True
    for p in range(P if K else 0):
        t = nr + p * (2 * K + 5) + 2 * K + 2
        pow2[t:t + 3] = True
    return F, pow2, nr


def stats(coef, vcov):
    """BETA / SE / CHISQ of the two rows and the 2-DF statistic (src/Interaction.cpp:206-273)."""
    se = np.sqrt(np.diag(vcov))
    return np.concatenate([coef, se, coef ** 2 / np.diag(vcov), [coef @ np.linalg.solve(vcov, coef)]])


def check_oracle(d, o, gimp, out, opts, counts, traits=None, E=None, X=None, state=None):
    """Every (variant, trait) of one interaction() call against interaction_oracle.py: the route rule, then on the HLM
    route the reference's trait order (an ignored trait is skipped; a near-singular trait gets -1 and ends the rows of
    the traits after it), on the robust route io.robust."""
    status, coef, vcov = out
    t = list(range(d.P)) if traits is None else list(traits)
    E = d.E if E is None else E
    X = d.X if X is None else X
    dinv, px, yres = state or (d.dinv, d.px, d.yres)
    K = px[t[0]].shape[1] if px else 0
    route = want_route(o, K, opts)
    min_mac = opts["min_mac"]
    for v in range(len(route)):
        if route[v] == 0:
            assert (status[v] == 0).all()
            continue
        mac = o["mac"][v]
        if route[v] == 2:
            dead = False
            for i, p in enumerate(t):
                if mac[i] < min_mac:
                    assert status[v, i] == 0
                    continue
                if dead:
                    assert status[v, i] == -1, (v, i)
                    continue
                want = io.hlm_test(gimp[v], E, dinv[:, p], px[p], yres[:, p])
                if want is None:
                    assert status[v, i] == -1, (v, i)
                    dead = True
                    continue
                assert status[v, i] == 2, (v, i, status[v, i])
                counts[2] += 1
                got, ref = stats(coef[v, i], vcov[v, i]), stats(*want)
                assert np.allclose(got, ref, rtol=RTOL, atol=0), (v, i, got, ref)
            continue
        r = io.robust(gimp[v], E, X, d.res[:, t], d.mask[:, t].astype(float), d.scf[t], d.n_analyzed, mac,
                      opts.get("rare_mac", 1000.0), opts.get("force_hc4", False), opts.get("no_robust", False))
        for i in range(len(t)):
            if mac[i] < min_mac:
                assert status[v, i] == 0
                continue
            if r is None:
                assert status[v, i] in (0, -1)
                continue
            assert status[v, i] == 1, (v, i, status[v, i])
            counts[1] += 1
            got, ref = stats(coef[v, i], vcov[v, i]), stats(r[0][i], r[1][i])
            assert np.allclose(got, ref, rtol=RTOL, atol=0), (v, i, got, ref)


def with_200_variants(d):
    """The case with 200 other variants."""
    from regenie_b200 import synth
    d2 = Data()
    d2.__dict__.update(d.__dict__)
    d2.M = 200
    d2.bed = synth.pack_bed(synth.genotypes(d.N, 200, seed=5, miss=0.02, maf_lo=0.005))
    d2.probs, d2.pmiss = helpers.synthetic_dosage_probs(200, d.N, seed=5)
    return d2


def same(a, b):
    """Two interaction() results give the same bits: every status, and coef / vcov of the pairs with rows (status 1 or 2;
    the library writes no coefficients for the others)."""
    assert np.array_equal(a[0], b[0])
    rows = a[0] > 0
    assert np.array_equal(a[1][rows], b[1][rows]) and np.array_equal(a[2][rows], b[2][rows])


# ---------------------------------------------------------------------------------------------------- feature rows
@pytest.mark.parametrize("hlm", [True, False], ids=["hlm", "no_hlm"])
@pytest.mark.parametrize("name", list(CASES))
def test_feature_rows_bit_for_bit(data, name, hlm):
    """int_F equals the numpy products of X, res, E and the HLM state in the host code's order; rows past N and rows
    outside the analysis (holes on both sides of every slab and chunk boundary) are zero."""
    d = data(name)
    st = handle(d, 40, hlm=hlm)
    run_block(st, d, "bed", 0, 40)
    st.interaction()
    check_paths(st, name, 40, d.K if hlm else 0)
    F, _, _ = feature_rows(d, hlm)
    got = st.debug("int_F", np.float64, F.size).reshape(F.shape)
    assert np.array_equal(got, F)
    assert not got[d.N:].any() and not got[:d.N][~d.ia].any()
    assert got[:d.N][d.ia].any(axis=1).all()


# ------------------------------------------------------------------------------------------------- routes and sums
@pytest.mark.parametrize("name", list(CASES))
def test_routes_and_sums(data, name):
    """int_route follows the route rule, and every (v, f) the route reads is sum_i g_v(i)^(1|2) F[i][f] within the bound
    of the in-chunk sequential sum plus the fixed-order chunk sum.  rare_mac splits the block between the routes, so CTAs
    that straddle the robust / HLM column boundary and CTAs that return early both run."""
    d = data(name)
    bs = 40
    st = handle(d, bs)
    o = run_block(st, d, "bed", 0, bs)
    opts = dict(rare_mac=split_mac(o), min_mac=5.0)
    st.interaction(**opts)
    check_paths(st, name, bs, d.K)
    nchunks = CASES[name][4][1]
    route = st.debug("int_route", np.int8, bs)
    want = want_route(o, d.K, opts)
    assert np.array_equal(route, want)
    assert (route == 1).sum() >= 8 and (route == 2).sum() >= 8
    F, pow2, nr = feature_rows(d, True)
    sums = st.debug("int_sums", np.float64, bs * F.shape[1]).reshape(bs, -1)
    code, _ = genotypes(d, "bed")
    npad = F.shape[0]
    G = np.zeros((bs, npad))
    G[:, :d.N] = np.where(code[:bs] < 0, 2.0 * o["af_all"][:, None], code[:bs] * (1.0 / 255.0))
    Fl = F.astype(np.longdouble)
    Gl = G.astype(np.longdouble)
    ref = np.zeros((bs, F.shape[1]), dtype=np.longdouble)
    ref[:, ~pow2] = Gl @ Fl[:, ~pow2]
    ref[:, pow2] = (Gl * Gl) @ Fl[:, pow2]
    mag = np.zeros((bs, F.shape[1]))
    mag[:, ~pow2] = np.abs(G) @ np.abs(F[:, ~pow2])
    mag[:, pow2] = (G * G) @ np.abs(F[:, pow2])
    tol = (CHUNK + nchunks + 4) * 2.0 ** -53 * mag
    cols = np.arange(F.shape[1])
    need = np.where(route[:, None] == 1, cols[None, :] < nr, np.where(route[:, None] == 2, cols[None, :] >= nr, False))
    err = np.abs((sums - ref).astype(np.float64))
    bad = need & ~(err <= tol)
    assert not bad.any(), (np.argwhere(bad)[:5], err[bad][:5], tol[bad][:5])


# ---------------------------------------------------------------------------------------- statistics vs the oracle
STAT_RUNS = [(n, "bed", False) for n in CASES] + [("chunk_part", "bed_rf", False), ("chunk_part", "bgen8", False),
                                                  ("slab_part", "bgen8", False), ("wide", "bgen8", False),
                                                  ("wide", "bed", True)]


@pytest.mark.parametrize("name,kind,e_in_x", STAT_RUNS,
                         ids=["%s-%s%s" % (n, k, "-e_in_x" if e else "") for n, k, e in STAT_RUNS])
def test_interaction_matches_oracle(data, name, kind, e_in_x):
    """BETA, SE, the Wald statistics and the 2-DF statistic of the HLM, split-MAC, HC3, HC4 and model-based runs within
    1e-5 of the oracle, in a block of a size that is not a multiple of 16 and a short final block.  e_in_x: E is a column
    of the orthonormal covariate basis, as when the driver keeps E as a covariate."""
    d = data(name, e_in_x)
    bs = 40 if d.M == 64 else 72
    st = handle(d, bs)
    _, graw = genotypes(d, kind)
    counts = {m: {1: 0, 2: 0} for m in MODES}
    for s in range(0, d.M, bs):
        e = min(d.M, s + bs)
        o = run_block(st, d, kind, s, e)
        gimp, _ = plink.mean_impute_block(graw[s:e], d.ia)
        for mode in MODES:
            opts = opts_for(mode, o)
            out = st.interaction(**opts)
            check_paths(st, name, e - s, d.K)
            check_oracle(d, o, gimp, out, opts, counts[mode])
    for mode in ("hc3", "hc4", "model"):
        assert counts[mode][1] > 50, (mode, counts)
    assert counts["hlm"][2] > 50, counts
    assert counts["split"][1] > 20 and counts["split"][2] > 20, counts


# --------------------------------------------------------------------------------------------- bit-exact invariants
@pytest.mark.parametrize("mode", ["hc3", "hc4", "hlm"])
def test_trait_of_17_equals_single_trait_handle(data, mode):
    """Trait p of a P = 17 handle (three trait groups of the meat kernel, HLM columns at nr + p (2K + 5)) gives the same
    bits as a P = 1 handle of that trait, with the same res column, mask, scf and HLM state."""
    d = data("chunks3")
    bs = d.M
    st = handle(d, bs)
    o = run_block(st, d, "bed", 0, bs)
    opts = opts_for(mode, o)
    status, coef, vcov = st.interaction(**opts)
    check_paths(st, "chunks3", bs, d.K)
    live = ((o["flags"] & 3) == 0)[:, None] & (o["mac"] >= 5.0)
    assert live.sum() > 50
    assert not (status == -1).any()                  # no near-singular trait ending the rows of the later ones
    assert (status[live] == (2 if mode == "hlm" else 1)).all()
    for p in range(d.P):
        s1 = handle(d, bs, traits=[p])
        o1 = run_block(s1, d, "bed", 0, bs)
        assert np.array_equal(o1["mac"][:, 0], o["mac"][:, p])
        r = s1.interaction(**opts)
        same(r, (status[:, [p]], coef[:, [p]], vcov[:, [p]]))


@pytest.mark.parametrize("kind", ["bed", "bgen8"])
def test_block_partition_gives_the_same_bits(data, kind):
    """The same 200 variants in one block, in blocks of 16, and in blocks of 72, 72 and 56."""
    d2 = with_200_variants(data("chunk_part"))
    st = handle(d2, 200)
    o = run_block(st, d2, kind, 0, 200)
    opts = dict(rare_mac=split_mac(o), min_mac=5.0)
    ref = st.interaction(**opts)
    assert (ref[0] == 1).sum() > 50 and (ref[0] == 2).sum() > 50
    for cuts in ([16] * 12 + [8], [72, 72, 56]):
        parts, s = [], 0
        for b in cuts:
            run_block(st, d2, kind, s, s + b)
            parts.append(st.interaction(**opts))
            s += b
        same(ref, [np.concatenate([p[k] for p in parts]) for k in range(3)])


def test_option_changes_on_one_resident_block(data):
    """HLM, robust HC3, HLM again and model-based on one resident block each equal the same call on a fresh handle."""
    d = data("chunks3")
    bs = 72
    st = handle(d, bs)
    o = run_block(st, d, "bed", 0, bs)
    for mode in ("hlm", "hc3", "hlm", "model"):
        opts = opts_for(mode, o)
        got = st.interaction(**opts)
        fresh = handle(d, bs)
        run_block(fresh, d, "bed", 0, bs)
        same(got, fresh.interaction(**opts))


def test_small_block_then_large_block(data):
    """A 16-variant block followed by a 200-variant block (the interaction buffers grow) equals the 200-variant block run
    first."""
    d = with_200_variants(data("chunks3"))
    st = handle(d, 200)
    o = run_block(st, d, "bed", 0, 16)
    st.interaction(**opts_for("split", o))
    check_paths(st, "chunks3", 16, d.K)
    o = run_block(st, d, "bed", 0, 200)
    opts = opts_for("split", o)
    got = st.interaction(**opts)
    check_paths(st, "chunks3", 200, d.K)
    fresh = handle(d, 200)
    run_block(fresh, d, "bed", 0, 200)
    want = fresh.interaction(**opts)
    same(got, want)
    assert (want[0] == 1).sum() > 50 and (want[0] == 2).sum() > 50


def test_chromosome_change(data):
    """Chromosome 1 with K = 64, then set_chr and chromosome 2 with K = 2, then chromosome 2 without HLM state: each
    equals a fresh handle for that chromosome."""
    from regenie_b200 import capi
    d = data("wide")
    bs = 72
    rng = np.random.default_rng(4)
    res2 = d.res * (1.0 + 0.1 * rng.normal(size=d.res.shape))
    V, _ = io.hlm_design(d.E, d.X, d.res[:, 0])
    st2 = []
    for p in range(d.P):                       # a K = 2 null state (b = 0: d = mask)
        Xh = np.column_stack([d.X[:, 0], d.E * d.E * d.ia])
        st2.append(io.hlm_state(d.res[:, p], d.mask[:, p], Xh, V, np.zeros(V.shape[1])))
    dinv2 = np.stack([s[0] for s in st2], 1)
    px2 = [s[1] for s in st2]
    yres2 = np.stack([s[2] for s in st2], 1)

    def chr2(h, hlm):
        h.set_chr(res2, d.scf)
        if hlm:
            h.set_interaction(d.E, dinv2, px2, yres2)
        else:
            h.set_interaction(d.E)

    st = handle(d, bs)
    o = run_block(st, d, "bed", 0, bs)
    opts = opts_for("split", o)
    got = [st.interaction(**opts)]
    check_paths(st, "wide", bs, 64)
    for hlm in (True, False):
        chr2(st, hlm)
        with pytest.raises(capi.RgError):
            st.debug("int_route", np.int8, bs)     # no interaction call on this chromosome yet
        run_block(st, d, "bed", 0, bs)
        got.append(st.interaction(**opts))
        check_paths(st, "wide", bs, 2 if hlm else 0)
    want = []
    for k in range(3):
        h = handle(d, bs)
        if k:
            chr2(h, k == 1)
        run_block(h, d, "bed", 0, bs)
        want.append(h.interaction(**opts))
    for a, b in zip(got, want):
        same(a, b)
    assert (got[1][0] == 2).sum() > 20 and (got[2][0] == 2).sum() == 0 and (got[2][0] == 1).sum() > 50


@pytest.mark.parametrize("kind", ["bed", "bgen8"])
def test_sample_subset_of_a_shuffled_file(data, kind):
    """A file with 1.3 N samples in shuffled order read through sample_idx equals the pre-subsetted rows."""
    from regenie_b200 import synth
    d = data("chunk_part")
    bs = 72
    n_file = int(1.3 * d.N)
    rng = np.random.default_rng(8)
    idx = rng.permutation(n_file)[:d.N].astype(np.int32)      # sample s of the analysis is file sample idx[s]
    if kind == "bed":
        gf = synth.genotypes(n_file, bs, seed=9, miss=0.02, maf_lo=0.005)
        src = synth.pack_bed(gf)
        sub = Data()
        sub.__dict__.update(d.__dict__)
        sub.bed = synth.pack_bed(gf[:, idx])
    else:
        pf, mf = helpers.synthetic_dosage_probs(bs, n_file, seed=9)
        src = (pf, mf)
        sub = Data()
        sub.__dict__.update(d.__dict__)
        sub.probs, sub.pmiss = pf[:, idx], mf[:, idx]
    st = handle(d, bs)
    o = run_block(st, d, kind, 0, bs, sample_idx=idx, src=src)
    opts = opts_for("split", o)
    got = st.interaction(**opts)
    ref = handle(sub, bs)
    o2 = run_block(ref, sub, kind, 0, bs)
    assert np.array_equal(o["mac"], o2["mac"])
    same(got, ref.interaction(**opts))
    assert (got[0] == 1).sum() > 50 and (got[0] == 2).sum() > 50


# ------------------------------------------------------------------------------------------------------ status edges
def test_zero_E_skips_every_pair(data):
    """E = 0 on every analysed sample: resid(E o G) has sd 0 < numtol, so skip_int gives status 0 for every (variant,
    trait), robust route or not."""
    d = data("chunk_part")
    bs = 72
    st = handle(d, bs, hlm=False, E=np.zeros(d.N))
    o = run_block(st, d, "bed", 0, bs)
    status, _, _ = st.interaction(force_robust=True, min_mac=5.0)
    live = ((o["flags"] & 3) == 0)[:, None] & (o["mac"] >= 5.0)
    assert live.sum() > 50
    assert (status == 0).all()
    route = st.debug("int_route", np.int8, bs)
    assert np.array_equal(route, np.where(o["flags"] & 3, 0, 1))


def test_constant_E_is_near_singular(data):
    """E constant over the analysed samples (several chunks): H^T H is near-singular, status -1 for every live pair."""
    d = data("chunk_part")
    bs = 72
    st = handle(d, bs, hlm=False, E=d.ia * 2.0)
    o = run_block(st, d, "bed", 0, bs)
    status, _, _ = st.interaction(force_robust=True, min_mac=5.0)
    live = ((o["flags"] & 3) == 0)[:, None] & (o["mac"] >= 5.0)
    assert live.sum() > 50
    assert (status[live] == -1).all() and (status[~live] == 0).all()


def test_hlm_trait_order(data):
    """P = 3, HLM state built by hand.  Trait 0's mask covers a few hundred samples on which E = 1, so E o G = G there:
    trait 0 is near-singular, and it ends the variant's rows (traits 0, 1 and 2 all -1), as the reference returns.  On
    variants where trait 0 has MAC < min_mac it is ignored instead, and traits 1 and 2 get their rows."""
    from regenie_b200 import capi, synth
    base = data("chunk_part")
    N, P, C = base.N, 3, base.C
    rng = np.random.default_rng(21)
    ia = base.ia
    t0 = np.zeros(N, dtype=bool)
    t0[rng.choice(np.where(ia)[0], 300, replace=False)] = True
    mask = np.stack([t0, ia, ia & (rng.random(N) > 0.1)], 1)
    E = np.where(t0, 1.0, base.E)
    X = base.X
    y = rng.normal(size=(N, P)) * mask
    res, _, scf = step2.compute_res((y - X @ (X.T @ y)) * mask, np.zeros((N, P)), mask, mask.sum(0), C, np.ones(P))
    dinv, px, yres = np.zeros((N, P)), [], np.zeros((N, P))
    for p in range(P):
        dd = mask[:, p].astype(float)
        Px = np.linalg.qr(X * dd[:, None])[0]
        m = dd * y[:, p]
        dinv[:, p], yres[:, p] = dd, m - Px @ (Px.T @ m)
        px.append(Px)
        assert np.abs(Px.T @ yres[:, p]).max() < 1e-10
    M = 96
    g = synth.genotypes(N, M, seed=17, miss=0.0, maf_lo=0.002, maf_hi=0.03)
    st = capi.Step2(X, mask, ia.astype(np.uint8), int(ia.sum()), M)
    st.set_chr(res, scf)
    st.set_interaction(E, dinv, px, yres)
    o = st.block_bed(synth.pack_bed(g), min_mac=5.0)
    opts = dict(rare_mac=INF, min_mac=5.0)
    status, coef, vcov = st.interaction(**opts)
    assert (st.debug("int_route", np.int8, M) == np.where(o["flags"] & 3, 0, 2)).all()
    ok = (o["flags"] & 3) == 0
    dead = ok & (o["mac"][:, 0] >= 5.0)
    ign = ok & (o["mac"][:, 0] < 5.0) & (o["mac"][:, 1:] >= 5.0).all(axis=1)
    assert dead.sum() >= 10 and ign.sum() >= 10, (dead.sum(), ign.sum())
    assert (status[dead] == -1).all()
    assert (status[ign, 0] == 0).all() and (status[ign, 1:] == 2).all()
    gimp, _ = plink.mean_impute_block(plink.decode_bed(synth.pack_bed(g), N).astype(float), ia)
    counts = {1: 0, 2: 0}
    d = Data()
    d.P, d.res, d.mask, d.scf, d.n_analyzed = P, res, mask, scf, int(ia.sum())
    check_oracle(d, o, gimp, (status, coef, vcov), opts, counts, E=E, X=X, state=(dinv, px, yres))
    assert counts[2] >= 20


# ---------------------------------------------------------------------------------------------------------- wrapper
def test_wrapper_sizes_outputs_for_the_last_block(data, monkeypatch):
    """interaction() sizes its outputs for the last block call; a different bs, or a call before any block, raises
    ValueError without reaching the library (which would write the last block's rows past smaller arrays)."""
    from regenie_b200 import capi
    d = data("chunk_full")
    st = handle(d, 72)
    L = capi.lib()

    def unreachable(*a):
        raise AssertionError("rg_s2_interaction reached")
    real = L.rg_s2_interaction
    monkeypatch.setattr(L, "rg_s2_interaction", unreachable)
    with pytest.raises(ValueError):
        st.interaction()
    run_block(st, d, "bed", 0, 72)
    with pytest.raises(ValueError):
        st.interaction(40)
    run_block(st, d, "bed", 0, 40)
    with pytest.raises(ValueError):
        st.interaction(72)
    monkeypatch.setattr(L, "rg_s2_interaction", real)
    a = st.interaction()
    b = st.interaction(40)
    assert a[0].shape == (40, d.P) and a[1].shape == (40, d.P, 2) and a[2].shape == (40, d.P, 2, 2)
    same(a, b)
    assert (a[0] == 1).sum() > 50
