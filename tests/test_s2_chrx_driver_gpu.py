"""rgb200 --step 2 on a fileset with chromosomes 1 and 23 and sex information, against the oracle rows.

On chromosome 23 the driver hands the kept samples' sex to the library before each chromosome call, and before each block
the non-PAR flags of its variants (in_non_par, src/Geno.cpp:2802-2814: outside [1, par1_max] and [par2_min, ...), hg38 by
default, --par-region b37 moves both bounds).  Flagged variants count their males, coded 0/2, half towards the MAC, so
--minMAC keeps or drops a variant by the male rule; chromosome 1 keeps the autosomal rule in the same run.  The calls are
written as .bed, .pgen (SEX in the .psam) and 8-bit .bgen (sex in the .sample); every row of every output must equal the
oracle's row (step2.sumstats_row), with male= / non_par= on chromosome 23 only.
"""
import math
import os
import subprocess

import numpy as np
import pytest

import helpers
from oracle import plink, prep, step2, step2_bt

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RGB = os.path.join(ROOT, "regenie_b200", "rgb200")
N, M1, P, C = 1200, 120, 2, 2
MIN_MAC = 20.25                     # MACs are halves: no variant sits on the threshold
PAR = {"hg38": (2781479, 155701383), "b37": (2699520, 154931044)}


def run(args):
    r = subprocess.run([RGB] + args, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


def close(a, b, rtol=1.5e-5):
    """Printed 6-significant-digit values: equal up to the reference's own rounding noise."""
    if a == b:
        return True
    if "NA" in (a, b):
        return False
    x, y = float(a), float(b)
    return abs(x - y) <= rtol * max(abs(x), abs(y)) + 1e-12


def _positions(rng):
    """Chromosome-23 positions on both sides of the hg38 and b37 PAR bounds: PAR1 in both builds, PAR1 in hg38 only, the
    non-PAR middle, PAR2 in b37 only, PAR2 in both."""
    zones = [(60000, 2699520, 40), (2699521, 2781479, 40), (2781480, 154931043, 180), (154931044, 155701382, 40),
             (155701383, 156030895, 40)]
    pos = [np.sort(rng.choice(np.arange(lo, hi + 1), n, replace=False)) for lo, hi, n in zones]
    pos = np.concatenate(pos)
    pos[[0, 40, 79, 80, 259, 260, 299, 300]] = [1, 2699520, 2781479, 2781480, 154931043, 154931044, 155701382, 155701383]
    return np.sort(pos)


def _fileset(tmp_path):
    """Chromosome 1 then 23; males (even samples, sex 1 in every sample file) coded 0/2 with a few 1s; 3 % missing.
    Most variants are rare, with an autosomal MAC of about 10-40, so that the male rule moves many across --minMAC."""
    from regenie_b200 import synth
    rng = np.random.default_rng(23)
    pos23 = _positions(rng)
    M = M1 + len(pos23)
    male = np.arange(N) % 2 == 0
    af = np.where(rng.random(M) < 0.7, rng.uniform(0.004, 0.016, M), rng.uniform(0.05, 0.6, M))
    g = rng.binomial(2, af[:, None], size=(M, N))
    g = np.where(male[None, :], 2 * rng.binomial(1, af[:, None], size=(M, N)), g)
    g = np.where(male[None, :] & (rng.random((M, N)) < 0.003), 1, g)
    g = np.where(rng.random((M, N)) < 0.03, 3, g).astype(np.uint8)
    Y, cov, na = synth.phenotypes(np.where(g == 3, 0, g).astype(np.uint8), P, C, seed=23, na_frac=0.04)
    prefix = helpers.write_fileset(str(tmp_path), g, Y, cov, na, n_chr=1)           # fam sex = 1 + s % 2
    chroms = np.array([1] * M1 + [23] * len(pos23))
    pos = np.concatenate([1000 + 10 * np.arange(M1), pos23])
    ids = ["rs%d" % i for i in range(M)]
    with open(prefix + ".bim", "w") as fh:
        for i in range(M):
            fh.write("%d %s 0 %d A G\n" % (chroms[i], ids[i], pos[i]))
    keys, _ = plink.read_fam(prefix + ".fam")
    helpers.write_pgen(prefix, g)
    helpers.write_pvar_psam(prefix, chroms, ids, pos, ["G"] * M, ["A"] * M, keys, sex=[1 + s % 2 for s in range(N)])
    probs = np.stack([(g == 2) * 255, (g == 1) * 255], axis=-1).astype(np.uint8)
    helpers.write_bgen(prefix + ".bgen", probs, g == 3, chroms, pos, ids, alleles=("A", "G"), sample_ids=keys)
    with open(prefix + ".sample", "w") as fh:
        fh.write("ID_1 ID_2 missing sex\n0 0 0 D\n")
        for k in keys:
            f, i = k.split("_", 1)
            fh.write("%s %s 0 %d\n" % (f, i, 1 if int(i[1:]) % 2 == 0 else 2))
    yb = Y > np.quantile(Y, 0.7, axis=0)
    with open(str(tmp_path / "pheno_bin.txt"), "w") as fh:
        fh.write("FID IID Y1 Y2\n")
        for s in range(N):
            fh.write("F%d I%d " % (s, s) + " ".join("NA" if na[s, p] else str(int(yb[s, p])) for p in range(P)) + "\n")
    gk = np.where(g == 3, -3.0, g.astype(np.float64))
    return dict(prefix=prefix, keys=keys, g=gk, male=male, chroms=chroms, pos=pos, ids=ids)


def _oracle_rows(fs, pheno, mode, par, bgen_fmt):
    """{trait: rows} of the oracle for the whole fileset: the male rule on the non-PAR variants of chromosome 23."""
    bt = mode != "qt"
    covar = os.path.dirname(fs["prefix"]) + "/covar.txt"
    pr = (prep.prepare(fs["keys"], pheno, covar, bt=True, step=2) if bt else
          helpers.prepare_step2_with_mask(fs["keys"], pheno, covar, np.ones((N, P), dtype=bool)))
    ia, mask, male = pr.in_analysis, pr.mask, fs["male"]
    lo, hi = PAR[par]
    rows = {nm: [] for nm in pr.pheno_names}
    n_moved = 0
    if bt:
        z_thr = math.sqrt(3.841458820694124)
        sts = [step2_bt.BtChrom(pr.Y_raw[:, j], pr.X, np.zeros(N), mask[:, j]) for j in range(P)]
    else:
        res, _, scf = step2.compute_res(pr.Y, np.zeros_like(pr.Y), mask, pr.neff, pr.ncov, pr.scale_Y)
        YtX = res.T @ pr.X
    for v in range(len(fs["ids"])):
        c, pos, g = int(fs["chroms"][v]), int(fs["pos"][v]), fs["g"][v]
        npar = c == 23 and not (pos <= lo or pos >= hi)
        sx = dict(male=male, non_par=True) if npar else {}
        head = (c, pos, fs["ids"][v], "G", "A")
        if npar:
            n_moved += step2.variant_stats(g, ia, mask, **sx)["ignored"] != step2.variant_stats(g, ia, mask)["ignored"]
        if bt:
            for j, nm in enumerate(pr.pheno_names):
                r = step2_bt.score_bt(g, np.zeros(N), ia, mask[:, j], pr.Y_raw[:, j], sts[j], z_thr, N,
                                      correction=mode, min_mac=MIN_MAC, **sx)
                if r is not None:
                    rows[nm].append(step2.sumstats_row(*head, r["af"], r["n"], r["beta"], r["se"], r["chisq"], r["logp"],
                                                       info=r["info"] if bgen_fmt else None, test_pass=not r["test_fail"]))
            continue
        vs = step2.variant_stats(g, ia, mask, **sx)
        if vs["ignored"]:
            continue
        sc = step2.score_qt(vs["g"], pr.X, res, mask, ia, pr.n_analyzed, pr.ncov, scf, YtX, False)
        if sc is None:
            continue
        for j, nm in enumerate(pr.pheno_names):
            if not vs["ignored_trait"][j]:
                rows[nm].append(step2.sumstats_row(*head, vs["af"][j], vs["ns"][j], sc["beta"][j], sc["se"][j], sc["chisq"][j],
                                                   sc["logp"][j], info=1.0 if bgen_fmt else None))
    return rows, n_moved


def _compare(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for x, y in zip(got, want):
        tx, ty = x.split(), y.split()
        assert len(tx) == len(ty), (what, x, y)
        exact = [0, 1, 2, 5, len(tx) - 7, len(tx) - 6, len(tx) - 1]                      # ..., A1FREQ, N, TEST, EXTRA
        assert [tx[k] for k in exact] == [ty[k] for k in exact], (what, x, y)
        for k in range(6, len(tx) - 1):
            if k not in exact:
                assert close(tx[k], ty[k]), (what, "column %d" % k, x, y)


@pytest.mark.parametrize("fmt,mode", [("bed", "qt"), ("pgen", "qt"), ("bgen", "qt"), ("bed", "firth"), ("pgen", "spa"),
                                      ("bgen", "firth")])
def test_driver_chromosome_x_rows(tmp_path, monkeypatch, fmt, mode):
    """Chromosome 23 in four blocks of --bsize 64 (300 variants, the flags change from block to block) after chromosome 1;
    --minMAC 20.25.  QT runs also with --par-region b37; the .bed runs also as a --chr 23 job, whose rows equal the
    chromosome-23 rows of the full run."""
    fs = _fileset(tmp_path)
    prefix = fs["prefix"]
    geno = {"bed": ["--bed", prefix], "pgen": ["--pgen", prefix], "bgen": ["--bgen", prefix + ".bgen", "--sample", prefix + ".sample"]}[fmt]
    pheno = str(tmp_path / ("pheno.txt" if mode == "qt" else "pheno_bin.txt"))
    base = ["--step", "2"] + geno + ["--phenoFile", pheno, "--covarFile", str(tmp_path / "covar.txt"), "--bsize", "64",
                                     "--ignore-pred", "--minMAC", str(MIN_MAC)]
    if mode != "qt":
        base += ["--bt", "--firth", "--approx"] if mode == "firth" else ["--bt", "--spa"]
    monkeypatch.setattr(step2, "MIN_MAC", MIN_MAC)
    runs = [("hg38", [])] + ([("b37", ["--par-region", "b37"])] if mode == "qt" else [])
    want_sets = {}
    for par, extra in runs:
        out = str(tmp_path / ("o_" + par))
        run(base + extra + ["--out", out])
        want, n_moved = _oracle_rows(fs, pheno, mode, par, fmt == "bgen")
        assert n_moved > 10, n_moved
        for nm, rows in want.items():
            got = open(out + "_%s.regenie" % nm).read().splitlines()
            assert got[0] == (step2.HEADER_INFO if fmt == "bgen" else step2.HEADER).strip()
            _compare(got[1:], rows, (fmt, mode, par, nm))
            assert sum(r.startswith("1 ") for r in rows) > 50 and sum(r.startswith("23 ") for r in rows) > 100
        want_sets[par] = {nm: {r.split()[2] for r in rows} for nm, rows in want.items()}
    if mode == "qt":                                                    # the b37 bounds change the variant set
        assert want_sets["hg38"] != want_sets["b37"]
    if fmt == "bed":
        run(base + ["--chr", "23", "--out", str(tmp_path / "x")])
        for nm in ("Y1", "Y2"):
            full = open(str(tmp_path / "o_hg38") + "_%s.regenie" % nm).read().splitlines()
            job = open(str(tmp_path / "x") + "_%s.regenie" % nm).read().splitlines()
            assert job[0] == full[0] and job[1:] == [r for r in full[1:] if r.startswith("23 ")], nm
