"""Conditional analysis (--condition-list / --condition-file) against its definition: a conditioned run equals an
unconditioned run whose covariate file carries the conditioning genotypes as extra columns, with the listed IDs passed to
--exclude (extract_condition_snps, src/Pheno.cpp:952-983: the variants become covariate columns before the basis is
formed).  Shared by the CPU (mock ABI) and the GPU driver tests."""
import os

import numpy as np

from oracle import bgen as obgen, pgen as opgen, plink
from regenie_b200 import synth
import helpers


def source_calls(fmt, path, ids, sample=None):
    """Genotypes of `ids` in a .bed / .pgen / .bgen fileset as the driver codes them, in integer units: allele counts
    (unit 1) or 8-bit dosages p1 + 2 p0 (unit 255).  -> (FID_IID keys in file order, {id: (num int64 [n], called bool [n])},
    unit)."""
    out = {}
    if fmt == "bed":
        keys, _ = plink.read_fam(path + ".fam")
        bim = plink.read_bim(path + ".bim")
        at = {v: int(bim.offset[k]) for k, v in enumerate(bim.ids)}
        for i in ids:
            g = plink.decode_bed(plink.read_bed_rows(path + ".bed", len(keys), [at[i]]), len(keys))[0]
            out[i] = (np.where(g == -3, 0, g).astype(np.int64), g != -3)
        return keys, out, 1
    if fmt == "pgen":
        keys, _ = opgen.read_psam(path + ".psam")
        at = {r[2]: k for k, r in enumerate(opgen.read_pvar(path + ".pvar"))}
        pg = opgen.Pgen(path + ".pgen")
        for i in ids:
            g = pg.read(at[i]).astype(np.int64)
            out[i] = (np.where(g == 3, 0, g), g != 3)
        return keys, out, 1
    b = obgen.Bgen(path)
    if sample:
        keys = ["_".join(l.split()[:2]) for l in open(sample).read().splitlines()[2:] if l.strip()]
    else:
        keys = list(b.sample_ids)
    for _c, _p, rsid, _a, p0, p1, miss in b.variants():
        if rsid in ids:
            out[rsid] = ((p1.astype(np.int64) + 2 * p0.astype(np.int64)) * ~miss, ~miss)
    return keys, out, 255


def write_conditioned_covariates(dst, covar, main_keys, src):
    """`covar` plus one column per conditioning variant (ID order), mean-imputed over the samples of the main genotype
    file with complete covariates that have a call, written with %.17g so that the values read back exactly."""
    keys_src, calls, unit = src
    ids = sorted(calls)
    rows = [l.split() for l in open(covar).read().splitlines() if l.strip()]
    main = set(main_keys)
    in_cov = {t[0] + "_" + t[1] for t in rows[1:] if "NA" not in t[2:]} & main
    pos = {k: j for j, k in enumerate(keys_src)}
    cols = []
    for i in ids:
        num, called = calls[i]
        sel = [pos[k] for k in keys_src if k in in_cov and called[pos[k]]]
        total, ns = int(num[sel].sum()), len(sel)
        mu = total / (unit * ns)
        col = {}
        for t in rows[1:]:
            k = t[0] + "_" + t[1]
            j = pos.get(k)
            col[k] = (num[j] / 255.0 if unit == 255 else float(num[j])) if (j is not None and called[j]) else mu
        cols.append(col)
    with open(dst, "w") as fh:
        fh.write(" ".join(rows[0] + ["cond_%s" % i for i in ids]) + "\n")
        for t in rows[1:]:
            k = t[0] + "_" + t[1]
            fh.write(" ".join(t + ["%.17g" % c[k] for c in cols]) + "\n")
    return ids


def write_external(tmp, fmt, keys, seed=5, n_var=3, shared_id=None):
    """An external fileset of `fmt` over `keys` (FID_IID, in file order) with n_var variants, every one with some missing
    calls; the first variant is named `shared_id` when given (an ID of the main file too).  -> (path, [ids])."""
    rng = np.random.default_rng(seed)
    N = len(keys)
    ids = ["ext_%d" % v for v in range(n_var)]
    if shared_id is not None:
        ids[0] = shared_id
    pos = [10 + v for v in range(n_var)]
    os.makedirs(tmp, exist_ok=True)
    if fmt == "bgen":
        probs, miss = helpers.synthetic_dosage_probs(n_var, N, seed=seed, miss_rate=0.05)
        path = os.path.join(tmp, "ext.bgen")
        helpers.write_bgen(path, probs, miss, [1] * n_var, pos, ids, sample_ids=keys)
        return path, ids
    g = rng.binomial(2, rng.uniform(0.1, 0.5, n_var)[:, None], (n_var, N))
    g[rng.random((n_var, N)) < 0.05] = 3
    prefix = os.path.join(tmp, "ext")
    if fmt == "bed":
        with open(prefix + ".bed", "wb") as fh:
            fh.write(b"\x6c\x1b\x01" + synth.pack_bed(g).tobytes())
        with open(prefix + ".bim", "w") as fh:
            for v in range(n_var):
                fh.write("1 %s 0 %d A G\n" % (ids[v], pos[v]))
        with open(prefix + ".fam", "w") as fh:
            for k in keys:
                f, i = k.split("_", 1)
                fh.write("%s %s 0 0 1 -9\n" % (f, i))
    else:
        synth.write_pgen(prefix, g)
        helpers.write_pvar_psam(prefix, [1] * n_var, ids, pos, ["A"] * n_var, ["G"] * n_var, keys)
    return prefix, ids


def shuffled_subset(keys, frac=0.85, seed=3):
    rng = np.random.default_rng(seed)
    sub = [keys[j] for j in rng.permutation(len(keys))[:int(frac * len(keys))]]
    return sub


MAIN = {"bed": ("--bed", "/example"), "pgen": ("--pgen", "/example"), "bgen": ("--bgen", "/example.bgen")}


def check_equivalence(run, read, tmp_path, golden_dir, main, bt, source, step1=False, extra=(), ids=("25", "512", "990")):
    """Step 2 (and with `step1` Step 1 first, whose predictions Step 2 then reads) conditioned on `ids` of the main
    file (source None) or on an external fileset (source = its format, over a shuffled subset of the samples): the
    .regenie / .loco / _pred.list outputs equal those of the oracle run byte for byte."""
    d = golden_dir
    tmp = str(tmp_path)
    os.makedirs(tmp, exist_ok=True)
    opt, suffix = MAIN[main]
    main_path = d + suffix
    main_keys, _ = plink.read_fam(d + "/example.fam")
    lst = os.path.join(tmp, "cond.txt")
    if source is None:
        src_fmt, src_path, cond_ids, cond_opts = main, main_path, list(ids), []
    else:
        src_fmt = source
        src_path, cond_ids = write_external(os.path.join(tmp, "ext"), source, shuffled_subset(main_keys), shared_id="300")
        cond_opts = ["--condition-file", "%s,%s" % (source, src_path)]
    with open(lst, "w") as fh:                               # unsorted, one duplicate: the driver sorts and counts it once
        fh.write("\n".join(list(reversed(cond_ids)) + [cond_ids[0]]) + "\n")
    src = source_calls(src_fmt, src_path, cond_ids)
    assert any((~c).any() for _n, c in src[1].values()) or source is None
    cov = os.path.join(tmp, "cov_oracle.txt")
    write_conditioned_covariates(cov, d + "/covariates.txt", main_keys, src)
    pheno = d + ("/phenotype_bin.txt" if bt else "/phenotype.txt")
    mode = ["--bt"] if bt else []
    outs = {}
    for tag, cv, cond in (("cond", d + "/covariates.txt", ["--condition-list", lst] + cond_opts),
                          ("orac", cov, ["--exclude", lst])):
        o = os.path.join(tmp, tag)
        pred = ["--ignore-pred"]
        if step1:
            log = run(["--step", "1", opt, main_path, "--phenoFile", pheno, "--covarFile", cv, "--bsize", "100", "--out", o + "_s1"]
                      + mode + cond + list(extra))
            if tag == "cond":
                assert "+conditioning on variants in [%s]" % lst in log
            pred = ["--pred", o + "_s1_pred.list"]
        log = run(["--step", "2", opt, main_path, "--phenoFile", pheno, "--covarFile", cv, "--bsize", "100", "--out", o]
                  + pred + mode + (["--firth", "--approx", "--pThresh", "0.1"] if bt else []) + cond + list(extra))
        if tag == "cond":
            want = ("    +conditioning on variants in [%s] n_used = %d" % (lst, len(cond_ids)) if source is None else
                    "      -n_used = %d" % len(cond_ids))
            assert want in log, log[-3000:]
        outs[tag] = o
    names = ("Y1", "Y2")
    for nm in names:
        a, b = read(outs["cond"] + "_%s.regenie" % nm), read(outs["orac"] + "_%s.regenie" % nm)
        assert a == b and len(a.splitlines()) > 100, nm
        tested = {l.split()[2] for l in a.splitlines()[1:]}
        assert not tested & set(cond_ids)
    if step1:
        for k in (1, 2):
            assert read(outs["cond"] + "_s1_%d.loco" % k) == read(outs["orac"] + "_s1_%d.loco" % k)
        la = [l.split()[0] for l in read(outs["cond"] + "_s1_pred.list").splitlines()]
        assert la == [l.split()[0] for l in read(outs["orac"] + "_s1_pred.list").splitlines()] == list(names)
