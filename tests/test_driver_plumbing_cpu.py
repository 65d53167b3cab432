"""The rgb200 driver end to end WITHOUT a GPU: its own sources linked against tests/mock/mock_abi.cpp, a CPU stand-in
for the C ABI whose outputs are simple deterministic functions of what the driver hands over (not regenie's
statistics).  What is checked here is the host control flow around the hot path - the equivalences the reference's own
test script checks (test/test_bash.sh: sharded == unsharded, job outputs concatenate, compressed == plain) and the
file formats - so that a change to the driver is caught where no GPU exists.  Numbers are never compared with the
oracle here; that is what tests/test_driver_gpu.py does on the real library.
"""
import glob
import gzip
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MOCK = os.path.join(ROOT, "tests", "mock", "rgb200_mock")


@pytest.fixture(scope="module", autouse=True)
def _built():
    srcs = sorted(glob.glob(os.path.join(ROOT, "regenie_b200", "host", "*.cpp"))) + [os.path.join(ROOT, "tests", "mock", "mock_abi.cpp")]
    deps = (srcs + glob.glob(os.path.join(ROOT, "regenie_b200", "host", "*.hpp")) + [os.path.join(ROOT, "include", "rg_b200.h"),
            os.path.join(ROOT, "regenie_b200", "csrc", "pgen_core.h")])
    if not os.path.exists(MOCK) or any(os.path.getmtime(s) > os.path.getmtime(MOCK) for s in deps):
        r = subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), "-o", MOCK] + srcs +
                           ["-lz", "-lpthread", "-ldl"], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]


def run(args, ok=True):
    r = subprocess.run([MOCK] + [str(a) for a in args], capture_output=True, text=True, timeout=300)
    if ok:
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return r.stdout


def read(path):
    return gzip.open(path, "rt").read() if str(path).endswith(".gz") else open(path).read()


def step1(d, fileset="example_3chr", extra=(), pheno="/phenotype.txt"):
    return ["--step", "1", "--bed", d + "/" + fileset, "--phenoFile", d + pheno, "--covarFile", d + "/covariates.txt",
            "--bsize", "100"] + list(extra)


def test_step1_outputs_gz_prs_and_sharded_equals_unsharded(tmp_path, golden_dir):
    d = golden_dir
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    log = run(step1(d) + ["--out", a])
    assert "<- min value" in log and "List of blup files written to" in log
    run(step1(d, extra=["--gz", "--print-prs", "--lowmem", "--keep-l0", "--lowmem-prefix", str(tmp_path / "tmp_rg")]) + ["--out", b])
    for k in (1, 2):
        plain = read(a + "_%d.loco" % k)
        assert read(b + "_%d.loco.gz" % k) == plain
        rows = {l.split()[0]: l.split()[1:] for l in plain.splitlines()}
        assert len(rows) == 24 and len(rows["FID_IID"]) == 500
        prs = read(b + "_%d.prs.gz" % k).splitlines()
        assert prs[0] == plain.splitlines()[0] and prs[1].split()[0] == "0" and prs[1].split()[1:] == rows["7"]
        assert os.path.getsize(str(tmp_path / "tmp_rg") + "_l0_Y%d" % k) == 8 * 500 * 5 * 6       # N x R x blocks doubles
    assert [l.split()[0] for l in open(a + "_pred.list")] == ["Y1", "Y2"]
    # --split-l0 / --run-l0 / --run-l1 (test/test_bash.sh:91-137), then level 1 for one phenotype only
    par = str(tmp_path / "par")
    run(step1(d) + ["--split-l0", par + ",3", "--out", str(tmp_path / "l0")])
    master = open(par + ".master").read().splitlines()
    assert master[0] == "500 100" and len(master) == 4
    for job in (1, 2, 3):
        run(step1(d) + ["--run-l0", par + ".master,%d" % job, "--out", str(tmp_path / "l0")])
        assert os.path.exists(par + "_job%d_l0_Y1" % job)
    run(step1(d) + ["--run-l1", par + ".master", "--keep-l0", "--out", str(tmp_path / "l1")])
    run(step1(d) + ["--run-l1", par + ".master", "--l1-phenoList", "Y2", "--out", str(tmp_path / "l1b")])
    for k in (1, 2):
        assert read(str(tmp_path / "l1") + "_%d.loco" % k) == read(a + "_%d.loco" % k)
    assert read(str(tmp_path / "l1b") + "_2.loco") == read(a + "_2.loco") and not os.path.exists(str(tmp_path / "l1b") + "_1.loco")
    assert not os.path.exists(par + "_job1_l0_Y1")                      # removed after level 1 unless --keep-l0
    # user grids equal to the default ones, short option names, exclusion lists
    run(["--step", "1", "--bed", d + "/example_3chr", "-p", d + "/phenotype.txt", "-c", d + "/covariates.txt", "-b", "100",
         "--setl0", "0.99,0.01,0.25,0.5,0.75", "--setl1", "0.01,0.25,0.5,0.75,0.99", "-o", str(tmp_path / "g")])
    assert read(str(tmp_path / "g") + "_1.loco") == read(a + "_1.loco")
    run(step1(d, extra=["--phenoCol", "Y2", "--covarColList", "V1,V2"]) + ["--out", str(tmp_path / "h1")])
    run(step1(d, extra=["--phenoExcludeList", "Y1", "--covarExcludeList", "V3"]) + ["--out", str(tmp_path / "h2")])
    assert read(str(tmp_path / "h1") + "_1.loco") == read(str(tmp_path / "h2") + "_1.loco")


def test_step2_qt_jobs_windows_compressed_io_and_prs(tmp_path, golden_dir):
    d = golden_dir
    pheno, covar = d + "/phenotype.txt", d + "/covariates.txt"
    fit = str(tmp_path / "fit")
    run(step1(d, extra=["--print-prs"]) + ["--out", fit])
    s2 = ["--step", "2", "--bed", d + "/example_3chr", "--phenoFile", pheno, "--covarFile", covar, "--bsize", "77", "--pred",
          fit + "_pred.list"]
    full = str(tmp_path / "full")
    run(s2 + ["--out", full])
    rows = read(full + "_Y1.regenie").splitlines()
    assert rows[0] == "CHROM GENPOS ID ALLELE0 ALLELE1 A1FREQ N TEST BETA SE CHISQ LOG10P EXTRA" and len(rows) > 400
    # chromosome jobs concatenate to the full run; a window is the matching slice
    cat = rows[:1]
    for c in (1, 2, 3):
        run(s2 + ["--chr", c, "--out", str(tmp_path / ("chr%d" % c))])
        cat += read(str(tmp_path / ("chr%d" % c)) + "_Y1.regenie").splitlines()[1:]
    assert cat == rows
    pos = sorted(int(l.split()[1]) for l in rows[1:] if l.startswith("2 "))
    lo, hi = pos[len(pos) // 3], pos[2 * len(pos) // 3]
    run(s2 + ["--range", "2:%d-%d" % (lo, hi), "--out", str(tmp_path / "win")])
    assert read(str(tmp_path / "win") + "_Y1.regenie").splitlines()[1:] == \
        [l for l in rows[1:] if l.startswith("2 ") and lo <= int(l.split()[1]) <= hi]
    # .gz everywhere: phenotypes, covariates, prediction files, outputs; sample lists
    for f in ("phenotype.txt", "covariates.txt"):
        with open(d + "/" + f, "rb") as src, gzip.open(tmp_path / (f + ".gz"), "wb") as dst:
            shutil.copyfileobj(src, dst)
    fitz = str(tmp_path / "fitz")
    run(step1(d, extra=["--gz"]) + ["--out", fitz])
    gz = str(tmp_path / "gz")
    run(["--step", "2", "--bed", d + "/example_3chr", "--phenoFile", tmp_path / "phenotype.txt.gz", "--covarFile",
         tmp_path / "covariates.txt.gz", "--bsize", "77", "--pred", fitz + "_pred.list", "--gz", "--write-samples", "--print-pheno",
         "--out", gz])
    for nm in ("Y1", "Y2"):
        assert read(gz + "_%s.regenie.gz" % nm) == read(full + "_%s.regenie" % nm)
        ids = open(gz + "_%s.regenie.ids" % nm).read().split("\n")
        assert ids[0] == nm + "\tNA" and len(ids) == 501 and ids[1] == "1\t1"
    # --use-prs == LOCO files whose rows all hold the PRS; --ignore-pred differs from both
    lst = tmp_path / "fake_pred.list"
    with open(lst, "w") as fl:
        for k, nm in ((1, "Y1"), (2, "Y2")):
            prs = read(fit + "_%d.prs" % k).splitlines()
            with open(tmp_path / ("fake_%d.loco" % k), "w") as fh:
                fh.write(prs[0] + "\n")
                for c in range(1, 24):
                    fh.write(str(c) + " " + prs[1].split(" ", 1)[1] + "\n")
            fl.write("%s %s\n" % (nm, tmp_path / ("fake_%d.loco" % k)))
    base = ["--step", "2", "--bed", d + "/example_3chr", "--phenoFile", pheno, "--covarFile", covar, "--bsize", "77"]
    run(base + ["--pred", lst, "--out", str(tmp_path / "u1")])
    log = run(base + ["--pred", fit + "_prs.list", "--use-prs", "--out", str(tmp_path / "u2")])
    run(base + ["--ignore-pred", "--out", str(tmp_path / "u3")])
    assert " * PRS predictions : [" in log
    u1, u2, u3 = (read(str(tmp_path / u) + "_Y1.regenie") for u in ("u1", "u2", "u3"))
    assert u1 == u2 and u1 != read(full + "_Y1.regenie") and u3 != u1 and u3 != read(full + "_Y1.regenie")
    # .pgen input == .bed input (the reference's fixture pair holds the same calls)
    one = ["--step", "2", "--phenoFile", pheno, "--covarFile", covar, "--bsize", "200", "--ignore-pred"]
    run(one + ["--bed", d + "/example", "--out", str(tmp_path / "pb")])
    run(one + ["--pgen", d + "/example", "--out", str(tmp_path / "pp")])
    assert read(str(tmp_path / "pb") + "_Y2.regenie") == read(str(tmp_path / "pp") + "_Y2.regenie")
    # a sample subset changes N, missing step-1 files are reported like the reference
    run(one + ["--bed", d + "/example", "--remove", d + "/fid_iid_to_remove.txt", "--out", str(tmp_path / "rm")])
    assert {l.split()[6] for l in read(str(tmp_path / "rm") + "_Y1.regenie").splitlines()[1:]} == {"494"}
    out = run(base + ["--pred", d + "/nope_pred.list", "--out", str(tmp_path / "x")], ok=False)
    assert "ERROR: cannot open file : " in out


def test_step2_bgen_index_inflate_paths_and_bt_corrections(tmp_path, golden_dir):
    d = golden_dir
    shutil.copy(d + "/example_3chr.bgen", tmp_path / "noidx.bgen")
    qt = ["--step", "2", "--phenoFile", d + "/phenotype.txt", "--covarFile", d + "/covariates.txt", "--bsize", "64", "--ignore-pred",
          "--sample", d + "/example_3chr.sample"]
    la = run(qt + ["--bgen", d + "/example_3chr.bgen", "--out", str(tmp_path / "a")])
    lb = run(qt + ["--bgen", tmp_path / "noidx.bgen", "--out", str(tmp_path / "b")])
    lc = run(qt + ["--bgen", d + "/example_3chr.bgen", "--gpu-inflate", "--remove", d + "/fid_iid_to_remove.txt", "--out", str(tmp_path / "c")])
    run(qt + ["--bgen", d + "/example_3chr.bgen", "--remove", d + "/fid_iid_to_remove.txt", "--out", str(tmp_path / "c0")])
    assert "-index bgi file [" in la and "-index bgi file [" not in lb and "inflated on the GPU" in lc
    a = read(str(tmp_path / "a") + "_Y1.regenie")
    assert a.splitlines()[0].split()[6] == "INFO" and a == read(str(tmp_path / "b") + "_Y1.regenie")
    assert read(str(tmp_path / "c") + "_Y2.regenie") == read(str(tmp_path / "c0") + "_Y2.regenie")
    # binary traits: Step 1 --bt, then Step 2 with the Firth and the SPA fallbacks on .bgen and .bed
    fit = str(tmp_path / "fitb")
    log = run(["--step", "1", "--bed", d + "/example", "--phenoFile", d + "/phenotype_bin.txt", "--covarFile", d + "/covariates.txt",
               "--remove", d + "/fid_iid_to_remove.txt", "--bsize", "100", "--bt", "--lowmem", "--out", fit])
    assert "-logLik/N = " in log and "using LOOCV" in log
    bt = ["--step", "2", "--covarFile", d + "/covariates.txt", "--phenoFile", d + "/phenotype_bin.txt", "--remove",
          d + "/fid_iid_to_remove.txt", "--bsize", "200", "--bt", "--pThresh", "0.2", "--pred", fit + "_pred.list"]
    lf = run(bt + ["--bgen", d + "/example.bgen", "--firth", "--approx", "--out", str(tmp_path / "f")])
    ls = run(bt + ["--bed", d + "/example", "--spa", "--out", str(tmp_path / "s")])
    lg = run(bt + ["--bgen", d + "/example.bgen", "--firth", "--approx", "--gpu-inflate", "--out", str(tmp_path / "fg")])
    assert "Number of tests with Firth correction : " in lf and "Number of tests with SPA correction : " in ls
    f = read(str(tmp_path / "f") + "_Y1.regenie").splitlines()
    assert read(str(tmp_path / "fg") + "_Y1.regenie").splitlines() == f and "inflated on the GPU" in lg
    n_fail = sum(l.endswith(" TEST_FAIL") for l in f)
    assert 0 < n_fail < len(f) and all(l.split()[11:13] == ["NA", "NA"] for l in f if l.endswith(" TEST_FAIL"))
    assert int(lf.split("Number of tests with Firth correction : ")[1].split("(")[1].split()[0]) >= n_fail
    assert len(read(str(tmp_path / "s") + "_Y2.regenie").splitlines()) > 900


@pytest.mark.parametrize("extra", [(), ("--ref-first",)])
def test_dominant_and_recessive_tests_are_two_passes_over_recoded_genotypes(tmp_path, golden_dir, extra):
    import helpers
    helpers.check_recoded_test(run, read, tmp_path, golden_dir, extra)
    # dosages: the option is accepted, the TEST column changes, counts stay those of the additive coding
    d = golden_dir
    b = ["--step", "2", "--bgen", d + "/example.bgen", "--phenoFile", d + "/phenotype_bin.txt", "--covarFile", d + "/covariates.txt",
         "--bsize", "200", "--ignore-pred", "--bt", "--spa"] + list(extra)
    run(b + ["--out", str(tmp_path / "ba")])
    run(b + ["--test", "recessive", "--gpu-inflate", "--out", str(tmp_path / "br")])
    a = {l.split()[2]: l.split() for l in read(str(tmp_path / "ba") + "_Y1.regenie").splitlines()[1:]}
    r = [l.split() for l in read(str(tmp_path / "br") + "_Y1.regenie").splitlines()[1:]]
    assert len(r) > 500 and all(t[8] == "REC" and t[:8] == a[t[2]][:8] for t in r)
    assert any(t[9:] != a[t[2]][9:] for t in r)


def test_reference_script_case_column_mapping_from_bim(tmp_path, golden_dir):
    """The checks of the reference's test/test_bash.sh:225-259 (its covariate file with a binary column is not among the
    fixtures; V{1:2},V3 of covariates.txt stand in): sample lists only for the selected trait, first line `Y2<TAB>NA`,
    no chromosome-1 variants with --chrList 2,3, no ADD rows with --test dominant, and CHROM GENPOS ID ALLELE0 ALLELE1 =
    .bim columns 1,4,2,5,6 under --ref-first."""
    d = golden_dir
    out = str(tmp_path / "test_out")
    run(["--step", "2", "--bed", d + "/example_3chr", "--ref-first", "--covarFile", d + "/covariates.txt", "--covarColList",
         "V{1:2},V3", "--phenoFile", d + "/phenotype_bin.txt", "--phenoColList", "Y2", "--bsize", "100", "--test", "dominant",
         "--force-qt", "--ignore-pred", "--chrList", "2,3", "--write-samples", "--print-pheno", "--out", out])
    assert os.path.exists(out + "_Y2.regenie.ids") and not os.path.exists(out + "_Y1.regenie.ids")
    first = open(out + "_Y2.regenie.ids").readline().rstrip("\n").split("\t")
    assert first == ["Y2", "NA"]
    rows = read(out + "_Y2.regenie").splitlines()
    assert not any("mog_" in l for l in rows) and not any(" ADD " in l for l in rows) and all(" DOM " in l for l in rows[1:])
    bim2 = next(l.split() for l in open(d + "/example_3chr.bim") if l.startswith("2"))
    assert rows[1].split()[:5] == [bim2[0], bim2[3], bim2[1], bim2[4], bim2[5]]


@pytest.mark.parametrize("bt", [False, True])
def test_na_rows_are_equivalent_to_absent_rows(tmp_path, golden_dir, bt):
    import helpers
    helpers.check_na_invariance(run, read, tmp_path, golden_dir, bt)


@pytest.mark.parametrize("extra,bt", [((), False), (("--ref-first",), False), ((), True), (("--test", "dominant"), False)])
def test_no_split_output(tmp_path, golden_dir, extra, bt):
    import helpers
    helpers.check_no_split(run, read, tmp_path, golden_dir, extra, bt)


@pytest.mark.parametrize("extra", [(), ("--ref-first",)])
def test_htp_output(tmp_path, golden_dir, extra):
    import helpers
    helpers.check_htp(run, read, tmp_path, golden_dir, extra)


@pytest.mark.parametrize("bt", [False, True])
def test_htp_output_on_pgen_equals_bed(tmp_path, golden_dir, bt):
    """--htp needs the 2-bit rows on the host for the genotype counts: with .pgen input the records are decoded by the host
    reader (not on the device) and the rows must be those of the .bed twin of the reference's fixture pair."""
    d = golden_dir
    base = ["--step", "2", "--phenoFile", d + ("/phenotype_bin.txt" if bt else "/phenotype.txt"), "--covarFile", d + "/covariates.txt",
            "--bsize", "100", "--ignore-pred", "--htp", "C"] + (["--bt", "--firth", "--approx"] if bt else [])
    run(base + ["--bed", d + "/example", "--out", str(tmp_path / "b")])
    log = run(base + ["--pgen", d + "/example", "--out", str(tmp_path / "p")])
    assert "decoded on the GPU" not in log
    for nm in ("Y1", "Y2"):
        a, b = read(str(tmp_path / "b") + "_%s.regenie" % nm), read(str(tmp_path / "p") + "_%s.regenie" % nm)
        assert a == b and len(a.splitlines()) > 900
        assert sum(int(l.split("\t")[13]) for l in a.splitlines()[1:]) > 0


def test_htp_output_on_chromosome_x(tmp_path, golden_dir):
    import helpers
    helpers.check_htp_chrx(run, read, tmp_path)
    helpers.check_htp_bgen_chrx(run, read, tmp_path, golden_dir)


@pytest.mark.parametrize("bt", [False, True])
def test_htp_output_on_dosages(tmp_path, golden_dir, bt):
    import helpers
    helpers.check_htp_bgen(run, read, tmp_path, golden_dir, bt)


@pytest.mark.parametrize("extra", [(), ("--firth", "--approx", "--pThresh", "0.1"), ("--ref-first",)])
def test_htp_output_binary_traits(tmp_path, golden_dir, extra):
    """Control flow of --htp --bt against the mock ABI (its allele sums are real, its statistics are not regenie's): rows,
    model string, case / control genotype counts, Info keys."""
    import helpers
    helpers.check_htp_bt(run, read, tmp_path, golden_dir, extra, numbers=False)


def test_min_case_count_drops_rare_binary_traits(tmp_path, golden_dir):
    """rm_phenoCols (src/Pheno.cpp:527-570): binary traits with fewer than --minCaseCount (10) cases are ignored."""
    d = golden_dir
    rows = open(d + "/phenotype_bin.txt").read().splitlines()
    out = [rows[0] + " Y3"]
    for k, l in enumerate(rows[1:]):
        out.append(l + (" 1" if k < 5 else " 0"))
    (tmp_path / "ph.txt").write_text("\n".join(out) + "\n")
    base = ["--step", "2", "--bed", d + "/example_3chr", "--phenoFile", tmp_path / "ph.txt", "--covarFile", d + "/covariates.txt",
            "--bsize", "200", "--bt", "--ignore-pred"]
    log = run(base + ["--out", str(tmp_path / "a")])
    assert "Phenotype 'Y3' has too few cases so it will be ignored." in log and "+ n_pheno = 2" in log
    assert os.path.exists(str(tmp_path / "a") + "_Y2.regenie") and not os.path.exists(str(tmp_path / "a") + "_Y3.regenie")
    run(base + ["--minCaseCount", "3", "--out", str(tmp_path / "b")])
    assert os.path.exists(str(tmp_path / "b") + "_Y3.regenie")
    r = run(base + ["--phenoCol", "Y3", "--out", str(tmp_path / "c")], ok=False)
    assert "ERROR: all phenotypes have less than 10 cases." in r


def test_min_info_drops_whole_variants_on_the_all_sample_info(tmp_path, golden_dir):
    """--minINFO: a variant whose INFO over all analysed samples is below the threshold is ignored altogether
    (src/Geno.cpp:2074), on top of the per-trait rule; the expected set comes from the oracle's formula."""
    import numpy as np
    import helpers
    from oracle import bgen as obgen
    d = golden_dir
    keys = ["_".join(l.split()[:2]) for l in open(d + "/example.fam")]
    M, N = 80, len(keys)
    probs, miss = helpers.synthetic_dosage_probs(M, N, seed=9)
    f = str(tmp_path / "syn.bgen")
    helpers.write_bgen(f, probs, miss, [1] * 40 + [2] * 40, range(1, M + 1), ["v%d" % v for v in range(M)], sample_ids=keys)
    info1 = []
    for v in range(M):
        g, ival = obgen.dosage(probs[v, :, 0], probs[v, :, 1], miss[v])
        ok = ~miss[v]
        af = g[ok].sum() / (2 * ok.sum())
        info1.append(1 - ival[ok].sum() / (2 * ok.sum() * af * (1 - af)))
    base = ["--step", "2", "--bgen", f, "--phenoFile", d + "/phenotype.txt", "--covarFile", d + "/covariates.txt", "--bsize", "32",
            "--ignore-pred", "--minMAC", "1"]
    run(base + ["--out", str(tmp_path / "all")])
    log = run(base + ["--minINFO", "0.5", "--gpu-inflate", "--out", str(tmp_path / "thr")])
    assert "inflating on the host" in log
    ids_all = [l.split()[2] for l in read(str(tmp_path / "all") + "_Y1.regenie").splitlines()[1:]]
    ids_thr = [l.split()[2] for l in read(str(tmp_path / "thr") + "_Y1.regenie").splitlines()[1:]]
    want = [i for i in ids_all if info1[int(i[1:])] >= 0.5]
    assert ids_thr == want and 0 < len(want) < len(ids_all)


@pytest.mark.parametrize("bt", [False, True])
def test_dominant_recessive_on_dosages(tmp_path, golden_dir, bt):
    import helpers
    helpers.check_recoded_test_bgen(run, read, tmp_path, golden_dir, bt)


@pytest.mark.parametrize("extra", [(), ("--ref-first", "--firth", "--approx", "--pThresh", "0.2")])
def test_af_cc_columns(tmp_path, golden_dir, extra):
    import helpers
    helpers.check_af_cc(run, read, tmp_path, golden_dir, extra)
    # the option is switched off, with the reference's warning, where it does not apply
    d = golden_dir
    log = run(["--step", "2", "--bed", d + "/example_3chr", "--phenoFile", d + "/phenotype.txt", "--covarFile", d + "/covariates.txt",
               "--bsize", "100", "--ignore-pred", "--af-cc", "--out", str(tmp_path / "qt")])
    assert "WARNING: disabling option --af-cc" in log
    assert read(str(tmp_path / "qt") + "_Y1.regenie").splitlines()[0].split()[6] == "N"


def test_no_split_output_on_dosages(tmp_path, golden_dir):
    import helpers
    helpers.check_no_split_bgen(run, read, tmp_path, golden_dir)


GENO = {"bed": lambda d: ["--bed", d + "/example_3chr"], "pgen": lambda d: ["--pgen", d + "/example"],
        "bgen": lambda d: ["--bgen", d + "/example_3chr.bgen", "--sample", d + "/example_3chr.sample"]}


@pytest.mark.parametrize("geno,extra", [(g, t + c) for g in GENO for t in ([], ["--bt"]) for c in ([], ["--loocv"])] +
                         [("bed", ["--print-prs", "--lowmem", "--keep-l0"])])
def test_step1_gpus_n_writes_the_single_gpu_files(tmp_path, golden_dir, monkeypatch, geno, extra):
    """--gpus N: each device feeds its range of level-0 blocks and fits the phenotypes it owns.  The mock stores every
    slab in the W of the phenotype's owner like the library's peer stores, so the files must be those of one device
    (on GPUs: tests/test_multigpu_gpu.py)."""
    d = golden_dir
    monkeypatch.setenv("RG_MOCK_DEVICES", "3")
    pheno = d + ("/phenotype_bin.txt" if "--bt" in extra else "/phenotype.txt")
    files = {}
    for g in (1, 2, 3):
        o = str(tmp_path / ("g%d" % g))
        log = run(["--step", "1"] + GENO[geno](d) + ["--phenoFile", pheno, "--covarFile", d + "/covariates.txt", "--bsize", "100",
                                                      "--gpus", g] + extra + ["--out", o])
        assert ("(gpu 2)" in log) == (g == 3)
        out = sorted(f for f in glob.glob(o + "_*") if not f.endswith(".list"))
        files[g] = {os.path.basename(f)[2:]: open(f, "rb").read() for f in out}
        files[g]["pred.list"] = [l.split()[0] for l in open(o + "_pred.list")]
    assert len(files[1]) == (7 if "--print-prs" in extra else 3)         # .loco (+ .prs, _l0_Y) per phenotype, pred.list
    assert files[2] == files[1] and files[3] == files[1]


def sexed_copies(t, d):
    """The fixtures carry no sex information: copies of the .bed, .pgen and .bgen filesets with alternating sexes (male
    first), each with the genotype arguments that select it and a --keep file of its males."""
    fam = [l.split() for l in open(d + "/example_3chr.fam")]
    for ext in (".bed", ".bim"):
        shutil.copy(d + "/example_3chr" + ext, t / ("sx" + ext))
    with open(t / "sx.fam", "w") as fh:
        fh.write("".join(" ".join(r[:4] + ["1" if k % 2 == 0 else "2"] + r[5:]) + "\n" for k, r in enumerate(fam)))
    for ext in (".pgen", ".pvar"):
        shutil.copy(d + "/example" + ext, t / ("sxp" + ext))
    psam = [l.split() for l in open(d + "/example.psam")]
    with open(t / "sxp.psam", "w") as fh:
        fh.write("\t".join(psam[0]) + "\n" + "".join("\t".join([r[0], r[1], "1" if k % 2 == 0 else "2"] + r[3:]) + "\n"
                                                  for k, r in enumerate(psam[1:])))
    shutil.copy(d + "/example_3chr.bgen", t / "sxg.bgen")
    sample = [l.split() for l in open(d + "/example_3chr.sample")]
    with open(t / "sxg.sample", "w") as fh:
        fh.write("".join(" ".join(r) + "\n" for r in sample[:2]) +
                 "".join(" ".join(r[:3] + ["1" if k % 2 == 0 else "2"] + r[4:]) + "\n" for k, r in enumerate(sample[2:])))
    out = {}
    for fmt, args, ids in (("bed", ["--bed", t / "sx"], fam), ("pgen", ["--pgen", t / "sxp"], psam[1:]),
                           ("bgen", ["--bgen", t / "sxg.bgen", "--sample", t / "sxg.sample"], sample[2:])):
        keep = t / ("males_%s.txt" % fmt)
        keep.write_text("".join("%s %s\n" % (r[0], r[1]) for r in ids[::2]))
        out[fmt] = (args, keep)
    return out


def test_sex_specific_and_starting_block(tmp_path, golden_dir):
    """--sex-specific keeps one sex like --keep would (src/Geno.cpp:1286-1293), in both steps and on every genotype format;
    --starting-block resumes a Step-2 run at a block (src/Data.cpp:2168, :2275): its rows are the tail of the full run."""
    d = golden_dir
    covs = ["--phenoFile", d + "/phenotype.txt", "--covarFile", d + "/covariates.txt", "--bsize", "100"]
    for fmt, (geno, males) in sexed_copies(tmp_path, d).items():
        s1 = ["--step", "1"] + geno + covs
        log = run(s1 + ["--sex-specific", "male", "--out", str(tmp_path / ("s1m_" + fmt))])
        run(s1 + ["--keep", males, "--out", str(tmp_path / ("s1k_" + fmt))])
        assert "-keeping only male individuals in the analysis" in log, fmt
        loco = read(str(tmp_path / ("s1m_" + fmt)) + "_1.loco")
        assert loco == read(str(tmp_path / ("s1k_" + fmt)) + "_1.loco") and len(loco.splitlines()[0].split()) == 251, fmt
        log = run(["--step", "2"] + geno + covs + ["--ignore-pred", "--sex-specific", "male", "--out", str(tmp_path / ("s2m_" + fmt))])
        assert "-keeping only male individuals in the analysis" in log, fmt
        rows = [l.split() for l in read(str(tmp_path / ("s2m_" + fmt)) + "_Y1.regenie").splitlines()]
        assert {r[rows[0].index("N")] for r in rows[1:]} == {"250"}, fmt
    base = ["--step", "2", "--bed", tmp_path / "sx"] + covs + ["--ignore-pred"]
    run(base + ["--sex-specific", "male", "--out", str(tmp_path / "m1")])
    run(base + ["--keep", tmp_path / "males_bed.txt", "--out", str(tmp_path / "m2")])
    m1 = read(str(tmp_path / "m1") + "_Y1.regenie")
    assert m1 == read(str(tmp_path / "m2") + "_Y1.regenie") and {l.split()[6] for l in m1.splitlines()[1:]} == {"250"}
    run(base + ["--out", str(tmp_path / "full")])
    log = run(base + ["--starting-block", "4", "--out", str(tmp_path / "tail")])
    assert "+ skipping to block #4" in log
    full, tail = read(str(tmp_path / "full") + "_Y2.regenie").splitlines(), read(str(tmp_path / "tail") + "_Y2.regenie").splitlines()
    assert tail[0] == full[0] and 0 < len(tail) < len(full) and full[-(len(tail) - 1):] == tail[1:]
    assert tail[1].split()[2] == open(d + "/example_3chr.bim").read().splitlines()[250].split()[1]        # blocks: 50 + 100 + 100 + ...
    r = run(base + ["--starting-block", "99", "--out", str(tmp_path / "x")], ok=False)
    assert "ERROR: Starting block > number of blocks analyzed" in r


def test_write_and_use_null_firth(tmp_path, golden_dir):
    """--write-null-firth (Step 1, src/Data.cpp:1873-1903) / --use-null-firth (Step 2, src/Step2_Models.cpp:1896-1980): file
    layout, and the written coefficients are a stationary point of the oracle's null Firth fit with the same LOCO offsets
    (the covariate basis comes from the driver's own prep through the host probe; the LOCO numbers are the mock's)."""
    import numpy as np
    from oracle import step2_bt
    from test_host_cpu import probe, read_dump
    d = golden_dir
    fit = str(tmp_path / "fit")
    args = ["--bed", d + "/example", "--phenoFile", d + "/phenotype_bin.txt", "--covarFile", d + "/covariates.txt", "--remove",
            d + "/fid_iid_to_remove.txt"]
    log = run(["--step", "1"] + args + ["--bsize", "100", "--bt", "--write-null-firth", "--out", fit])
    assert "List of files with null Firth estimates written to" in log
    lst = [l.split() for l in open(fit + "_firth.list")]
    assert [t[0] for t in lst] == ["Y1", "Y2"] and all(os.path.isabs(t[1]) for t in lst)
    probe("prep", tmp_path / "d.bin", *args, "--bt")
    dump = read_dump(tmp_path / "d.bin")
    N, P, C = dump["hdr"]["N"], dump["hdr"]["P"], dump["hdr"]["C"]
    X = dump["X"].reshape(C, N).T
    keys = ["_".join(l.split()[:2]) for l in open(d + "/example.fam")]
    rm = {"_".join(l.split()[:2]) for l in open(d + "/fid_iid_to_remove.txt") if l.strip()}
    keys = [k for k in keys if k not in rm]
    pos = {k: i for i, k in enumerate(keys)}
    for j in range(P):
        rows = [l.split() for l in open(fit + "_%d.firth" % (j + 1))]
        assert [t[0] for t in rows] == [str(c) for c in range(1, 24)] and all(len(t) == 1 + C for t in rows)
        loco = [l.split() for l in open(fit + "_%d.loco" % (j + 1))]
        mask = dump["mask"].reshape(P, N)[j].astype(bool)
        y = dump["Y_raw"].reshape(P, N)[j]
        for c in (0, 1, 22):
            blup = np.zeros(N)
            for k, v in zip(loco[0][1:], loco[1 + c][1:]):
                blup[pos[k]] = 0.0 if v == "NA" else float(v)
            beta = np.array([float(x) for x in rows[c][1:]])
            ok, b2 = step2_bt.firth_nr(y, X, blup * mask, mask, beta.copy(), 25, 1000, 5e-5)
            assert ok and np.abs(b2 - beta).max() < 1e-4 * max(1.0, np.abs(beta).max()), (j, c, beta, b2)
    # Step 2 reads them as starting values
    s2 = ["--step", "2"] + args + ["--bsize", "200", "--bt", "--firth", "--approx", "--pred", fit + "_pred.list"]
    run(s2 + ["--out", str(tmp_path / "a")])
    log = run(s2 + ["--use-null-firth", fit + "_firth.list", "--out", str(tmp_path / "b")])
    assert " * reading null Firth estimates using file : [" in log
    assert read(str(tmp_path / "a") + "_Y1.regenie") == read(str(tmp_path / "b") + "_Y1.regenie")
    r = run(s2 + ["--use-null-firth", str(tmp_path / "nope.list"), "--out", str(tmp_path / "c")], ok=False)
    assert "ERROR: cannot open file : " in r
