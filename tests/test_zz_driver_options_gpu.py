"""Driver options added after the last run of the GPU suite on hardware in round 1 (--range, --setl0/--setl1 and friends,
--test dominant|recessive, --no-split, the check_na.sh invariance, the ring-buffer inflate kernel).  Every one of them
passes against the mock ABI on the CPU (tests/test_driver_plumbing_cpu.py, same helper functions); they sit in their
own file, collected after the others, so that a first failure on hardware cannot hide the results of the verified suite."""
import os
import subprocess

import pytest

import helpers

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RGB = os.path.join(ROOT, "regenie_b200", "rgb200")


def run(args):
    r = subprocess.run([RGB] + args, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


def test_step2_range_is_a_window_of_the_full_run(tmp_path, golden_dir):
    """--range CHR:MIN-MAX (src/Regenie.cpp:741-755, in_range src/Geno.cpp:2790-2800) on .bed and .bgen input."""
    d = golden_dir
    for kind, geno in (("bed", ["--bed", d + "/example_3chr"]),
                       ("bgen", ["--bgen", d + "/example_3chr.bgen", "--sample", d + "/example_3chr.sample"])):
        common = ["--step", "2"] + geno + ["--phenoFile", d + "/phenotype.txt", "--covarFile", d + "/covariates.txt",
                                           "--bsize", "100", "--ignore-pred"]
        run(common + ["--out", str(tmp_path / (kind + "_all"))])
        full = open(str(tmp_path / (kind + "_all")) + "_Y1.regenie").read().splitlines()
        pos = sorted(int(l.split()[1]) for l in full[1:] if l.startswith("2 "))
        lo, hi = pos[len(pos) // 4], pos[3 * len(pos) // 4]
        run(common + ["--range", "2:%d-%d" % (hi, lo), "--out", str(tmp_path / (kind + "_win"))])      # min / max in any order
        win = open(str(tmp_path / (kind + "_win")) + "_Y1.regenie").read().splitlines()
        want = [l for l in full[1:] if l.startswith("2 ") and lo <= int(l.split()[1]) <= hi]
        assert win[0] == full[0] and win[1:] == want and len(want) > 50


def test_user_ridge_grids_exclude_lists_aliases_and_l1_subset(tmp_path, golden_dir):
    """--setl0/--setl1 with the default grid values, --phenoExcludeList/--covarExcludeList against the positive
    column lists, the short option names, and --l1-phenoList after --split-l0/--run-l0 (src/Regenie.cpp:845-868)."""
    d = golden_dir
    pheno, covar = d + "/phenotype.txt", d + "/covariates.txt"
    base = ["--step", "1", "--bed", d + "/example_3chr", "--phenoFile", pheno, "--covarFile", covar, "--bsize", "100"]
    run(base + ["--out", str(tmp_path / "a")])
    run(["--step", "1", "--bed", d + "/example_3chr", "-p", pheno, "-c", covar, "-b", "100", "--setl0", "0.99,0.01,0.25,0.5,0.75",
         "--setl1", "0.01,0.25,0.5,0.75,0.99,0.5", "-o", str(tmp_path / "b")])
    for k in (1, 2):
        assert open(str(tmp_path / "a") + "_%d.loco" % k).read() == open(str(tmp_path / "b") + "_%d.loco" % k).read()
    # a different grid changes the fit
    log = run(base + ["--setl1", "0.1,0.9", "--out", str(tmp_path / "c")])
    assert log.count("Rsq = ") == 4
    # exclusion lists == positive lists
    hdr = open(covar).readline().split()[2:]
    run(base + ["--phenoCol", "Y2", "--covarColList", ",".join(hdr[:2]), "--out", str(tmp_path / "d")])
    run(base + ["--phenoExcludeList", "Y1", "--covarExcludeList", ",".join(hdr[2:]), "--out", str(tmp_path / "e")])
    assert open(str(tmp_path / "d") + "_1.loco").read() == open(str(tmp_path / "e") + "_1.loco").read()
    assert [l.split()[0] for l in open(str(tmp_path / "e") + "_pred.list")] == ["Y2"]
    # level 1 for a subset of the phenotypes
    par = str(tmp_path / "par")
    run(base + ["--split-l0", par + ",2", "--out", str(tmp_path / "l0")])
    for job in (1, 2):
        run(base + ["--run-l0", par + ".master,%d" % job, "--out", str(tmp_path / "l0")])
    run(base + ["--run-l1", par + ".master", "--l1-phenoList", "Y2", "--keep-l0", "--out", str(tmp_path / "l1")])
    assert open(str(tmp_path / "l1") + "_2.loco").read() == open(str(tmp_path / "a") + "_2.loco").read()
    assert not os.path.exists(str(tmp_path / "l1") + "_1.loco")
    assert [l.split()[0] for l in open(str(tmp_path / "l1") + "_pred.list")] == ["Y2"]


@pytest.mark.parametrize("extra", [(), ("--ref-first",)])
def test_dominant_recessive_equal_additive_on_recoded_genotypes(tmp_path, golden_dir, extra):
    """--test dominant / recessive (src/Geno.cpp:2509-2530): A1FREQ / N / MAC filter from the additive coding, the test on
    the recoded genotypes == an additive run on a fileset recoded the same way."""
    def read(path):
        return open(path).read()
    helpers.check_recoded_test(run, read, tmp_path, golden_dir, extra)


@pytest.mark.parametrize("bt", [False, True])
def test_na_rows_are_equivalent_to_absent_rows(tmp_path, golden_dir, bt):
    """test/check_na.sh of the reference, for quantitative and binary (Firth) runs, on the real library."""
    def read(path):
        return open(path).read()
    helpers.check_na_invariance(run, read, tmp_path, golden_dir, bt)


@pytest.mark.parametrize("extra,bt", [((), False), (("--ref-first",), True)])
def test_no_split_output(tmp_path, golden_dir, extra, bt):
    """--no-split on the real library: per-trait columns == the split files, N_RR / N_RA / N_AA == the .bed counts."""
    def read(path):
        return open(path).read()
    helpers.check_no_split(run, read, tmp_path, golden_dir, extra, bt)


@pytest.mark.xfail(strict=False, reason="the ring-buffer inflate kernel (RG_B200_INFLATE=window) is verified against zlib on the CPU "
                                        "but was written after the round's GPU budget was spent: first run on hardware")
def test_gpu_inflate_window_variant_equals_host_inflate(tmp_path, golden_dir, monkeypatch):
    d = golden_dir
    qt = ["--step", "2", "--bgen", d + "/example_3chr.bgen", "--sample", d + "/example_3chr.sample", "--phenoFile",
          d + "/phenotype.txt", "--covarFile", d + "/covariates.txt", "--bsize", "77", "--ignore-pred"]
    run(qt + ["--out", str(tmp_path / "host")])
    monkeypatch.setenv("RG_B200_INFLATE", "window")
    log = run(qt + ["--out", str(tmp_path / "dev"), "--gpu-inflate"])
    assert "inflated on the GPU" in log
    for nm in ("Y1", "Y2"):
        assert open(str(tmp_path / "host") + "_%s.regenie" % nm).read() == open(str(tmp_path / "dev") + "_%s.regenie" % nm).read()


@pytest.mark.parametrize("bt", [False, True])
def test_dominant_recessive_on_dosages(tmp_path, golden_dir, bt):
    """--test dominant / recessive on a synthetic .bgen with real imputation uncertainty (real library)."""
    def read(path):
        return open(path).read()
    helpers.check_recoded_test_bgen(run, read, tmp_path, golden_dir, bt)


@pytest.mark.parametrize("extra", [(), ("--ref-first", "--firth", "--approx", "--pThresh", "0.2")])
def test_af_cc_columns(tmp_path, golden_dir, extra):
    """--af-cc on the real library: a second Step-2 handle masked to the cases of each trait."""
    def read(path):
        return open(path).read()
    helpers.check_af_cc(run, read, tmp_path, golden_dir, extra)


def test_htp_output(tmp_path, golden_dir):
    """--htp on the real library: variants, AAF and N of the native file; genotype counts == the .bed counts per trait."""
    def read(path):
        return open(path).read()
    helpers.check_htp(run, read, tmp_path, golden_dir, ())


@pytest.mark.xfail(strict=False, reason="--htp for binary traits was written after the GPU budget of round 2 was spent: green "
                   "against the mock ABI (tests/test_driver_plumbing_cpu.py, same helper), the row formatter is checked "
                   "against the oracle restatement on its binary-trait branches; not yet run on hardware")
@pytest.mark.parametrize("extra", [("--firth", "--approx", "--pThresh", "0.1")])
def test_htp_output_binary_traits(tmp_path, golden_dir, extra):
    """--htp --bt on the real library: case / control genotype counts == the .bed counts, Effect / CI / Pval / Info against
    the native file of the same run options."""
    def read(path):
        return open(path).read()
    helpers.check_htp_bt(run, read, tmp_path, golden_dir, extra, numbers=True)


def test_htp_output_on_chromosome_x(tmp_path, golden_dir):
    def read(path):
        return open(path).read()
    helpers.check_htp_chrx(run, read, tmp_path)
    helpers.check_htp_bgen_chrx(run, read, tmp_path, golden_dir)


@pytest.mark.xfail(strict=False, reason="--htp on dosages was written after the GPU budget of round 2 was spent: the counts are "
                   "formed on the host and are green against the oracle on the mock ABI; not yet run on hardware")
@pytest.mark.parametrize("bt", [False, True])
def test_htp_output_on_dosages(tmp_path, golden_dir, bt):
    def read(path):
        return open(path).read()
    helpers.check_htp_bgen(run, read, tmp_path, golden_dir, bt)


def test_no_split_output_on_dosages(tmp_path, golden_dir):
    def read(path):
        return open(path).read()
    helpers.check_no_split_bgen(run, read, tmp_path, golden_dir)
