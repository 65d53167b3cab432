"""Conditional analysis (--condition-list / --condition-file / --max-condition-vars) through the driver linked against
the mock ABI (tests/mock/mock_abi.cpp; see tests/test_driver_plumbing_cpu.py): a conditioned run gives the outputs of the
unconditioned run whose covariate file carries the conditioning genotypes, and the option checks fail with the
reference's messages."""
import glob
import os
import re
import subprocess

import pytest

import condition_oracle as co

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
    return open(path).read()


@pytest.mark.parametrize("source", [None, "bed", "pgen", "bgen"])
@pytest.mark.parametrize("bt", [False, True])
@pytest.mark.parametrize("main", ["bed", "pgen", "bgen"])
def test_conditioned_step2_equals_covariate_run(tmp_path, golden_dir, main, bt, source):
    co.check_equivalence(run, read, tmp_path, golden_dir, main, bt, source)


@pytest.mark.parametrize("bt", [False, True])
def test_conditioned_step1_and_step2_equal_covariate_runs(tmp_path, golden_dir, bt):
    co.check_equivalence(run, read, tmp_path, golden_dir, "bed", bt, None, step1=True)
    co.check_equivalence(run, read, tmp_path / "ext", golden_dir, "bed", bt, "pgen", step1=True)


def test_conditioning_variant_with_missing_calls_in_the_main_file(tmp_path, golden_dir):
    """A same-file conditioning variant whose missing calls are replaced by the mean (read_snp, src/Geno.cpp:3978-3996):
    a copy of example.bed with calls of the listed variants set to missing."""
    import numpy as np
    import shutil
    from oracle import plink
    from regenie_b200 import synth
    d = golden_dir
    keys, _ = plink.read_fam(d + "/example.fam")
    bim = plink.read_bim(d + "/example.bim")
    G = plink.decode_bed(plink.read_bed_rows(d + "/example.bed", len(keys), bim.offset), len(keys))
    g = np.where(G == -3, 3, G).astype(np.int64)
    rng = np.random.default_rng(1)
    for v in (24, 511):                                      # IDs "25", "512"
        g[v, rng.random(len(keys)) < 0.1] = 3
    src = tmp_path / "gm"
    src.mkdir()
    with open(src / "example.bed", "wb") as fh:
        fh.write(b"\x6c\x1b\x01" + synth.pack_bed(g).tobytes())
    for ext in ("bim", "fam"):
        shutil.copy(d + "/example." + ext, str(src / ("example." + ext)))
    for f in ("covariates.txt", "phenotype.txt", "phenotype_bin.txt"):
        shutil.copy(d + "/" + f, str(src / f))
    _, calls, _ = co.source_calls("bed", str(src / "example"), ["25", "512"])
    assert all((~c).sum() > 20 for _n, c in calls.values())
    co.check_equivalence(run, read, tmp_path / "t", str(src), "bed", False, None, step1=True, ids=("25", "512"))


def _base(d, tmp_path, step=2):
    return ["--step", str(step), "--bed", d + "/example", "--phenoFile", d + "/phenotype.txt", "--covarFile", d + "/covariates.txt",
            "--bsize", "100", "--out", str(tmp_path / "o")] + (["--ignore-pred"] if step == 2 else [])


def _fails(args, msg):
    out = run(args, ok=False)
    assert "ERROR: " in out and msg in out, (args, out[-1500:])


def test_condition_option_errors(tmp_path, golden_dir):
    d = golden_dir
    lst = tmp_path / "l.txt"
    lst.write_text("25\n512\n990\n")
    empty = tmp_path / "e.txt"
    empty.write_text("")
    missing = tmp_path / "m.txt"
    missing.write_text("25\nnot_there\nnor_this\n")
    none = tmp_path / "n.txt"
    none.write_text("not_there\n")
    base = _base(d, tmp_path)
    _fails(base + ["--condition-list", str(empty)], "no variants for conditional analysis given in file " + str(empty))
    _fails(base + ["--condition-list", str(lst), "--max-condition-vars", "2"],
           "number of variants used for conditional analysis is greater than maximum of 2 (otherwise use --max-condition-vars)")
    _fails(base + ["--condition-list", str(lst), "--condition-file", "bed"], "invalid option input for --condition-file")
    _fails(base + ["--condition-list", str(lst), "--condition-file", "vcf,x"], "invalid file format for --condition-file (either bed/bge/pgen)")
    _fails(base + ["--condition-file", "bed," + d + "/example"], "must use --condition-list if using --condition-file.")
    _fails(base + ["--condition-list", str(missing)], "2 of the variants could not be found in the genotype file")
    _fails(base + ["--condition-list", str(none)], "none of the variants were found in the genotype file")
    _fails(base + ["--condition-list", str(none), "--condition-file", "bed," + d + "/example_3chr"],
           "none of the conditional variants were found in the genotype file")
    _fails(base + ["--condition-list", str(missing), "--condition-file", "pgen," + d + "/example"],
           "2 of the variants could not be found in the genotype file")
    # the lookup runs on the variants of the --chr / --range selection, before --extract / --exclude
    _fails(base + ["--condition-list", str(lst), "--chr", "1", "--range", "1:1-100"], "2 of the variants could not be found in the genotype file")
    run(base + ["--condition-list", str(lst), "--exclude", str(lst)])
    # an external file without any analysed sample
    other = tmp_path / "other"
    path, ids = co.write_external(str(other), "bed", ["x%d_x%d" % (k, k) for k in range(40)])
    (tmp_path / "x.txt").write_text(ids[0] + "\n")
    _fails(base + ["--condition-list", str(tmp_path / "x.txt"), "--condition-file", "bed," + path],
           "none of the analyzed samples are present in the file")
    out = run(["--help"])
    assert "--condition-list" in out and "--condition-file" in out and "--max-condition-vars" in out


def test_covariate_limit_is_checked_before_any_gpu_work(tmp_path, golden_dir):
    """Intercept + 3 covariates + K conditioning variants above the 64 columns the kernels take stop on the host with both
    counts and the limit in the message; exactly 64 columns run."""
    d = golden_dir
    for K, ok in ((60, True), (61, False)):
        lst = tmp_path / ("l%d.txt" % K)
        lst.write_text("\n".join(str(10 + 7 * k) for k in range(K)) + "\n")
        for step in (1, 2):
            args = _base(d, tmp_path, step) + ["--condition-list", str(lst)]
            if ok:
                out = run(args)
                assert "n_used = %d" % K in out
            else:
                _fails(args, "too many covariates for conditional analysis: 4 covariate columns (with the intercept) and 61 "
                             "conditioning variants make 65, more than the maximum of 64 columns")


def test_host_limit_matches_the_kernels():
    src = open(os.path.join(ROOT, "regenie_b200", "csrc", "kernels.cuh")).read()
    hdr = open(os.path.join(ROOT, "regenie_b200", "host", "condition.hpp")).read()
    assert re.search(r"kMaxCov = (\d+);", src).group(1) == re.search(r"kMaxCovColumns = (\d+);", hdr).group(1)


def test_extract_with_condition_list_keeps_variants_in_both(tmp_path, golden_dir):
    """--extract together with the list: the reference's warning, and the listed IDs are not tested even when extracted."""
    d = golden_dir
    lst = tmp_path / "l.txt"
    lst.write_text("25\n512\n")
    ext = tmp_path / "x.txt"
    ext.write_text("\n".join(str(k) for k in range(1, 600)) + "\n")
    out = run(_base(d, tmp_path) + ["--condition-list", str(lst), "--extract", str(ext)])
    assert "WARNING: only variants which satisfy both extract/exclude options will be kept." in out
    ids = {l.split()[2] for l in read(str(tmp_path / "o") + "_Y1.regenie").splitlines()[1:]}
    assert ids and ids <= {str(k) for k in range(1, 600)} and not ids & {"25", "512"}


def test_conditioning_changes_the_statistics(tmp_path, golden_dir):
    """The conditioning columns reach the statistics: the run differs from one that only excludes the listed variants."""
    d = golden_dir
    lst = tmp_path / "l.txt"
    lst.write_text("25\n512\n990\n")
    run(_base(d, tmp_path) + ["--condition-list", str(lst)])
    a = read(str(tmp_path / "o") + "_Y1.regenie")
    b_args = _base(d, tmp_path)
    b_args[b_args.index("--out") + 1] = str(tmp_path / "x")
    run(b_args + ["--exclude", str(lst)])
    b = read(str(tmp_path / "x") + "_Y1.regenie")
    assert [l.split()[2] for l in a.splitlines()] == [l.split()[2] for l in b.splitlines()] and a != b


def test_level0_jobs_condition_on_the_same_variants(tmp_path, golden_dir):
    """--split-l0 / --run-l0 / --run-l1 with the list give the .loco files of the single conditioned run."""
    d = golden_dir
    ids = [open(d + "/example_3chr.bim").read().splitlines()[k].split()[1] for k in (10, 300)]
    lst = tmp_path / "l.txt"
    lst.write_text("\n".join(ids) + "\n")
    base = ["--step", "1", "--bed", d + "/example_3chr", "--phenoFile", d + "/phenotype.txt", "--covarFile", d + "/covariates.txt",
            "--bsize", "100", "--condition-list", str(lst)]
    run(base + ["--out", str(tmp_path / "one")])
    par = str(tmp_path / "par")
    run(base + ["--split-l0", par + ",3", "--out", str(tmp_path / "l0")])
    snps = set(open(par + "_job1.snplist").read().split() + open(par + "_job3.snplist").read().split())
    assert snps and not snps & set(ids)
    for job in (1, 2, 3):
        out = run(base + ["--run-l0", par + ".master,%d" % job, "--out", str(tmp_path / "l0")])
        assert "n_used = 2" in out
    run(base + ["--run-l1", par + ".master", "--out", str(tmp_path / "l1")])
    for k in (1, 2):
        assert read(str(tmp_path / "l1") + "_%d.loco" % k) == read(str(tmp_path / "one") + "_%d.loco" % k)
