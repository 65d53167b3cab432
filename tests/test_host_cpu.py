"""Host-side logic of the rgb200 driver against the oracle, without a GPU.

`regenie_b200/rgb200_hostprobe` links the driver's own translation units (readers, phenotype preparation, null models,
text formats; everything under regenie_b200/host/ except main.cpp) and dumps what they produce; these tests compare the
dumps with the numpy restatement in oracle/ and with the reference's fixtures:
  * .bgi index (SQLite) vs sequential scan of the .bgen, and vs oracle/bgen.py        (read_bgi_file src/Geno.cpp:180-309)
  * inflated BGEN probability bytes vs oracle/bgen.py
  * the C++ .pgen decoder vs the .bed rows of the reference's own fixture pair
  * read_pheno_and_cov + prep_run vs oracle/prep.py (QT / BT, step 1 / step 2, --remove, gz inputs, RINT)
  * the covariate-only logistic offsets vs oracle/step1_bt.py
  * .loco / .prs writers and readers, plain and --gz                                  (src/Data.cpp:1795-1982)
  * .regenie rows + LOG10P vs scipy                                                   (src/Step2_Models.cpp:2502-2540)
  * .regenie.ids                                                                      (src/Pheno.cpp:1538-1576)
  * --no-split / --htp genotype counts vs oracle/plink.py and oracle/bgen.py           (update_genocounts src/Geno.cpp:2986-3018)
"""
import gzip
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import bgen as obgen
from oracle import plink, prep, step1_bt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE = os.path.join(ROOT, "regenie_b200", "rgb200_hostprobe")


@pytest.fixture(scope="module", autouse=True)
def _built():
    if not os.path.exists(PROBE):
        from regenie_b200 import build
        build.build_probe()
    assert os.path.exists(PROBE)


def probe(*args, stdin=None, ok=True):
    r = subprocess.run([PROBE] + [str(a) for a in args], capture_output=True, text=True, input=stdin, timeout=120)
    if ok:
        assert r.returncode == 0, r.stdout[-500:] + r.stderr[-500:]
    return r


def read_dump(path):
    out = {}
    with open(path, "rb") as f:
        hdr = f.readline().split()
        out["hdr"] = {hdr[i].decode(): int(hdr[i + 1]) for i in range(0, len(hdr), 2)}
        out["names"] = [t.decode() for t in f.readline().split()[1:]]
        while True:
            line = f.readline()
            if not line:
                break
            name, dt, n = line.split()
            dt = np.dtype(dt.decode())
            out[name.decode()] = np.frombuffer(f.read(int(n) * dt.itemsize), dtype=dt).copy()
            f.readline()
    return out


# ------------------------------------------------------------------------------------------- BGEN + .bgi
@pytest.mark.parametrize("name", ["example", "example_3chr"])
def test_bgi_index_equals_scan_and_oracle(golden_dir, name):
    f = "%s/%s.bgen" % (golden_dir, name)
    a = probe("bgen-variants", f).stdout.splitlines()
    b = probe("bgen-variants", f, "--no-bgi").stdout.splitlines()
    assert a[0].startswith("used_bgi 1") and b[0].startswith("used_bgi 0")
    assert a[1:] == b[1:] and len(a) > 100
    ob = list(obgen.Bgen(f).variants())
    got = [l.split() for l in a[1:]]
    assert len(got) == len(ob)
    for t, (chrom, pos, rsid, alleles, _p0, _p1, _m) in zip(got, ob):
        # default is ref-last: ALLELE0 = second allele of the file, ALLELE1 = first
        assert (int(t[0]), t[1], int(t[2]), t[3], t[4]) == (plink.chr_str_to_int(chrom), rsid, pos, alleles[1], alleles[0])


def test_bgi_chr_filter_and_mismatched_index(golden_dir):
    f = golden_dir + "/example_3chr.bgen"
    rows = probe("bgen-variants", f, "--chr", "2").stdout.splitlines()[1:]
    assert len(rows) == 400 and all(r.split()[0] == "2" for r in rows)
    r = probe("bgen-variants", f, "--bgi", golden_dir + "/example.bgen.bgi", ok=False)
    assert r.returncode != 0 and "bgi index does not match" in r.stdout
    r = probe("bgen-variants", f, "--bgi", golden_dir + "/nope.bgi", ok=False)
    assert r.returncode != 0 and "cannot open file" in r.stdout


def test_ref_first_swaps_alleles(golden_dir):
    f = golden_dir + "/example_3chr.bgen"
    a = [l.split() for l in probe("bgen-variants", f).stdout.splitlines()[1:]]
    b = [l.split() for l in probe("bgen-variants", f, "--ref-first").stdout.splitlines()[1:]]
    assert all(x[3] == y[4] and x[4] == y[3] and x[:3] == y[:3] for x, y in zip(a, b))


def test_bgen_probability_bytes_equal_oracle(golden_dir, tmp_path):
    f = golden_dir + "/example.bgen"
    ob = obgen.Bgen(f)
    first, n = 37, 25
    probe("bgen-probs", f, first, n, tmp_path / "p.bin")
    raw = np.fromfile(tmp_path / "p.bin", dtype=np.uint8)
    N = ob.n_samples
    probs = raw[: n * N * 2].reshape(n, N, 2)
    pm = raw[n * N * 2:].reshape(n, N)
    for v, (_c, _p, _r, _a, p0, p1, miss) in enumerate(ob.variants()):
        j = v - first
        if j < 0:
            continue
        if j >= n:
            break
        assert np.array_equal(probs[j, :, 0], p0) and np.array_equal(probs[j, :, 1], p1), j
        assert np.array_equal((pm[j] & 0x80) != 0, miss), j


# ------------------------------------------------------------------------------------------- PGEN
def test_host_pgen_decoder_reproduces_the_bed_rows(golden_dir, tmp_path):
    a = probe("rows", "--bed", golden_dir + "/example", tmp_path / "bed.bin").stdout.split()
    b = probe("rows", "--pgen", golden_dir + "/example", tmp_path / "pgen.bin").stdout.split()
    assert a == b == ["1000", "125", "500"]
    x = np.fromfile(tmp_path / "bed.bin", dtype=np.uint8)
    y = np.fromfile(tmp_path / "pgen.bin", dtype=np.uint8)
    assert x.size == 1000 * 125 and np.array_equal(x, y)


def test_host_pgen_decoder_all_record_types(tmp_path):
    import helpers
    from test_pgen_cpu import synthetic_calls
    g = synthetic_calls()
    pfx = str(tmp_path / "syn")
    types = helpers.write_pgen(pfx, g, storage=5)
    assert set(types) == set(range(8))
    M, N = g.shape
    helpers.write_pvar_psam(pfx, [1 + (3 * v) // M for v in range(M)], ["v%d" % v for v in range(M)], list(range(1, M + 1)),
                            ["A"] * M, ["G"] * M, ["f%d_i%d" % (i, i) for i in range(N)])
    out = probe("rows", "--pgen", pfx, tmp_path / "rows.bin").stdout.split()
    m, stride, n = int(out[0]), int(out[1]), int(out[2])
    assert (m, n) == g.shape
    rows = np.fromfile(tmp_path / "rows.bin", dtype=np.uint8).reshape(m, stride)
    codes = np.stack([(rows >> (2 * k)) & 3 for k in range(4)], axis=-1).reshape(m, -1)[:, :n]
    # PLINK 1 codes (ref-last): 00 -> 2 copies of ALT, 01 -> missing, 10 -> 1, 11 -> 0
    want = np.array([3, 2, 0, 1], dtype=np.uint8)[g]           # ALT count 0/1/2/missing(3) -> code
    assert np.array_equal(codes, want)


def big_pgen_calls(N, M, seed=5):
    """Calls whose records need difflists of many groups (> 32 groups = more than one round of a warp), every record type,
    LD records whose base lies in an earlier block, and a sample count that leaves a partial last word."""
    rng = np.random.default_rng(seed)
    g = np.zeros((M, N), dtype=np.uint8)
    inv = np.array([2, 1, 0, 3], dtype=np.uint8)

    def near(src):                                                                # src with N / 12 calls redrawn
        t = src.copy()
        idx = rng.choice(N, size=N // 12, replace=False)
        t[idx] = rng.integers(0, 4, idx.size)
        return t
    for v in range(M):
        kind = v % 10
        if kind == 0:
            g[v] = rng.binomial(2, 0.35, N)                                       # plain 2-bit
        elif kind == 1:
            g[v] = near(g[v - 1])                                                 # LD against a plain record
        elif kind == 2:
            g[v] = rng.binomial(2, 0.03, N)                                       # difflist over 0, many groups
        elif kind == 3:
            g[v] = inv[near(g[v - 1])]                                            # inverted LD against a difflist record
        elif kind == 4:
            g[v] = 2 - rng.binomial(2, 0.02, N)                                   # difflist over 2
        elif kind == 5:
            g[v] = np.where(rng.random(N) < 0.93, 3, rng.binomial(2, 0.5, N))     # difflist over missing
        elif kind == 6:
            g[v] = np.where(rng.random(N) < 0.04, 3, 1 + rng.binomial(1, 0.4, N))  # 1 bit (1 / 2) + exceptions
        elif kind == 7:
            g[v] = near(g[v - 1])                                                 # LD against a 1-bit record
        elif kind == 8:
            g[v] = inv[near(g[v - 2])]                                            # inverted LD, base two records back
        # kind 9: all hom-ref
    return g


@pytest.mark.parametrize("N,M,bs,storage", [(700, 160, 7, 5), (33333, 40, 3, 6), (70001, 20, 20, 2)])
def test_pgen_device_core_on_the_host_equals_the_host_decoder(tmp_path, N, M, bs, storage):
    """csrc/pgen_core.h (what pgen_fill_kernel / pgen_patch_kernel execute), lanes run serially, fed through
    PgenFile::gather in blocks of bs variants: byte-identical to host/pgen.cpp and to the calls that were written."""
    import helpers
    if N == 700:
        from test_pgen_cpu import synthetic_calls
        g = synthetic_calls()
    else:
        g = big_pgen_calls(N, M)
    pfx = str(tmp_path / "syn")
    types = helpers.write_pgen(pfx, g, storage=storage)
    assert set(types) >= {0, 1, 2, 3, 4, 5, 6, 7}, sorted(set(types))
    M, N = g.shape
    helpers.write_pvar_psam(pfx, [1] * M, ["v%d" % v for v in range(M)], list(range(1, M + 1)), ["A"] * M, ["G"] * M,
                            ["f%d_i%d" % (i, i) for i in range(N)])
    probe("rows", "--pgen", pfx, tmp_path / "host.bin")
    out = probe("pgen-rows", pfx, tmp_path / "core.bin", bs).stdout.split()
    m, stride, n, nrec = int(out[0]), int(out[1]), int(out[2]), int(out[3])
    assert (m, n) == g.shape and nrec >= m
    a = np.fromfile(tmp_path / "host.bin", dtype=np.uint8)
    b = np.fromfile(tmp_path / "core.bin", dtype=np.uint8)
    assert np.array_equal(a, b)
    rows = b.reshape(m, stride)
    codes = np.stack([(rows >> (2 * k)) & 3 for k in range(4)], axis=-1).reshape(m, -1)
    assert np.array_equal(codes[:, :n], np.array([3, 2, 0, 1], dtype=np.uint8)[g]) and not codes[:, n:].any()


def test_pgen_device_core_on_the_reference_fixture(golden_dir, tmp_path):
    probe("rows", "--bed", golden_dir + "/example", tmp_path / "bed.bin")
    for bs in (1, 100):
        probe("pgen-rows", golden_dir + "/example", tmp_path / "core.bin", bs)
        assert np.array_equal(np.fromfile(tmp_path / "bed.bin", dtype=np.uint8), np.fromfile(tmp_path / "core.bin", dtype=np.uint8))


# ------------------------------------------------------------------------------------------- phenotype preparation
def _keys(golden_dir, remove=False):
    keys, _ = plink.read_fam(golden_dir + "/example.fam")
    if remove:
        rm = {"_".join(l.split()[:2]) for l in open(golden_dir + "/fid_iid_to_remove.txt") if l.strip()}
        keys = [k for k in keys if k not in rm]
    return keys


def _check_prep(d, pr, bt, step1):
    N, P, C = d["hdr"]["N"], d["hdr"]["P"], d["hdr"]["C"]
    assert (N, P, C) == (len(pr.keys), len(pr.pheno_names), pr.ncov) and d["names"] == pr.pheno_names
    assert d["hdr"]["n_analyzed"] == pr.n_analyzed
    assert np.array_equal(d["mask"].reshape(P, N).T.astype(bool), pr.mask)
    assert np.array_equal(d["in_analysis"].astype(bool), pr.in_analysis)
    assert np.array_equal(d["neff"], pr.neff)
    # the basis is unique up to the sign / rotation of eigenvectors: compare the projector X X^T applied to Y-like vectors
    X = d["X"].reshape(C, N).T
    rng = np.random.default_rng(0)
    v = rng.normal(size=(N, 3))
    assert np.allclose(X @ (X.T @ v), pr.X @ (pr.X.T @ v), rtol=0, atol=1e-10)
    assert np.allclose(X.T @ X, np.eye(C), atol=1e-10)
    if (not bt) or step1:
        assert np.allclose(d["Y"].reshape(P, N).T, pr.Y, rtol=1e-10, atol=1e-10)
        assert np.allclose(d["scale_Y"], pr.scale_Y, rtol=1e-12)
    if bt:
        assert np.array_equal(d["Y_raw"].reshape(P, N).T * pr.mask, pr.Y_raw * pr.mask)


def test_prep_qt_step1_matches_oracle(golden_dir, tmp_path):
    g = golden_dir
    probe("prep", tmp_path / "d.bin", "--bed", g + "/example", "--phenoFile", g + "/phenotype.txt", "--covarFile",
          g + "/covariates.txt", "--cv", 5, "--bsize", 100)
    d = read_dump(tmp_path / "d.bin")
    pr = prep.prepare(_keys(g), g + "/phenotype.txt", g + "/covariates.txt", bt=False, step=1)
    _check_prep(d, pr, False, True)
    assert np.array_equal(d["folds"], prep.set_folds(pr.in_analysis, 5))
    bim = plink.read_bim(g + "/example.bim")
    assert [tuple(x) for x in d["blocks"].reshape(-1, 3)] == [tuple(b) for b in prep.set_blocks(bim.chrom, 100)]


def test_prep_bt_step1_with_remove_and_null_offsets(golden_dir, tmp_path):
    g = golden_dir
    probe("prep", tmp_path / "d.bin", "--bed", g + "/example", "--phenoFile", g + "/phenotype_bin.txt", "--covarFile",
          g + "/covariates.txt", "--remove", g + "/fid_iid_to_remove.txt", "--bt", "--null-eta")
    d = read_dump(tmp_path / "d.bin")
    pr = prep.prepare(_keys(g, True), g + "/phenotype_bin.txt", g + "/covariates.txt", bt=True, step=1)
    _check_prep(d, pr, True, True)
    N, P = d["hdr"]["N"], d["hdr"]["P"]
    eta = d["null_eta"].reshape(P, N).T
    for p in range(P):
        want = step1_bt.null_offset(pr.Y_raw[:, p], pr.X, pr.mask[:, p])
        m = pr.mask[:, p]
        assert np.allclose(eta[m, p], want[m], rtol=1e-8, atol=1e-10)


def test_prep_step2_with_missing_values(golden_dir, tmp_path):
    g = golden_dir
    for bt, ph in ((True, "/phenotype_bin_wNA.txt"), (False, "/phenotype.txt")):
        args = ["prep", tmp_path / "d.bin", "--bed", g + "/example", "--phenoFile", g + ph, "--covarFile",
                g + "/covariates.txt", "--step2"] + (["--bt"] if bt else [])
        probe(*args)
        d = read_dump(tmp_path / "d.bin")
        pr = prep.prepare(_keys(g), g + ph, g + "/covariates.txt", bt=bt, step=2)
        _check_prep(d, pr, bt, False)


def test_prep_rint_and_pgen_bgen_sample_sets(golden_dir, tmp_path):
    g = golden_dir
    probe("prep", tmp_path / "a.bin", "--bed", g + "/example", "--phenoFile", g + "/phenotype.txt", "--apply-rint")
    d = read_dump(tmp_path / "a.bin")
    pr = prep.prepare(_keys(g), g + "/phenotype.txt", None, bt=False, step=1, rint=True)
    _check_prep(d, pr, False, True)
    # the same samples through .psam and through the identifiers embedded in the .bgen
    probe("prep", tmp_path / "b.bin", "--pgen", g + "/example", "--phenoFile", g + "/phenotype.txt", "--apply-rint")
    probe("prep", tmp_path / "c.bin", "--bgen", g + "/example.bgen", "--phenoFile", g + "/phenotype.txt", "--apply-rint")
    for f in ("b.bin", "c.bin"):
        e = read_dump(tmp_path / f)
        assert np.array_equal(e["Y"], d["Y"]) and np.array_equal(e["mask"], d["mask"])


def test_gz_inputs_give_identical_results(golden_dir, tmp_path):
    g = golden_dir
    for f in ("phenotype_bin.txt", "covariates.txt", "fid_iid_to_remove.txt"):
        with open(g + "/" + f, "rb") as src, gzip.open(tmp_path / (f + ".gz"), "wb") as dst:
            shutil.copyfileobj(src, dst)
    common = ["--bed", g + "/example", "--bt"]
    probe("prep", tmp_path / "a.bin", *common, "--phenoFile", g + "/phenotype_bin.txt", "--covarFile", g + "/covariates.txt",
          "--remove", g + "/fid_iid_to_remove.txt")
    probe("prep", tmp_path / "b.bin", *common, "--phenoFile", tmp_path / "phenotype_bin.txt.gz", "--covarFile",
          tmp_path / "covariates.txt.gz", "--remove", tmp_path / "fid_iid_to_remove.txt.gz")
    assert open(tmp_path / "a.bin", "rb").read() == open(tmp_path / "b.bin", "rb").read()
    want = open(g + "/covariates.txt").read().splitlines()
    assert probe("cat", tmp_path / "covariates.txt.gz").stdout.splitlines() == want
    # CRLF line ends and a missing final newline
    with open(tmp_path / "crlf.txt", "wb") as fh:
        fh.write(b"a b\r\nc d\r\ne f")
    assert probe("cat", tmp_path / "crlf.txt").stdout.splitlines() == ["a b", "c d", "e f"]


# ------------------------------------------------------------------------------------------- prediction files
def _pred_reference(n, prs):
    keys = ["F%d_I%d" % (i, i) for i in range(n)]
    mask = [(i % 7) != 3 for i in range(n)]
    order = [i for k, i in sorted((keys[i], i) for i in range(n) if i % 11 != 5)]
    lines = ["FID_IID " + "".join(keys[i] + " " for i in order)]
    for r in range(1 if prs else 23):
        row = "%d " % (0 if prs else r + 1)
        for i in order:
            v = math.sin(0.37 * (r + 1) * (i + 1)) * 10.0 ** ((i % 13) - 6)
            row += ("%g " % v) if mask[i] else "NA "
        lines.append(row)
    return "\n".join(lines) + "\n", [keys[i] for i in order]


@pytest.mark.parametrize("prs", [False, True])
@pytest.mark.parametrize("gz", [False, True])
def test_loco_and_prs_files_plain_and_gz(tmp_path, prs, gz):
    n = 257
    path = str(tmp_path / ("x.prs" if prs else "x.loco")) + (".gz" if gz else "")
    probe("pred-file", path, n, *(["--prs"] if prs else []))
    raw = open(path, "rb").read()
    assert (raw[:2] == b"\x1f\x8b") == gz
    text = (gzip.decompress(raw) if gz else raw).decode()
    want, ids = _pred_reference(n, prs)
    assert text == want
    out = probe("read-pred", path, *(["--prs"] if prs else [])).stdout.splitlines()
    assert out[0] == "ids %d" % len(ids) and out[1:1 + len(ids)] == ids
    k = 1 + len(ids)
    assert out[k] == "first %d" % len(ids)
    assert out[k + 1:k + 1 + len(ids)] == want.splitlines()[1].split()[1:]
    k += 1 + len(ids)
    want_rows = {l.split()[0]: l.split()[1:] for l in want.splitlines()[1:]}
    seen = []
    while k < len(out):
        tag, c, n = out[k].split()
        assert tag == "row" and int(n) == len(ids)
        label = "0" if prs else c
        assert out[k + 1:k + 1 + len(ids)] == want_rows[label], (c, prs, gz)
        seen.append(int(c))
        k += 1 + len(ids)
    assert seen == ([23] if prs else list(range(23, 0, -1)))


def test_loco_writer_threaded_path_and_lazy_rows_at_scale(tmp_path):
    """Above 2^20 values the rows are formatted on several threads; the file must not depend on that, and the reader
    must serve any row on demand (seek in the plain file)."""
    n = 60000
    path = str(tmp_path / "big.loco")
    probe("pred-file", path, n)
    want, ids = _pred_reference(n, False)
    assert open(path).read() == want
    out = probe("read-pred", path).stdout.splitlines()
    k = out.index("row 7 %d" % len(ids))
    assert out[k + 1:k + 1 + len(ids)] == want.splitlines()[7].split()[1:]


def test_prs_reader_rejects_a_loco_file(tmp_path):
    probe("pred-file", tmp_path / "x.loco", 50)
    r = probe("read-pred", tmp_path / "x.loco", "--prs", ok=False)
    assert r.returncode != 0 and "second line must start with 0" in r.stdout


# ------------------------------------------------------------------------------------------- summary statistics rows
def _g(v):
    return "%g" % v


def test_sumstats_rows_and_log10p():
    from scipy.stats import chi2
    cases = [(0.25, 0.9876543, 494, 0.123456789, 0.0456, 7.3291, 1), (0.5, 1.0, 10, -1.5e-7, 2.5e-8, 36.0, 1),
             (0.01234567, 0.3, 500000, 0.5, -1.0, 2.0, 1), (0.3, -0.2, 77, 1.0, 0.5, 4.0, 0), (0.3, 0.5, 77, 1.0, 0.5, -1.0, 1),
             (0.11, 0.99, 1234, 3.0, 0.05, 3600.0, 1), (0.2, 0.8, 99, 0.0, 1.0, 0.0, 1)]
    stdin = "".join(" ".join(repr(x) for x in c) + "\n" for c in cases)
    out = probe("sumstats", stdin=stdin).stdout.splitlines()
    assert out[0] == "CHROM GENPOS ID ALLELE0 ALLELE1 A1FREQ INFO N TEST BETA SE CHISQ LOG10P EXTRA"
    assert out[1] == "CHROM GENPOS ID ALLELE0 ALLELE1 A1FREQ N TEST BETA SE CHISQ LOG10P EXTRA"
    for k, (af, info, n, beta, se, chisq, ok) in enumerate(cases):
        r1, r2, lp = out[2 + 3 * k], out[3 + 3 * k], float(out[4 + 3 * k])
        if chisq >= 0:
            want_lp = -chi2.logsf(chisq, 1) / math.log(10)
            assert abs(lp - want_lp) <= 1e-9 * max(1.0, want_lp), (chisq, lp, want_lp)      # incl. the underflow branch (3600)
        bs = "%s %s" % (_g(beta), _g(se)) if se >= 0 else "NA NA"
        cp = "%s %s" % (_g(chisq), _g(lp)) if (chisq >= 0 and ok) else "NA NA"
        extra = "NA" if ok else "TEST_FAIL"
        info_s = _g(info) if info >= 0 else "NA"
        assert r1 == "1 100 rs1 A G %s %s %d ADD %s %s %s" % (_g(af), info_s, n, bs, cp, extra)
        assert r2 == "23 5 rs2 AT G %s %d ADD %s %s %s" % (_g(af), n, bs, cp, extra)


def test_htp_rows_match_the_oracle_restatement():
    """host/output.cpp append_htp_row vs oracle/step2.htp_row (print_sum_stats_htp, src/Step2_Models.cpp:2542-2646) on
    randomised inputs covering every branch: QT, BT with Firth, BT without (allelic odds ratio + SE=), failed tests, missing
    SE, capped / tiny / large p-values (the three convert_logp_raw ranges), INFO present or not."""
    from oracle import step2
    rng = np.random.default_rng(9)
    cases = []
    for k in range(400):
        bt = int(k % 3 != 0)
        firth = int(bt and k % 2)
        ok = int(k % 11 != 5)
        beta = float(rng.normal() * 10 ** rng.uniform(-4, 1))
        se = float(abs(rng.normal()) * 10 ** rng.uniform(-4, 0)) if k % 13 != 7 else -1.0
        chisq = float(rng.chisquare(1) * 10 ** rng.uniform(-1, 2.5)) if k % 17 != 3 else -1.0
        logp = float(10 ** rng.uniform(-3, 2.6)) if k % 19 != 4 else 400.0
        if k % 23 == 6:
            logp = 0.0
        af = float(rng.uniform(0, 1)) if k % 29 != 8 else -1.0
        mac = float(rng.uniform(0.5, 5000))
        gc = [int(x) for x in rng.integers(0, 3000, 6)]
        score, skat = float(rng.normal() * 100), float(abs(rng.normal()) * 10 ** rng.uniform(-6, 5))
        cal = -1.0 if not bt else float(rng.uniform(0.1, 2))
        info = float(rng.uniform(0, 1)) if k % 5 == 0 else -1.0
        cases.append((bt, firth, ok, beta, se, chisq, logp, af, mac, *gc, score, skat, cal, info))
    stdin = "".join(" ".join(repr(x) for x in c) + "\n" for c in cases)
    out = probe("htp", stdin=stdin).stdout.splitlines(keepends=True)
    assert out[0] == step2.HTP_HEADER
    assert len(out) == 1 + len(cases)
    for row, c in zip(out[1:], cases):
        bt, firth, ok, beta, se, chisq, logp, af, mac = c[:9]
        want = step2.htp_row("rs1", 1, 100, "A", "G", "Y1", "COHORT", step2.htp_model(bt=bool(bt), firth=bool(firth)), beta, se,
                             chisq, logp, af, mac, list(c[9:15]), test_pass=bool(ok), bt=bool(bt), firth=bool(firth),
                             score=c[15], skat_var=c[16], cal_factor=c[17], info=c[18] if c[18] >= 0 else None)
        assert row == want, (c, row, want)


def test_golden_rows_are_reproduced_by_the_row_formatter(golden_dir):
    """Feed the numbers of the reference's golden file back through the formatter: every row must come out identical
    (the LOG10P column is recomputed from CHISQ, so rows whose CHISQ was rounded to 6 digits are compared on the other
    columns)."""
    rows = open(golden_dir + "/test_bin_out_firth_Y1.regenie").read().splitlines()[1:]
    stdin, keep = "", []
    for r in rows[:200]:
        t = r.split()
        if "NA" in t[9:11] or t[13] != "NA":
            continue
        keep.append(t)
        stdin += " ".join([t[5], t[6], t[7], t[9], t[10], t[11], "1"]) + "\n"
    out = probe("sumstats", stdin=stdin).stdout.splitlines()[2:]
    assert len(keep) > 150
    for k, t in enumerate(keep):
        got = out[3 * k].split()
        assert got[5:12] == t[5:12], (got, t)


def test_ids_file(tmp_path):
    stdin = "f1 i1 1\nf2 i2 0\nf3 i3 1\nf4 i4 1\n"
    probe("ids", tmp_path / "a.ids", "Y1", 0, stdin=stdin)
    assert open(tmp_path / "a.ids").read() == "f1\ti1\nf3\ti3\nf4\ti4"
    probe("ids", tmp_path / "b.ids", "Y1", 1, stdin=stdin)
    assert open(tmp_path / "b.ids").read() == "Y1\tNA\nf1\ti1\nf3\ti3\nf4\ti4"


# ------------------------------------------------------------------------------------------- device inflate core on the host
@pytest.mark.parametrize("variant", [(), ("window",)])
def test_inflate_core_reproduces_zlib_on_every_bgen_payload(golden_dir, variant):
    """csrc/inflate_core.h is the decoder the GPU runs (one warp per variant stream); compiled for the host with a
    one-lane warp it must reproduce zlib byte for byte on every variant of the reference's fixtures, and reject
    truncated / corrupted streams."""
    for name, m in (("example", 1000), ("example_3chr", 500)):
        out = probe("inflate-bgen", "%s/%s.bgen" % (golden_dir, name), *variant).stdout.splitlines()[-1].split()
        assert out[:4] == ["variants", str(m), "bad", "0"], out


@pytest.mark.parametrize("variant", [(), ("window",)])
def test_inflate_core_block_types_and_error_paths(tmp_path, variant):
    import zlib
    rng = np.random.default_rng(5)
    payloads = {
        "empty": b"",
        "one": b"x",
        "run": b"\x00" * 70000,                                                  # distance-1 matches longer than the distance
        "pairs": bytes([255, 0]) * 40000 + bytes([0, 0]) * 3000,                 # what hard-call-like probabilities look like
        "random": rng.integers(0, 256, 100000, dtype=np.uint8).tobytes(),        # incompressible: stored blocks at level 0/1
        "text": (b"the quick brown fox jumps over the lazy dog " * 3000)[:120001],
        "probs": np.clip(rng.normal(128, 60, 200000), 0, 255).astype(np.uint8).tobytes(),   # long Huffman codes
        "far": rng.integers(0, 4, 40000, dtype=np.uint8).tobytes() * 3,          # matches at distances up to 32K
    }
    strategies = [(zlib.Z_DEFAULT_STRATEGY, "default"), (zlib.Z_FIXED, "fixed"), (zlib.Z_HUFFMAN_ONLY, "huff"), (zlib.Z_RLE, "rle")]
    n = 0
    for name, data in payloads.items():
        for level in (0, 1, 6, 9):
            for strat, sname in strategies:
                c = zlib.compressobj(level, zlib.DEFLATED, 15, 9, strat)
                z = c.compress(data) + c.flush()
                (tmp_path / "in.z").write_bytes(z)
                r = probe("inflate", tmp_path / "in.z", len(data), tmp_path / "out.bin", *variant).stdout.split()
                assert r == ["status", "0"], (name, level, sname, r)
                assert (tmp_path / "out.bin").read_bytes() == data, (name, level, sname)
                n += 1
    assert n == 8 * 4 * 4
    z = zlib.compress(payloads["text"], 6)
    cases = {
        "short output": (z, len(payloads["text"]) - 1, 7),          # kErrOutput
        "long output": (z, len(payloads["text"]) + 1, 9),           # kErrLength
        "bad header": (b"\x79" + z[1:], len(payloads["text"]), 1),
        "bad adler": (z[:-1] + bytes([z[-1] ^ 1]), len(payloads["text"]), 10),
        "truncated": (z[: len(z) // 2], len(payloads["text"]), None),
        "raw deflate": (z[2:], len(payloads["text"]), None),
    }
    for name, (blob, out_len, want) in cases.items():
        (tmp_path / "in.z").write_bytes(blob)
        st = int(probe("inflate", tmp_path / "in.z", out_len, tmp_path / "out.bin", *variant).stdout.split()[1])
        assert st != 0 and (want is None or st == want), (name, st)


# ------------------------------------------------------------------------------------------- variant-level INFO (--minINFO)
@pytest.mark.parametrize("ref_first", [False, True])
def test_variant_level_info_matches_the_oracle_formula(tmp_path, ref_first):
    """info1 of compute_aaf_info (src/Geno.cpp:3134-3137) from the host's integer sums vs the per-sample floating-point
    formula of oracle/bgen.py, on a synthetic file with real imputation uncertainty and missing calls; the file also goes
    through the oracle's own BGEN reader and the device decoder's host build."""
    import helpers
    M, N = 60, 700
    probs, miss = helpers.synthetic_dosage_probs(M, N, seed=4)
    f = str(tmp_path / "syn.bgen")
    helpers.write_bgen(f, probs, miss, [1] * M, range(1, M + 1), ["v%d" % v for v in range(M)])
    got = [float(x) for x in probe("bgen-info", f, *(["--ref-first"] if ref_first else [])).stdout.split()]
    assert len(got) == M
    ob = list(obgen.Bgen(f).variants())
    assert len(ob) == M
    lo = 2.0
    for v, (_c, _p, rsid, _a, p0, p1, m) in enumerate(ob):
        assert rsid == "v%d" % v and np.array_equal(p0[~m], probs[v, ~miss[v], 0]) and np.array_equal(m, miss[v])
        g, ival = obgen.dosage(p0, p1, m, ref_first)
        ok = ~m
        ns, tot = ok.sum(), g[ok].sum()
        af = tot / (2 * ns)
        want = 1.0 if af in (0.0, 1.0) else 1 - ival[ok].sum() / (2 * ns * af * (1 - af))
        assert abs(got[v] - want) < 1e-10, (v, got[v], want)
        lo = min(lo, want)
    assert lo < 0.8                                                  # the file really has low-INFO variants
    assert probe("inflate-bgen", f, "window").stdout.splitlines()[-1].split()[:4] == ["variants", str(M), "bad", "0"]


# ------------------------------------------------------------------------------------------- genotype counts (--no-split, --htp)
def _counts_fileset(tmp_path, kind):
    """239 samples (a partial last word of 32 and a partial last byte), 5 % missing calls, a remove list of 17 samples, a
    male vector and non-PAR flags.  On the .bgen every third male call of a non-PAR variant is set to dosage exactly 1
    (p1 + 2 hom = 255, for either allele order) or to a pair with p0 + p1 = 255."""
    import helpers
    from regenie_b200 import synth
    M, N = 48, 239
    rng = np.random.default_rng(17)
    male = rng.random(N) < 0.5
    non_par = rng.random(M) < 0.5
    removed = np.sort(rng.choice(N, 17, replace=False))
    pfx = str(tmp_path / "c")
    if kind == "bed":
        g = synth.genotypes(N, M, seed=17, miss=0.05)
        with open(pfx + ".bed", "wb") as fh:
            fh.write(b"\x6c\x1b\x01" + synth.pack_bed(g).tobytes())
        with open(pfx + ".bim", "w") as fh:
            fh.write("".join("1 rs%d 0 %d A G\n" % (v, 1000 + v) for v in range(M)))
        with open(pfx + ".fam", "w") as fh:
            fh.write("".join("F%d I%d 0 0 1 -9\n" % (s, s) for s in range(N)))
        ids = ["F%d I%d" % (s, s) for s in removed]
        bim = plink.read_bim(pfx + ".bim")
        raw = plink.read_bed_rows(pfx + ".bed", N, bim.offset)
        geno = lambda rf: plink.decode_bed(raw, N, ref_first=rf)
    else:
        probs, miss = helpers.synthetic_dosage_probs(M, N, seed=17, miss_rate=0.05)
        one = [(p0, 255 - 2 * p0) for p0 in range(128)]                                   # ref-last dosage 1
        one += [(x, 2 * x - 255) for x in range(128, 256)]                                # --ref-first dosage 1
        one += [(p0, 255 - p0) for p0 in range(0, 256, 5)]                                # p0 + p1 = 255
        vs, ss = np.nonzero(non_par[:, None] & male[None, :])
        for k, (v, s) in enumerate(zip(vs[::3], ss[::3])):
            probs[v, s] = one[k % len(one)]
        f = pfx + ".bgen"
        helpers.write_bgen(f, probs, miss, [1] * M, range(1, M + 1), ["v%d" % v for v in range(M)])
        ids = ["s%d s%d" % (s, s) for s in removed]
        geno = lambda rf: np.stack([obgen.dosage(p0, p1, m, rf)[0] for *_, p0, p1, m in obgen.Bgen(f).variants()])
    with open(pfx + ".remove", "w") as fh:
        fh.write("\n".join(ids) + "\n")
    kept = np.setdiff1d(np.arange(N), removed)
    return (["--" + kind, pfx if kind == "bed" else pfx + ".bgen", "--remove", pfx + ".remove"], geno, kept, male[kept],
            non_par, N)


@pytest.mark.parametrize("ref_first", [False, True])
@pytest.mark.parametrize("cfg", ["nosplit", "qt", "bt"])
@pytest.mark.parametrize("kind", ["bed", "bgen"])
def test_genotype_counts_match_numpy(tmp_path, kind, cfg, ref_first):
    """host/counts.cpp: the hard-call counter on the 2-bit rows and the dosage counter on the probability pairs against
    oracle/plink.decode_bed and oracle/bgen.dosage.  --no-split's table: the analysed samples as one column, no male rule;
    --htp's: one column per trait, cases and controls apart for a binary trait, the male rule on non-PAR variants (a male
    call with g >= 1 is alt, any other male call ref; update_genocounts, src/Geno.cpp:2986-3018)."""
    args, geno, kept, male, non_par, n_file = _counts_fileset(tmp_path, kind)
    M, N = len(non_par), len(kept)
    assert n_file % 32 != 0 and N < n_file
    rng = np.random.default_rng(3)
    T, binary, rule = {"nosplit": (1, False, False), "qt": (2, False, True), "bt": (3, True, True)}[cfg]
    cls = rng.integers(0, 3 if binary else 2, (T, N)).astype(np.uint8)
    with open(tmp_path / "cls.bin", "wb") as fh:
        fh.write(b"%d %d %d %d\n" % (T, binary, rule, rule))
        fh.write(cls.tobytes() + (male.astype(np.uint8).tobytes() + non_par.astype(np.uint8).tobytes() if rule else b""))
    out = probe("counts", tmp_path / "cls.bin", tmp_path / "out.bin", *args, *(["--ref-first"] if ref_first else [])).stdout.split()
    assert [int(x) for x in out] == [M, N, n_file]
    got = np.fromfile(tmp_path / "out.bin", dtype=np.int64).reshape(M, T, 6)

    g = geno(ref_first)[:, kept]
    ok = g >= 0
    alt, het = ok & (g >= 1.5), ok & (g >= 0.5) & (g < 1.5)
    xm = ok & non_par[:, None] & male[None, :] & rule
    alt, het = np.where(xm, g >= 1, alt), het & ~xm
    ref = ok & ~alt & ~het
    want = np.zeros((M, T, 6), dtype=np.int64)
    for t in range(T):
        for k, c in enumerate((2, 1) if binary else (1,)):
            sel = cls[t] == c
            want[:, t, 3 * k:3 * k + 3] = np.stack([(x & sel).sum(1) for x in (ref, het, alt)], axis=1)
    assert np.array_equal(got, want)
    assert (~ok).any() and ((g == 1) & ~ok).sum() == 0
    if cfg == "nosplit":
        # N_RA of the --no-split row: the het count is the analysed non-missing calls minus N_RR and N_AA
        assert np.array_equal(got[:, 0, 1], (ok & (cls[0] == 1)).sum(1) - got[:, 0, 0] - got[:, 0, 2])
    if rule:
        if kind == "bed":
            assert (xm & (g == 1)).any()                                                 # heterozygous males, counted as alt
        else:
            assert (xm & (g == 1.0)).any()                                               # dosage exactly 1 in the float expression
            if ref_first:                                                                # ... and pairs at 255 / 255 that it puts below 1
                assert (xm & (g < 1) & (g > 1 - 1e-12)).any()
