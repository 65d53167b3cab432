"""Option-combination sweeps of the rgb200 driver, used when the driver changes:

    python tools/driver_sweeps.py regress <commit>   # build the driver of <commit> and that of the working tree, both against
                                                     # the working tree's mock ABI (tests/mock/mock_abi.cpp) and
                                                     # include/rg_b200.h, run Step 1 / Step 2 over the option grid with both
                                                     # binaries, compare every output file and the mock's call trace byte for byte
    python tools/driver_sweeps.py regress OLD NEW    # the same grid on two prebuilt rgb200 binaries, e.g. linked against the
                                                     # real library on a GPU host (which writes no trace: output files only)
    python tools/driver_sweeps.py htp                # every --htp combination under -fsanitize=address,undefined: exit code,
                                                     # no sanitizer report, 22 columns, Num = Ref + Het + Alt > 0

The Step-2 grid: bed / bgen / pgen x QT / BT / Firth / SPA, with --ignore-pred, under each single extra option and a fixed
list of option pairs; the same inputs and trait kinds with LOCO predictions of one Step-1 run per trait kind (and one
--use-null-firth run); a chromosome-23 fileset with alternating sexes and variants in PAR1, the non-PAR part and PAR2.
The mock writes one line per Step-2 entry point to RG_MOCK_TRACE (name, handle, bs, min_mac, pending non-PAR flags,
checksum of uploads), so a call that moves to another handle or loses its non-PAR flags shows up even where no output
file changes.  The mock's block routes each need their own chromosome call (rg_s2_set_chr or rg_s2_set_chr_bt), so a
driver that calls the route of the other trait kind fails there and `regress` reports the pair.  The htp sweep found
--htp --bt --pgen decoding on the device, where the genotype counts could not see the rows."""
import concurrent.futures
import glob
import gzip
import itertools
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = os.path.join(ROOT, "tests", "golden", "example")
LIBS = ["-lz", "-lpthread", "-ldl"]
PAIRS = {"dom+afcc": ("dom", "afcc"), "rec+nosplit": ("rec", "nosplit"), "dom+htp": ("dom", "htp"), "afcc+reffirst": ("afcc", "reffirst"),
         "nosplit+htp": ("nosplit", "htp"), "mininfo+nosplit": ("mininfo", "nosplit"), "rec+start2": ("rec", "start2"),
         "remove+afcc": ("remove", "afcc")}


# the driver sources under src_root/regenie_b200/host, linked with the working tree's mock ABI; they include
# src_root/include/rg_b200.h
def build(src_root, out, flags):
    srcs = sorted(glob.glob(os.path.join(src_root, "regenie_b200", "host", "*.cpp"))) + [os.path.join(ROOT, "tests", "mock", "mock_abi.cpp")]
    subprocess.run(["g++", "-O1", "-std=c++17", "-o", out] + flags + srcs + LIBS, check=True)
    return out


def grids(t):
    fam = [l.split() for l in open(D + "/example_3chr.fam")]
    rem = t + "/rem.txt"
    open(rem, "w").write("".join("%s %s\n" % (x[0], x[1]) for x in fam[5:300:11]))
    inputs = {"bed": ["--bed", D + "/example_3chr"], "bgen": ["--bgen", D + "/example_3chr.bgen", "--sample", D + "/example_3chr.sample"],
              "pgen": ["--pgen", D + "/example"]}
    traits = {"qt": ["--phenoFile", D + "/phenotype.txt"], "bt": ["--phenoFile", D + "/phenotype_bin.txt", "--bt"],
              "firth": ["--phenoFile", D + "/phenotype_bin.txt", "--bt", "--firth", "--approx", "--pThresh", "0.1"],
              "spa": ["--phenoFile", D + "/phenotype_bin.txt", "--bt", "--spa", "--pThresh", "0.1"]}
    extras = {"plain": [], "remove": ["--remove", rem], "dom": ["--test", "dominant"], "rec": ["--test", "recessive"],
              "reffirst": ["--ref-first"], "nosplit": ["--no-split"], "start2": ["--starting-block", "2"], "minmac": ["--minMAC", "20"],
              "afcc": ["--af-cc"], "mininfo": ["--minINFO", "0.5"], "gpuinfl": ["--gpu-inflate"], "ws": ["--write-samples"],
              "gz": ["--gz"], "chr2": ["--chr", "2"]}
    return inputs, traits, extras


def skip(ik, eks):
    return (("mininfo" in eks or "gpuinfl" in eks) and ik != "bgen") or (ik == "pgen" and "chr2" in eks)   # example.pgen: chromosome 1 only


# example_3chr as chromosome 23: every other sample male, variants in turn in PAR1, the non-PAR part and PAR2 (default hg38 bounds)
def chrx_fileset(t):
    x = t + "/chrx"
    shutil.copy(D + "/example_3chr.bed", x + ".bed")
    with open(x + ".bim", "w") as fh:
        for i, l in enumerate(open(D + "/example_3chr.bim")):
            c = l.split()
            fh.write("23\t%s\t0\t%d\t%s\t%s\n" % (c[1], (1000, 5_000_000, 156_000_000)[i % 3] + i, c[4], c[5]))
    with open(x + ".fam", "w") as fh:
        for i, l in enumerate(open(D + "/example_3chr.fam")):
            c = l.split()
            fh.write("%s\t%s\t0\t0\t%d\t%s\n" % (c[0], c[1], 1 + i % 2, c[5]))
    return x


def same_outputs(o_old, o_new, what):
    skip = (".log", "pred.list", "prs.list")                                   # hold paths
    fo = sorted(f for f in glob.glob(o_old + "*") if not f.endswith(skip))
    fn = sorted(f for f in glob.glob(o_new + "*") if not f.endswith(skip))
    if not fo or [os.path.basename(f)[3:] for f in fo] != [os.path.basename(f)[3:] for f in fn]:
        print("FILES", what)
        return False
    for a, b in zip(fo, fn):
        if open(a, "rb").read() != open(b, "rb").read():
            print("DIFF", what, os.path.basename(a))
            return False
    return True


def run_pair(bins, t, name, args, must):
    """runs both binaries on one option set into t/name/; True when they agree: the same exit code and, for a run that
    succeeds (which `must` requires), the same output files and mock trace"""
    os.makedirs(os.path.join(t, name))
    rc, outs = [], []
    for tag, b in bins:
        o = os.path.join(t, name, tag)
        rc.append(subprocess.run([b] + args + ["--out", o], capture_output=True, text=True,
                                 env=dict(os.environ, RG_MOCK_TRACE=o + ".trace")).returncode)
        outs.append(o)
    return rc[0] == rc[1] and (rc[0] != 0 and not must or same_outputs(outs[0], outs[1], name))


def regress(args):
    t = tempfile.mkdtemp()
    if len(args) == 2:                                                         # two prebuilt binaries
        what, bins = " vs ".join(args), (("old", os.path.abspath(args[0])), ("new", os.path.abspath(args[1])))
    else:                                                                      # the driver of a commit, on today's ABI
        what, old_root = args[0], os.path.join(t, "old_src")
        os.makedirs(old_root)
        tar = subprocess.run(["git", "-C", ROOT, "archive", args[0], "regenie_b200/host"], capture_output=True, check=True).stdout
        subprocess.run(["tar", "-x", "-C", old_root], input=tar, check=True)
        shutil.copytree(os.path.join(ROOT, "include"), os.path.join(old_root, "include"))
        bins = (("old", build(old_root, t + "/mock_old", [])), ("new", build(ROOT, t + "/mock_new", [])))
    inputs, traits, extras = grids(t)
    extras["htp"] = ["--htp", "C"]
    cov = ["--covarFile", D + "/covariates.txt", "--bsize", "100"]
    jobs = []                                                                  # (name, args, must succeed)
    for (ik, iv), (tk, tv) in itertools.product(inputs.items(), traits.items()):
        s2 = ["--step", "2"] + iv + tv + cov
        for ek in list(extras) + list(PAIRS):
            eks = PAIRS.get(ek, (ek,))
            if not skip(ik, eks):
                jobs.append(("s2_%s_%s_%s" % (ik, tk, ek), s2 + ["--ignore-pred"] + sum((extras[e] for e in eks), []), False))
        jobs.append(("s2_%s_%s_loco" % (ik, tk), s2 + ["--pred", t + "/fit_%s_pred.list" % ("qt" if tk == "qt" else "bt")], True))
    jobs.append(("s2_bed_firth_nullfirth", ["--step", "2"] + inputs["bed"] + traits["firth"] + cov +
                 ["--pred", t + "/fit_bt_pred.list", "--use-null-firth", t + "/fit_bt_firth.list"], True))
    x = chrx_fileset(t)
    for (tk, tv), ek in itertools.product(list(traits.items())[:2], ("plain", "htp", "dom", "afcc")):
        jobs.append(("s2_chrx_%s_%s" % (tk, ek), ["--step", "2", "--bed", x] + tv + cov + ["--ignore-pred"] + extras[ek], True))
    for ik, iv in {"bed": ["--bed", D + "/example"], "pgen": ["--pgen", D + "/example"], "bgen": ["--bgen", D + "/example.bgen"]}.items():
        for tk, tv in {"qt": ["--phenoFile", D + "/phenotype.txt"], "bt": ["--phenoFile", D + "/phenotype_bin.txt", "--bt"]}.items():
            for ek, ev in {"plain": [], "loocv": ["--loocv"], "lowmem": ["--lowmem", "--lowmem-prefix", t + "/lm_" + ik + tk], "prs": ["--print-prs"],
                           "gpus1": ["--gpus", "1"]}.items():
                jobs.append(("s1_%s_%s_%s" % (ik, tk, ek), ["--step", "1"] + iv + tv + cov + ev, True))
    # the LOCO predictions of the --pred runs: one Step-1 fit per trait kind, by the new binary
    for tk, tv in (("qt", traits["qt"]), ("bt", traits["bt"] + ["--write-null-firth"])):
        subprocess.run([bins[1][1], "--step", "1", "--bed", D + "/example_3chr"] + tv + cov + ["--out", t + "/fit_" + tk],
                       capture_output=True, check=True)
    with concurrent.futures.ThreadPoolExecutor(min(8, os.cpu_count() or 1)) as ex:
        bad = sum(not ok for ok in ex.map(lambda j: run_pair(bins, t, *j), jobs))
    print("regress vs %s: %d pairs, %d differ" % (what, len(jobs), bad))
    return bad


def htp():
    t = tempfile.mkdtemp()
    b = build(ROOT, t + "/mock_asan", ["-g", "-fsanitize=address,undefined"])
    inputs, traits, extras = grids(t)
    n = bad = 0
    for (ik, iv), (tk, tv), (ek, ev) in itertools.product(inputs.items(), traits.items(), extras.items()):
        if skip(ik, (ek,)):
            continue
        out = "%s/%s_%s_%s" % (t, ik, tk, ek)
        r = subprocess.run([b, "--step", "2"] + iv + tv + ["--covarFile", D + "/covariates.txt", "--bsize", "100", "--ignore-pred", "--htp", "C"]
                           + ev + ["--out", out], capture_output=True, text=True, env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0"))
        n += 1
        if r.returncode != 0 or "runtime error" in r.stderr or "AddressSanitizer" in r.stderr:
            bad += 1
            print("FAIL", ik, tk, ek, r.returncode, (r.stdout + r.stderr)[-300:])
            continue
        f = out + "_Y1.regenie" + (".gz" if ek == "gz" else "")
        rows = (gzip.open(f, "rt") if ek == "gz" else open(f)).read().splitlines()
        ok = len(rows) > 50
        for l in rows[1:]:
            c = l.split("\t")
            a = [int(x) for x in c[13:17]] if len(c) == 22 else [0, 1]
            ok &= a[0] == sum(a[1:]) and a[0] > 0
            if tk != "qt" and len(c) == 22:
                k = [int(x) for x in c[17:21]]
                ok &= k[0] == sum(k[1:]) and k[0] > 0
        if not ok:
            bad += 1
            print("ROWS", ik, tk, ek)
    print("htp: %d runs, %d bad" % (n, bad))
    return bad


if __name__ == "__main__":
    sys.exit(1 if (regress(sys.argv[2:]) if sys.argv[1] == "regress" else htp()) else 0)
