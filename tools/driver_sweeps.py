"""Option-combination sweeps of the rgb200 driver against the mock ABI (tests/mock/mock_abi.cpp), used when the driver
changes without a GPU at hand:

    python tools/driver_sweeps.py regress <commit>   # build the driver + mock of <commit>, run Step 1 / Step 2 over the option
                                                     # grid with both binaries, compare every output file byte for byte
    python tools/driver_sweeps.py htp                # every --htp combination under -fsanitize=address,undefined: exit code,
                                                     # no sanitizer report, 22 columns, Num = Ref + Het + Alt > 0

The mock's block routes each need their own chromosome call (rg_s2_set_chr or rg_s2_set_chr_bt), so a driver that calls the
route of the other trait kind fails there and `regress` reports the pair.  The htp sweep found --htp --bt --pgen decoding
on the device, where the genotype counts could not see the rows."""
import glob
import gzip
import itertools
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = os.path.join(ROOT, "tests", "golden", "example")
LIBS = ["-lz", "-lpthread", "-ldl"]


def build(src_root, out, flags):
    srcs = sorted(glob.glob(os.path.join(src_root, "regenie_b200", "host", "*.cpp"))) + [os.path.join(src_root, "tests", "mock", "mock_abi.cpp")]
    subprocess.run(["g++", "-O1", "-std=c++17", "-I", os.path.join(src_root, "include"), "-o", out] + flags + srcs + LIBS, check=True)
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


def same_outputs(o_old, o_new, what):
    skip = (".log", "pred.list", "prs.list")                                   # hold paths
    fo = sorted(f for f in glob.glob(o_old + "*") if not f.endswith(skip))
    fn = sorted(f for f in glob.glob(o_new + "*") if not f.endswith(skip))
    if not fo or [os.path.basename(f)[4:] for f in fo] != [os.path.basename(f)[4:] for f in fn]:
        print("FILES", what)
        return False
    for a, b in zip(fo, fn):
        if open(a, "rb").read() != open(b, "rb").read():
            print("DIFF", what, os.path.basename(a))
            return False
    return True


def regress(commit):
    t = tempfile.mkdtemp()
    old_root = os.path.join(t, "old_src")
    os.makedirs(old_root)
    tar = subprocess.run(["git", "-C", ROOT, "archive", commit, "regenie_b200/host", "include", "tests/mock", "regenie_b200/csrc/pgen_core.h",
                          "regenie_b200/csrc/inflate_core.h"], capture_output=True, check=True).stdout
    subprocess.run(["tar", "-x", "-C", old_root], input=tar, check=True)
    bins = (("old", build(old_root, t + "/mock_old", [])), ("new", build(ROOT, t + "/mock_new", [])))
    inputs, traits, extras = grids(t)
    extras["htp"] = ["--htp", "C"]
    n = bad = 0
    for (ik, iv), (tk, tv), (ek, ev) in itertools.product(inputs.items(), traits.items(), extras.items()):
        if (ek in ("mininfo", "gpuinfl") and ik != "bgen") or (ik == "pgen" and ek == "chr2"):    # example.pgen holds chromosome 1 only
            continue
        rc, outs = [], []
        for tag, b in bins:
            o = "%s/%s_s2_%s_%s_%s" % (t, tag, ik, tk, ek)
            rc.append(subprocess.run([b, "--step", "2"] + iv + tv + ["--covarFile", D + "/covariates.txt", "--bsize", "100", "--ignore-pred"]
                                     + ev + ["--out", o], capture_output=True, text=True).returncode)
            outs.append(o)
        n += 1
        bad += not (rc[0] == rc[1] and (rc[0] != 0 or same_outputs(outs[0], outs[1], ("step2", ik, tk, ek))))
    for ik, iv in {"bed": ["--bed", D + "/example"], "pgen": ["--pgen", D + "/example"], "bgen": ["--bgen", D + "/example.bgen"]}.items():
        for tk, tv in {"qt": ["--phenoFile", D + "/phenotype.txt"], "bt": ["--phenoFile", D + "/phenotype_bin.txt", "--bt"]}.items():
            for ek, ev in {"plain": [], "loocv": ["--loocv"], "lowmem": ["--lowmem", "--lowmem-prefix", t + "/lm"], "prs": ["--print-prs"],
                           "gpus1": ["--gpus", "1"]}.items():
                rc, outs = [], []
                for tag, b in bins:
                    o = "%s/%s_s1_%s_%s_%s" % (t, tag, ik, tk, ek)
                    rc.append(subprocess.run([b, "--step", "1"] + iv + tv + ["--covarFile", D + "/covariates.txt", "--bsize", "100"] + ev
                                             + ["--out", o], capture_output=True, text=True).returncode)
                    outs.append(o)
                n += 1
                bad += not (rc[0] == rc[1] == 0 and same_outputs(outs[0], outs[1], ("step1", ik, tk, ek)))
    print("regress vs %s: %d pairs, %d differ" % (commit, n, bad))
    return bad


def htp():
    t = tempfile.mkdtemp()
    b = build(ROOT, t + "/mock_asan", ["-g", "-fsanitize=address,undefined"])
    inputs, traits, extras = grids(t)
    n = bad = 0
    for (ik, iv), (tk, tv), (ek, ev) in itertools.product(inputs.items(), traits.items(), extras.items()):
        if (ek in ("mininfo", "gpuinfl") and ik != "bgen") or (ik == "pgen" and ek == "chr2"):    # example.pgen holds chromosome 1 only
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
    sys.exit(1 if (regress(sys.argv[2]) if sys.argv[1] == "regress" else htp()) else 0)
