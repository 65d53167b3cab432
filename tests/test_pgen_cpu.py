"""The .pgen restatement (oracle/pgen.py) against the reference's own fixture pair: example/example.pgen must decode to
exactly the genotypes of example/example.bed (both ship with the reference and hold the same 1000 x 500 calls), and a
synthetic file written record type by record type (tests/helpers.write_pgen) must round-trip."""
import collections
import hashlib
import os

import numpy as np

import helpers
from oracle import pgen, plink


def test_example_pgen_equals_example_bed(golden_dir):
    d = golden_dir
    pg = pgen.Pgen(d + "/example.pgen")
    bim = plink.read_bim(d + "/example.bim")
    keys, _ = plink.read_fam(d + "/example.fam")
    G = plink.decode_bed(plink.read_bed_rows(d + "/example.bed", len(keys), bim.offset), len(keys))
    assert (pg.m, pg.n) == (1000, 500) and int(pg.fpos[-1]) == len(pg.d)
    for v in range(pg.m):
        g = pg.read(v).astype(float)
        g[g == 3] = -3.0
        assert np.array_equal(g, G[v]), v
    pv = pgen.read_pvar(d + "/example.pvar")
    ks, _ = pgen.read_psam(d + "/example.psam")
    assert ks == keys
    assert [(r[2], r[3], r[4]) for r in pv] == list(zip(bim.ids, bim.allele0, bim.allele1))   # ALLELE0 = REF, ALLELE1 = ALT


def synthetic_calls(N=700, M=160, seed=1):
    rng = np.random.default_rng(seed)
    g = np.zeros((M, N), dtype=np.uint8)
    for v in range(M):
        kind = v % 8
        if kind == 0:
            pass                                              # all hom-ref
        elif kind == 1:
            g[v] = rng.binomial(2, 0.15, N)                   # common (hom-alt below n / 16: a 1-bit record)
        elif kind == 2:
            g[v] = rng.binomial(2, 0.01, N)                   # rare
        elif kind == 3:
            g[v] = 2 - rng.binomial(2, 0.01, N)               # almost fixed for ALT
        elif kind == 4:
            g[v] = np.where(rng.random(N) < 0.95, 3, rng.binomial(2, 0.4, N))   # mostly missing
        elif kind == 5:
            g[v] = g[v - 4].copy(); g[v, rng.integers(0, N, 5)] = 1              # in LD with a common one
        elif kind == 6:
            t = g[v - 5].copy(); t[rng.integers(0, N, 4)] = 3
            g[v] = np.array([2, 1, 0, 3], dtype=np.uint8)[t]                      # inverted LD
        elif v % 16 == 7:
            g[v] = rng.integers(0, 4, N)                      # nothing compresses
        else:
            g[v] = g[v - 2].copy(); g[v, rng.integers(0, N, 6)] = 2              # LD with the latest non-LD record
    return g


def test_pgen_round_trip_all_record_types(tmp_path):
    g = synthetic_calls()
    for storage in (1, 6):
        prefix = str(tmp_path / ("syn%d" % storage))
        types = helpers.write_pgen(prefix, g, storage=storage)
        assert set(types) >= {0, 1, 2, 3, 4, 5, 6, 7}, collections.Counter(types)
        pg = pgen.Pgen(prefix + ".pgen")
        for v in list(range(g.shape[0])) + [150, 7, 6, 5, 13, 14]:       # sequential, then random access into LD records
            assert np.array_equal(pg.read(v), g[v]), (storage, v, types[v])


# ------------------------------------------------------------------------------------ pinned on the reference's own pgenlib
# The reference's vendored pgenlib was run on these inputs when the digests under tests/golden/pgenlib/ were stored:
# PgrValidate accepted every file, and ReadHardcalls (allele 1, missing = -3) returned int8 calls.  Stored: the SHA-256
# of those calls and, for the synthetic files, of the .pgen bytes pgenlib validated and decoded.
def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(np.asarray(a, dtype=np.int8)).tobytes()).hexdigest()


def _pgenlib_digests(golden_dir, name):
    path = os.path.join(os.path.dirname(golden_dir), "pgenlib", name)
    return [line.split() for line in open(path).read().splitlines() if line.strip()]


def test_oracle_equals_pgenlib_on_the_reference_fixture(golden_dir):
    """oracle/pgen.py vs the reference's vendored pgenlib, called as the reference calls it (ReadHardcalls, allele 1)."""
    [[want]] = _pgenlib_digests(golden_dir, "example_hardcalls.sha256")
    pg = pgen.Pgen(golden_dir + "/example.pgen")
    got = np.stack([pg.read(v) for v in range(1000)]).astype(np.int8)
    got[got == 3] = -3
    assert _digest(got) == want


def test_synthetic_files_pass_pgenlib_validation_and_read_back(tmp_path, golden_dir):
    """The test writer (helpers.write_pgen) is itself checked by the reference library: PgrValidate accepts the files
    (record types, difflist group byte counts, trailing bits) and ReadHardcalls returns the calls that were written - with
    all samples and with a sample subset (pgenlib's proper-subset readers skip difflist groups by their byte counts) - and
    oracle/pgen.py agrees.  Covers difflists of > 32 groups and 1 / 2 / 3-byte sample ids, which the fixture does not."""
    from test_host_cpu import big_pgen_calls
    digests = {int(n): (full, part, file) for n, full, part, file in _pgenlib_digests(golden_dir, "synthetic_hardcalls.sha256")}
    for N, M, storage in ((700, 160, 5), (33333, 40, 6), (70001, 20, 2)):
        g = synthetic_calls() if N == 700 else big_pgen_calls(N, M)
        pfx = str(tmp_path / ("s%d" % N))
        types = helpers.write_pgen(pfx, g, storage=storage)
        assert set(types) >= set(range(8))
        # the writer reproduces, byte for byte, the files pgenlib validated and read back
        assert hashlib.sha256(open(pfx + ".pgen", "rb").read()).hexdigest() == digests[N][2], N
        want = g.astype(np.int8)
        want[want == 3] = -3
        sub = np.sort(np.random.default_rng(N).choice(g.shape[1], g.shape[1] // 3, replace=False))
        assert _digest(want) == digests[N][0]
        assert _digest(want[:, sub]) == digests[N][1]
        pg = pgen.Pgen(pfx + ".pgen")
        for v in (list(range(g.shape[0])) + [g.shape[0] - 1, 3, 1]):
            assert np.array_equal(pg.read(v), g[v]), (N, v)
