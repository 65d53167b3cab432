"""The Step-1 relayout pass that writes the 2-bit rows, the sample-major rows and the per-(SNP row, column tile) missing
lists in one go (bed_kernels.cu, launch_bed_relayout_miss), and the sparse Miss sums that read them (miss_gram.cu).

Against the forced-dense run (RG_B200_GRAM=dense: 2-bit rows only, the Miss rows as tensor-core tiles) every block must
give bit-identical gp, zz, tstat and W; zz must also equal the CUDA-core reference Gram, and the lists must hold exactly
the missing calls numpy decodes from the same packed rows.
"""
import numpy as np
import pytest

import helpers
from oracle import plink
from regenie_b200 import synth

pytestmark = pytest.mark.gpu


def dense_tile_mask(rp):
    """Entries of one fold's [2 rp][2 rp] Gram that gram_tile_list's 128 x 256 tiles write."""
    m = np.zeros((2 * rp, 2 * rp), dtype=bool)
    for nj in range(2 * rp // 256):
        for mi in range(2 * nj, 2 * rp // 128):
            m[128 * mi:128 * mi + 128, 256 * nj:256 * nj + 256] = True
    return m


def make_problem(tmp, g, bs, K, remove=None):
    Y, cov, na = synth.phenotypes(g, 3, 3, seed=7, na_frac=0.03)
    prefix = helpers.write_fileset(str(tmp), g, Y, cov, na, n_chr=1)
    return helpers.Problem(prefix, str(tmp) + "/pheno.txt", str(tmp) + "/covar.txt", bs, K=K, remove=remove)


def expected_missing(pb, b, ref_first):
    """Per block row: the padded-layout positions of its missing calls among the analysed samples."""
    _, s, bs = pb.blocks[b]
    g = plink.decode_bed(pb.packed[s:s + bs], pb.n_file, keep=pb.keep, ref_first=ref_first)
    pad_of = np.asarray(pb.prep_pad_of)
    miss = (g == -3) & pb.prep.in_analysis[None, :]
    return [set(pad_of[np.nonzero(miss[i])[0]].tolist()) for i in range(bs)]


def check_lists(pb, st, b, ref_first):
    """Every (row, column tile) segment holds exactly the row's missing calls inside the tile's words."""
    Npad, rp = [int(x) for x in st.debug("dims", np.int64, 8)[:2]]
    ctile = st.debug("miss_ctile", np.int32, 4 * (Npad // 16)).reshape(-1, 4)
    nct = len(ctile)
    assert ctile[0, 0] == 0 and (ctile[1:, 0] == ctile[:-1, 0] + ctile[:-1, 1]).all()
    assert ctile[-1, 0] + ctile[-1, 1] == Npad // 16 and (ctile[:, 1] <= 32).all()
    cut = np.concatenate([[0], np.cumsum(pb.fold_pad_len)]) // 16
    for f in range(len(cut) - 1):
        own = ctile[ctile[:, 2] == f]
        assert own[0, 0] == cut[f] and own[-1, 0] + own[-1, 1] == cut[f + 1]
    _, total, cap = [int(x) for x in st.debug("gram_path", np.int64, 3)]
    seg = st.debug("miss_seg", np.int32, rp * nct * 2).reshape(rp, nct, 2)
    lst = st.debug("miss_list", np.int32, max(cap, 1))
    exp = expected_missing(pb, b, ref_first)
    assert seg[:, :, 1].sum() == total
    for i in range(rp):
        want = exp[i] if i < len(exp) else set()
        got = []
        for ct in range(nct):
            off, cnt = seg[i, ct]
            part = lst[off:off + cnt]
            lo, hi = 16 * ctile[ct, 0], 16 * (ctile[ct, 0] + ctile[ct, 1])
            assert ((part >= lo) & (part < hi)).all()
            got.extend(part.tolist())
        assert len(got) == len(set(got)) and set(got) == want, "row %d" % i


def run(pb, mode, monkeypatch, ref_first=False, lanes=None, check=None):
    """Level 0 over every block with RG_B200_GRAM=mode ("dense", or unset); per block gp, zz, tstat, W and check()."""
    if mode == "dense":
        monkeypatch.setenv("RG_B200_GRAM", "dense")
    else:
        monkeypatch.delenv("RG_B200_GRAM", raising=False)
    if lanes:
        monkeypatch.setenv("RG_B200_LANES", str(lanes))
    st = pb.gpu_step1()
    out = []
    for b, (_, s, bs) in enumerate(pb.blocks):
        idx = None if pb.keep.all() else pb.sample_idx
        st.l0_block_bed(pb.packed[s:s + bs], bs, b, sample_idx=idx, ref_first=ref_first)
        assert st.status() == 0
        Npad, rp, _, _, _, K, _, _ = [int(x) for x in st.debug("dims", np.int64, 8)]
        paths = st.debug("paths", np.int64, 3)
        r = {"gp": st.debug("gp", np.uint32, rp * Npad // 16),
             "zz": st.debug("zz", np.float32, K * 4 * rp * rp).reshape(K, 2 * rp, 2 * rp),
             "path": [int(x) for x in st.debug("gram_path", np.int64, 3)]}
        if paths[0]:
            r["tstat"] = st.debug("tstat", np.float32, K * 2 * rp * 1024)   # [K][2 rp][digit rows]
        zr = st.debug("zz_ref", np.float32, r["zz"].size).reshape(r["zz"].shape)
        tri = np.tril(np.ones((2 * rp, 2 * rp), dtype=bool))
        assert np.array_equal(r["zz"][:, tri], zr[:, tri])
        if check:
            check(st, b, r)
        out.append(r)
    st.sync()
    for b, r in enumerate(out):
        r["W"] = [st.fetch_W(b, ph) for ph in range(pb.prep.Y.shape[1])]
    return out


# (N, M, bs, missing rate, folds, --remove subset, ref_first, lanes, sparse path expected)
CASES = [
    (1203, 390, 130, 0.0, 5, False, 0, None, True),       # N not a multiple of 16, bs not of 128, uneven folds
    (1500, 600, 200, 0.005, 5, True, 0, None, True),      # --remove holes: non-contiguous words
    (1500, 600, 200, 0.01, 3, False, 1, None, True),      # ref_first
    (2100, 700, 256, 0.01, 4, True, 1, 2, True),          # more blocks than lanes; the last block is short
    (1203, 260, 130, 0.0135, 5, False, 0, None, True),    # just under the list capacity (1.5 % of bs x N)
    (1203, 260, 130, 0.03, 5, False, 0, None, False),     # over it: the dense Miss tiles in the same run
]


@pytest.mark.parametrize("N,M,bs,miss,K,subset,ref_first,lanes,sparse", CASES)
def test_fused_relayout_matches_dense(tmp_path, monkeypatch, N, M, bs, miss, K, subset, ref_first, lanes, sparse):
    g = synth.genotypes(N, M, seed=31, miss=miss)
    remove = None
    if subset:
        keys, _ = plink.read_fam(helpers.write_fileset(str(tmp_path / "k"), g[:1], np.zeros((N, 1)), np.zeros((N, 1)),
                                                       np.zeros((N, 1), bool)) + ".fam")
        remove = {keys[5], keys[17], keys[18], keys[300], keys[N // 2], keys[N - 2]}
    pb = make_problem(tmp_path, g, bs, K, remove=remove)
    pb.prep_pad_of = None
    pb.fold_pad_len = [-(-int(n) // 256) * 256 for n in pb.fold_sizes]
    dense = run(pb, "dense", monkeypatch, ref_first=bool(ref_first), lanes=lanes)

    def check(st, b, r):
        if pb.prep_pad_of is None:
            pb.prep_pad_of = st.debug("pad_of", np.int32, len(pb.prep.in_analysis))
        sparse_path, total, cap = r["path"]
        assert sparse_path == int(sparse) and (total <= cap) == sparse
        if sparse:
            check_lists(pb, st, b, bool(ref_first))

    fused = run(pb, "auto", monkeypatch, ref_first=bool(ref_first), lanes=lanes, check=check)
    for b, (d, f) in enumerate(zip(dense, fused)):
        assert d["path"][1] == -1
        assert np.array_equal(d["gp"], f["gp"]), "block %d" % b
        m = dense_tile_mask(d["zz"].shape[1] // 2)
        assert np.array_equal(d["zz"][:, m], f["zz"][:, m]), "block %d" % b
        assert ("tstat" in d) == ("tstat" in f)
        if "tstat" in d:
            assert np.array_equal(d["tstat"], f["tstat"])
        for x, y in zip(d["W"], f["W"]):
            assert np.array_equal(x, y)
