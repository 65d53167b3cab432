"""Step-2 statistics tiles with their genotype operand built on chip from the block's 2-bit rows.

The tensor sums of a 2-bit block are exact integer sums of the planes Z = [G; G^2; Miss] (missing calls: G = G^2 = 0,
Miss = 1) against the int8 digit rows of the feature matrix F, one set per sample chunk.  For every chunk, "s2_T" must
equal numpy's integer products of the planes decoded from "s2_gp" against "s2_FD", over the chunk ranges that "s2_paths"
reports.  The cases cover both 2-bit routes (rg_s2_block_bed, rg_s2_block_bed_bt), rows_p 128 and 1024, N not a
multiple of 16, a sample subset, missing calls, ref_first, chrX (rg_s2_set_sex adds the male columns to F), many
chunks at N ~ 20k, and 1, 2 and 5 digit groups of F.
"""
import numpy as np
import pytest

from regenie_b200 import synth

pytestmark = pytest.mark.gpu
PATH_KEYS = ("tc", "nchunk", "chunk_len", "drows", "nchunks", "Npad", "dp", "bt_dp")


def check_tensor_sums(st, bs):
    pa = dict(zip(PATH_KEYS, (int(x) for x in st.debug("s2_paths", np.int64, 8))))
    assert pa["tc"] == 1
    npad, nchunk, clen, drows = pa["Npad"], pa["nchunk"], pa["chunk_len"], pa["drows"]
    assert nchunk >= 3 and clen * (nchunk - 1) < npad <= clen * nchunk
    rp = (bs + 127) // 128 * 128
    words = st.debug("s2_gp", np.uint32, rp * (npad // 16)).reshape(rp, npad // 16)
    codes = ((words[:, :, None] >> (2 * np.arange(16, dtype=np.uint32))) & 3).reshape(rp, npad).astype(np.uint8)
    assert (codes[:bs] == 3).any()
    FD = st.debug("s2_FD", np.int8, drows * npad).reshape(drows, npad)
    T = st.debug("s2_T", np.float32, nchunk * 3 * rp * drows).reshape(nchunk, 3 * rp, drows)
    for ch in range(nchunk):
        c = codes[:, ch * clen:(ch + 1) * clen]
        g = np.where(c == 3, 0, c).astype(np.float64)
        Z = np.concatenate([g, g * g, (c == 3).astype(np.float64)])
        ref = Z @ FD[:, ch * clen:(ch + 1) * clen].astype(np.float64).T      # exact: integers far below 2^53
        assert np.array_equal(T[ch].astype(np.float64), ref), "tensor sums, chunk %d" % ch


# (route, samples in the file, kept samples, variants, traits, ref_first, chrX)
CASES = [
    ("qt", 20003, None, 100, 1, False, False),     # rows_p 128, N not a multiple of 16, one digit group of F
    ("qt", 20040, 19991, 1000, 3, True, False),    # rows_p 1024, a sample subset, two digit groups
    ("qt", 19997, None, 1000, 10, False, True),    # chrX: five digit groups with the male columns
    ("bt", 20003, None, 1000, 1, True, False),
    ("bt", 20040, 19991, 120, 3, False, True),
    ("bt", 20001, None, 900, 10, False, False),
]


@pytest.mark.parametrize("route,n_file,n_keep,bs,P,ref_first,chrx", CASES)
def test_s2_tensor_sums_exact(monkeypatch, route, n_file, n_keep, bs, P, ref_first, chrx):
    from regenie_b200 import capi
    monkeypatch.delenv("RG_B200_S2_STATS", raising=False)
    rng = np.random.default_rng(n_file + bs + P)
    C = 3
    sample_idx = None
    N = n_file
    if n_keep is not None:
        sample_idx = np.sort(rng.choice(n_file, n_keep, replace=False)).astype(np.int32)
        N = n_keep
    ia = rng.random(N) > 0.02
    X = np.asfortranarray(np.hstack([np.ones((N, 1)), rng.standard_normal((N, C - 1))]) * ia[:, None])
    mask = ia[:, None] & (rng.random((N, P)) > 0.05)
    st = capi.Step2(X, mask, ia, int(ia.sum()), 1024 if bs > 128 else 128)
    try:
        if chrx:
            st.set_sex(rng.random(N) < 0.5)
        if route == "qt":
            st.set_chr(np.asfortranarray(rng.standard_normal((N, P)) * mask), rng.uniform(0.5, 2.0, P))
        else:
            p = rng.uniform(0.2, 0.8, (N, P))
            gs = np.sqrt(p * (1 - p))
            y = (rng.random((N, P)) < p).astype(float) * mask
            st.set_chr_bt(gs * mask, gs, (y - p) / gs, [X * gs[:, [j]] for j in range(P)], y)
        g = synth.genotypes(n_file, bs, seed=n_file + P, miss=0.02)
        packed = synth.pack_bed(g)
        if route == "qt":
            st.block_bed(packed, sample_idx=sample_idx, ref_first=ref_first)
        else:
            st.block_bed_bt(packed, sample_idx=sample_idx, ref_first=ref_first)
        check_tensor_sums(st, bs)
    finally:
        st.close()
