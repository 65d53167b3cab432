"""Level-0 standardisation from the prediction kernels' own column sums.

Both prediction kernels (INT8 tensor cores up to 2 rows_p = 4096, FP64 CUDA cores beyond) write the raw predictions of
a block to the lane's scratch ("wraw") and per-128-sample-tile column sums (sum, sum of squares) beside them; one
reduction turns the tile sums into mean and 1/sd per (ridge, phenotype) column ("mean_invsd") and one pass writes
W = (wraw - mean) * invsd on the rows of real samples and 0 on layout padding.  The INT8 kernel builds its genotype
operand from the block's 2-bit rows.  Checked here, per block:
  * W is exactly (wraw - mean) * invsd on real rows and exactly 0 on padding rows, and matches the numpy oracle;
  * mean_invsd agrees with a long-double recomputation from wraw within the bound of an FP64 sum in any order;
  * the same block run twice gives bit-identical W;
at shapes that exercise the kernel's edges: two digit-row groups (Q > 50), a block size that is not a multiple of 128,
a sample count that is not a multiple of 128, removed samples, and a bsize > 2048 block on the FP64 route.
"""
import numpy as np
import pytest

import helpers
from oracle import plink
from regenie_b200 import synth

pytestmark = pytest.mark.gpu
U = 2.0 ** -53
LD = np.longdouble


def _fileset(d, N, M, P, bsize, seed, remove_n=0):
    g = synth.genotypes(N, M, seed=seed, miss=0.02)
    Y, cov, na = synth.phenotypes(g, P, 3, seed=seed, na_frac=0.03)
    prefix = helpers.write_fileset(str(d), g, Y, cov, na, n_chr=1, drop_pheno={5, N - 3}, drop_cov={11})
    keys, _ = plink.read_fam(prefix + ".fam")
    remove = set(keys[i] for i in np.random.default_rng(seed).choice(N, remove_n, replace=False)) if remove_n else None
    return helpers.Problem(prefix, str(d) + "/pheno.txt", str(d) + "/covar.txt", bsize, remove=remove)


class _DevArray:
    """A device array of FP64 values, for torch.as_tensor."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (ptr, False), "version": 3}


def _W_cols(st, b):
    """The R columns of block b of every phenotype's W, all Npad rows (padding included): [P][R][Npad]."""
    import ctypes as C
    import torch
    from regenie_b200 import capi
    st.sync()
    out = []
    for ph in range(st.P):
        ptr, ld, ncols = C.c_void_p(), C.c_int64(), C.c_int64()
        capi.check(capi.lib().rg_W_info(st.h, ph, C.byref(ptr), C.byref(ld), C.byref(ncols)))
        col = torch.as_tensor(_DevArray(ptr.value, ld.value * ncols.value), device="cuda").cpu().numpy()
        out.append(col.reshape(ncols.value, ld.value)[b * st.R:(b + 1) * st.R].copy())
    return np.stack(out)


def _check_block(pb, st, b, i8):
    pb.gpu_l0_block(st, b)
    assert st.status() == 0
    P, R, N = st.P, st.R, st.N
    paths = tuple(int(x) for x in st.debug("paths", np.int64, 3))
    assert paths[1] == (1 if i8 else 0), paths
    Npad = int(st.debug("dims", np.int64, 8)[0])
    wraw = st.debug("wraw", np.float64, P * R * Npad).reshape(P, R, Npad)
    mi = st.debug("mean_invsd", np.float64, 2 * R * P).reshape(R, P, 2)      # column q = r P + p
    W = _W_cols(st, b)
    real = np.zeros(Npad, dtype=bool)
    real[st.debug("pad_of", np.int32, N)] = True

    # W = (wraw - mean) * invsd on real rows, 0 on padding
    mean, invsd = mi[..., 0].T[:, :, None], mi[..., 1].T[:, :, None]
    assert np.array_equal(W[:, :, real], ((wraw - mean) * invsd)[:, :, real]), "W is not (wraw - mean) * invsd"
    assert not W[:, :, ~real].any(), "layout padding rows of W are not zero"
    W_o = pb.oracle_l0(b)[0]
    for ph in range(P):
        got = W[ph][:, real].T
        assert np.abs(got - W_o[ph]).max() <= 1e-9 * np.abs(W_o[ph]).max(), (b, ph)

    # mean / invsd against long double: an FP64 sum of n terms in any order is within (n - 1) u sum|terms|
    neff = pb.prep.neff.astype(LD)[None, :]
    v = wraw.transpose(1, 0, 2).astype(LD)                                  # [R][P][Npad]
    s1, s2 = v.sum(axis=2), (v * v).sum(axis=2)
    a1 = np.abs(v).sum(axis=2).astype(np.float64)
    m_ld = s1 / neff
    D = s2 - neff * m_ld * m_ld
    isd_ld = np.sqrt((neff - 1) / D)
    n = Npad + 4
    mean_bound = (n * U * a1 + U * np.abs(s1).astype(np.float64)) / neff.astype(np.float64) + 1e-300
    assert (np.abs(mi[..., 0] - m_ld.astype(np.float64)) <= mean_bound).all(), "mean outside the summation bound"
    dD = n * U * (s2 + neff * m_ld * m_ld).astype(np.float64) + 2 * neff.astype(np.float64) * np.abs(
        m_ld.astype(np.float64)) * mean_bound
    rel_bound = 0.5 * dD / D.astype(np.float64) + 8 * U
    rel_err = np.abs(mi[..., 1] - isd_ld.astype(np.float64)) / isd_ld.astype(np.float64)
    assert (rel_err <= rel_bound).all(), "1/sd outside the summation bound (%.3g)" % float((rel_err / rel_bound).max())
    return W


@pytest.mark.parametrize("N,M,P,bsize,remove_n", [
    (1500, 400, 12, 300, 0),         # Q = 60: two digit-row groups; 300 and 100 SNP blocks (rows_p 384, 128)
    (1037, 257, 3, 200, 0),          # N not a multiple of 128; 200 and 57 SNP blocks
    (1300, 300, 12, 150, 37),        # --remove: 1263 kept samples, 150-SNP blocks, two groups
])
def test_int8_route_standardises_from_its_tile_sums(tmp_path, monkeypatch, N, M, P, bsize, remove_n):
    monkeypatch.setenv("RG_B200_LANES", "2")
    pb = _fileset(tmp_path, N, M, P, bsize, 100 + N, remove_n)
    st = pb.gpu_step1()
    for b in range(len(pb.blocks)):
        _check_block(pb, st, b, i8=True)
    W1 = _W_cols(st, 0)
    pb.gpu_l0_block(st, 0)                        # the same block again, on the other lane
    assert st.status() == 0
    assert np.array_equal(_W_cols(st, 0), W1), "a rerun of the block changed W"
    st.close()


def test_fp64_route_above_2048_standardises_from_its_tile_sums(tmp_path, monkeypatch):
    monkeypatch.setenv("RG_B200_LANES", "2")
    pb = _fileset(tmp_path, 900, 2200, 2, 2200, 7)
    st = pb.gpu_step1()
    W1 = _check_block(pb, st, 0, i8=False)
    pb.gpu_l0_block(st, 0)
    assert st.status() == 0
    assert np.array_equal(_W_cols(st, 0), W1), "a rerun of the block changed W"
    st.close()
