"""GPU parity: level-0 ridge (k-fold) through the C ABI vs the numpy oracle.

Tolerance: the north_star asks for 1e-5 relative on the final statistics; the level-0 predictors
are FP64 end to end (integer Grams are exact), so we hold them to 1e-9 relative here.
"""
import numpy as np
import pytest

import helpers

pytestmark = pytest.mark.gpu
TOL = 1e-9


def rel(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def run_blocks(pb):
    st = pb.gpu_step1()
    out = []
    for b in range(len(pb.blocks)):
        pb.gpu_l0_block(st, b)
        assert st.status() == 0
        out.append([st.fetch_W(b, ph) for ph in range(pb.prep.Y.shape[1])])
    return st, out


@pytest.mark.parametrize("N,M,bs,miss,P,K", [(1000, 300, 128, 0.02, 3, 5), (777, 150, 100, 0.0, 3, 5), (2051, 130, 130, 0.05, 3, 5),
                                            # ragged edges: N not a multiple of 4, one phenotype (strict mode), 3 uneven folds,
                                            # chromosomes whose last block holds a single SNP (M = 3 * 43, bsize 42)
                                            (203, 129, 42, 0.03, 1, 3)])
def test_l0_kfold_matches_oracle(tmp_path, N, M, bs, miss, P, K):
    pb = helpers.synthetic_problem(tmp_path, N=N, M=M, bsize=bs, miss=miss, P=P, K=K)
    assert N != 203 or min(b[2] for b in pb.blocks) == 1
    st, out = run_blocks(pb)
    for b in range(len(pb.blocks)):
        W_o, mu_o, sd_o, _ = pb.oracle_l0(b)
        for ph in range(len(W_o)):
            assert rel(out[b][ph], W_o[ph]) < TOL


def test_integer_gram_is_exact(tmp_path):
    """wgmma int8 Gram == CUDA-core integer Gram == numpy integer Gram, bit for bit."""
    pb = helpers.synthetic_problem(tmp_path, N=1500, M=256, bsize=256, miss=0.03)
    st = pb.gpu_step1()
    pb.gpu_l0_block(st, 0)
    assert st.status() == 0
    Npad, rp, nC, n_aug, nmat, K, cpp, nch = [int(x) for x in st.debug("dims", np.int64, 8)]
    zz = st.debug("zz", np.float32, K * 4 * rp * rp).reshape(K, 2 * rp, 2 * rp)
    zr = st.debug("zz_ref", np.float32, K * 4 * rp * rp).reshape(K, 2 * rp, 2 * rp)
    tri = np.tril(np.ones((2 * rp, 2 * rp), dtype=bool))
    assert np.array_equal(zz[:, tri], zr[:, tri])
    # numpy: G0 and Miss planes of fold 0 from the raw calls
    from oracle import plink
    c, s, bs = pb.blocks[0]
    g = plink.decode_bed(pb.packed[s:s + bs], pb.n_file)
    g = np.where(pb.prep.in_analysis[None, :], g, 0.0)
    f0 = slice(0, int(pb.fold_sizes[0]))
    G0 = np.where(g[:, f0] == -3, 0, g[:, f0]); Mi = (g[:, f0] == -3).astype(float)
    assert np.array_equal(np.tril(zz[0, :bs, :bs]), np.tril(G0 @ G0.T))
    assert np.array_equal(zz[0, rp:rp + bs, :bs], Mi @ G0.T)
    assert np.array_equal(np.tril(zz[0, rp:rp + bs, rp:rp + bs]), np.tril(Mi @ Mi.T))


def test_l0_sample_subset_and_shard_invariance(tmp_path):
    """--remove style sample subsetting (sample_idx) and block-order independence: the reference
    pins sharded == unsharded byte-for-byte (test/test_bash.sh:127-137)."""
    g_dir = tmp_path / "a"
    pb = helpers.synthetic_problem(g_dir, N=900, M=260, bsize=130, miss=0.01)
    keys_file, _ = __import__("oracle.plink", fromlist=["x"]).read_fam(str(g_dir) + "/syn.fam")
    remove = {keys_file[3], keys_file[400], keys_file[899]}
    pb2 = helpers.Problem(str(g_dir) + "/syn", str(g_dir) + "/pheno.txt", str(g_dir) + "/covar.txt", 130,
                          remove=remove)
    st, out = run_blocks(pb2)
    for b in range(len(pb2.blocks)):
        W_o, _, _, _ = pb2.oracle_l0(b)
        for ph in range(len(W_o)):
            assert rel(out[b][ph], W_o[ph]) < TOL
    # reversed block order on a fresh handle gives bit-identical predictors
    st2 = pb2.gpu_step1()
    for b in reversed(range(len(pb2.blocks))):
        pb2.gpu_l0_block(st2, b)
    assert st2.status() == 0
    for b in range(len(pb2.blocks)):
        for ph in range(pb2.prep.Y.shape[1]):
            assert np.array_equal(st2.fetch_W(b, ph), out[b][ph])


@pytest.mark.parametrize("lanes", ["2", "8"])
def test_many_blocks_per_lane_from_host_rows(tmp_path, monkeypatch, lanes):
    """Host rows go through two staging buffers per lane, filled on the lane's copy stream ahead of the lane's kernels:
    with 40 blocks on 2 (and 8) lanes every buffer is reused many times while earlier blocks are still in flight; every
    block must still match the oracle, and a run from one big device-resident... host array must equal a run that hands
    over the same bytes block by block from a buffer that is overwritten right after rg_l0_wait_input."""
    monkeypatch.setenv("RG_B200_LANES", lanes)
    pb = helpers.synthetic_problem(tmp_path, N=700, M=640, P=2, C=3, bsize=16, miss=0.02)
    st, out = run_blocks(pb)
    for b in range(len(pb.blocks)):
        W_o, _, _, _ = pb.oracle_l0(b)
        for ph in range(len(W_o)):
            assert rel(out[b][ph], W_o[ph]) < TOL, b
    st.close()


def test_l0_example_fileset(golden_dir):
    """The reference's own example/ fileset (500 x 1000, 2 QTs), --bsize 100."""
    pb = helpers.Problem(golden_dir + "/example", golden_dir + "/phenotype.txt", golden_dir + "/covariates.txt", 100)
    st, out = run_blocks(pb)
    for b in (0, 4, 9):
        W_o, _, _, _ = pb.oracle_l0(b)
        for ph in range(2):
            assert rel(out[b][ph], W_o[ph]) < TOL


def test_low_variance_snp_is_reported(tmp_path):
    """Monomorphic SNP -> error like the reference (src/Data.cpp:205-209)."""
    from regenie_b200 import synth
    g = synth.genotypes(600, 64, seed=3, miss=0.0)
    g[10] = 1
    Y, cov, na = synth.phenotypes(g, 2, 3, seed=3)
    prefix = helpers.write_fileset(str(tmp_path), g, Y, cov, na)
    pb = helpers.Problem(prefix, str(tmp_path) + "/pheno.txt", str(tmp_path) + "/covar.txt", 64)
    st = pb.gpu_step1()
    pb.gpu_l0_block(st, 0)
    assert st.status() == 11   # 1 + SNP index


def test_poll_status_reads_the_sticky_word_without_draining(tmp_path):
    """rg_l0_poll_status: 0 while nothing was flagged, and - once the block that holds the monomorphic SNP has run - the
    same word rg_l0_status returns; polling between blocks must not disturb the results."""
    from regenie_b200 import synth
    pb = helpers.synthetic_problem(tmp_path, N=900, M=192, P=2, bsize=64, miss=0.01)
    st = pb.gpu_step1()
    for b in range(len(pb.blocks)):
        pb.gpu_l0_block(st, b)
        assert st.poll_status() == 0
    assert st.status() == 0 and st.poll_status() == 0
    W_o, _, _, _ = pb.oracle_l0(1)
    assert rel(st.fetch_W(1, 0), W_o[0]) < TOL
    st.close()
    g = synth.genotypes(600, 64, seed=3, miss=0.0)
    g[10] = 1
    Y, cov, na = synth.phenotypes(g, 2, 3, seed=3)
    d = tmp_path / "mono"; d.mkdir()
    prefix = helpers.write_fileset(str(d), g, Y, cov, na)
    pb2 = helpers.Problem(prefix, str(d) + "/pheno.txt", str(d) + "/covar.txt", 64)
    st2 = pb2.gpu_step1()
    pb2.gpu_l0_block(st2, 0)
    st2.fence()
    import torch
    torch.cuda.synchronize()
    assert st2.poll_status() == 11 and st2.status() == 11
