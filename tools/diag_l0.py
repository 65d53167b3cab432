"""GPU diagnostic: stage-by-stage comparison of one level-0 block against the oracle."""
import sys, os, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import helpers


def rel(a, b):
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-300))


def main():
    N = int(sys.argv[1]) if len(sys.argv) > 1 else 1000
    M = int(sys.argv[2]) if len(sys.argv) > 2 else 300
    bs = int(sys.argv[3]) if len(sys.argv) > 3 else 128
    pb = helpers.synthetic_problem("/tmp/diag_syn", N=N, M=M, bsize=bs)
    pr = pb.prep
    st = pb.gpu_step1()
    st.set_timing(True)
    for b in range(len(pb.blocks)):
        t0 = time.time()
        pb.gpu_l0_block(st, b)
        code = st.status()
        print("block", b, "status", code, "wall %.3fs" % (time.time() - t0), flush=True)
        dims = st.debug("dims", np.int64, 8)
        Npad, rp, nC, n_aug, nmat, K, cpp, nch = [int(x) for x in dims]
        bsz = pb.blocks[b][2]
        zz = st.debug("zz", np.float32, K * 4 * rp * rp).reshape(K, 2 * rp, 2 * rp)
        zr = st.debug("zz_ref", np.float32, K * 4 * rp * rp).reshape(K, 2 * rp, 2 * rp)
        tri = np.tril(np.ones((2 * rp, 2 * rp), dtype=bool))
        d = np.abs(zz - zr)[:, tri]
        print("  gram wgmma vs cuda-core ref: max abs diff", d.max(), " ref max", zr.max(), " nonzero frac", (zz[:, tri] != 0).mean())
        if d.max() != 0:
            bad = np.argwhere(np.abs(zz - zr) * tri[None] > 0)
            print("  first bad entries", bad[:10], "count", len(bad))
            for (f, i, j) in bad[:5]:
                print("   ", f, i, j, zz[f, i, j], zr[f, i, j])
        # numpy integer gram for fold 0
        gi, mu_o = pb.oracle_block(b)
        W_o, mu_o, sd_o, Gt = pb.oracle_l0(b)
        mu = st.debug("mu", np.float64, rp)[:bsz]
        isd = st.debug("inv_sd", np.float64, rp)[:bsz]
        print("  mu rel", rel(mu, mu_o), " sd rel", rel(1 / isd, sd_o))
        # rhs vs oracle
        starts = np.concatenate([[0], np.cumsum(pb.fold_sizes)])
        GtY = [Gt[:, starts[f]:starts[f + 1]] @ pr.Y[starts[f]:starts[f + 1]] for f in range(K)]
        GTY = sum(GtY)
        rhs = st.debug("rhs", np.float64, K * rp * pr.Y.shape[1]).reshape(K, rp, -1)[:, :bsz]
        print("  rhs rel", max(rel(rhs[f], GTY - GtY[f]) for f in range(K)))
        cm = st.debug("cm", np.float64, nmat * n_aug * nC).reshape(nmat, n_aug, nC)
        GG = [Gt[:, starts[f]:starts[f + 1]] @ Gt[:, starts[f]:starts[f + 1]].T for f in range(K)]
        GGt = sum(GG)
        R = len(pb.lam)
        errs = []
        for f in range(K):
            for r in range(R):
                beta_o = np.linalg.solve(GGt - GG[f] + pb.lam[r] * np.eye(bsz), GTY - GtY[f])
                beta = cm[f * R + r, nC:nC + pr.Y.shape[1], :bsz].T
                errs.append(rel(beta, beta_o))
        print("  beta rel (max over f,r)", max(errs))
        for ph in range(pr.Y.shape[1]):
            W = st.fetch_W(b, ph)
            print("  W ph", ph, "rel", rel(W, W_o[ph]))
    for k in ["h2d", "bed_relayout", "l0_stats", "gram_wgmma", "l0_assemble", "chol_factor",
              "chol_backsolve", "l0_predict"]:
        ms, n = st.timing(k)
        print("  time %-16s %8.3f ms over %d" % (k, ms, n))
    print("launches", st.launch_count())


if __name__ == "__main__":
    main()
