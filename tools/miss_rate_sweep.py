"""Level-0 pass time against the missing-call rate, with the Miss rows of the Gram as dense tensor-core tiles
(RG_B200_GRAM=dense) and as sparse sums over the missing lists (RG_B200_GRAM=sparse): the crossover sets
kMissSparseRate (csrc/kernels.cuh, DESIGN.md section 3).

    python tools/miss_rate_sweep.py [--blocks 12] [--passes 3] [--out sweep.json]

The benchmark's shape (N = 100k, bsize 1000, 10 traits, 5 folds) on --blocks blocks, through the C ABI with device
rows.  Prints ms per pass on the default lanes and the single-lane `gram_wgmma` timer (which holds the list, transpose
and sparse kernels too), per block.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from regenie_b200 import capi, hostprep  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=12)
    ap.add_argument("--passes", type=int, default=3)
    ap.add_argument("--rates", default="0,0.005,0.01,0.02,0.04,0.08,0.16")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    dev = torch.device("cuda", 0)
    c = bench.CFG
    N, bs, P, C, K, R = c["N"], c["bsize"], c["P"], c["C"], c["K"], c["R"]
    nb = args.blocks
    M = nb * bs
    Yr, cov, na = bench.gen_pheno(N, P, C, bench.SEED)
    X, Y, mask, in_an, neff = hostprep.prepare_qt(Yr, cov, na)
    fsz = hostprep.fold_sizes(N, K)
    h = hostprep.ridge_grid(R)
    lam = c["M"] * (1 - h) / h
    print("%s, N=%d, bsize=%d, %d blocks, %d traits" % (torch.cuda.get_device_name(0), N, bs, nb, P), flush=True)
    rows = []
    for rate in [float(x) for x in args.rates.split(",")]:
        panel = bench.gen_panel_gpu(torch, N, M, bs, bench.SEED + 1, dev, rate)
        stride = panel.shape[1]
        ptr = panel.data_ptr()
        torch.cuda.synchronize()
        rec = {"miss_rate": rate}
        for mode in ("dense", "sparse"):
            os.environ["RG_B200_GRAM"] = mode
            st = capi.Step1(X, Y, mask, in_an, fsz, lam, neff, N, bs, nb, device=0)
            ext = torch.cuda.ExternalStream(st.stream(), device=dev)

            def one_pass(handle):
                for b in range(nb):
                    handle.l0_block_bed(ptr + b * bs * stride, bs, b, row_stride=stride)

            one_pass(st)
            st.sync()
            assert st.status() == 0, capi.lib().rg_last_error().decode()
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(ext)
            for _ in range(args.passes):
                one_pass(st)
            st.fence()
            e1.record(ext)
            e1.synchronize()
            assert st.status() == 0, capi.lib().rg_last_error().decode()
            rec[mode + "_ms_per_pass"] = e0.elapsed_time(e1) / args.passes
            st.close()
            os.environ["RG_B200_LANES"] = "1"
            st1 = capi.Step1(X, Y, mask, in_an, fsz, lam, neff, N, bs, nb, device=0)
            os.environ.pop("RG_B200_LANES")
            one_pass(st1)
            st1.sync()
            st1.set_timing(True)
            one_pass(st1)
            st1.sync()
            t, n = st1.timing("gram_wgmma")
            rec[mode + "_gram_us_per_block"] = 1e3 * t / max(n, 1)
            st1.close()
        os.environ.pop("RG_B200_GRAM", None)
        del panel
        rows.append(rec)
        print("miss %5.3f  ms/pass dense %7.2f sparse %7.2f (%+.1f %%)   single-lane Gram us/block dense %7.1f sparse %7.1f"
              % (rate, rec["dense_ms_per_pass"], rec["sparse_ms_per_pass"],
                 100 * (rec["dense_ms_per_pass"] / rec["sparse_ms_per_pass"] - 1),
                 rec["dense_gram_us_per_block"], rec["sparse_gram_us_per_block"]), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(rows, fh, indent=1)


if __name__ == "__main__":
    main()
