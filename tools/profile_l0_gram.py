"""Kernel times of the level-0 Gram phase on the bench.py workload, one lane.

    python tools/profile_l0_gram.py [--blocks 20] [--passes 2]

Runs blocks of BASELINE.json configs[1] (N = 100k, bsize 1000, 1 % missing calls, 5 folds) through a handle with a
single lane, first under torch.profiler and then with the library's CUDA-event timers on, once with the Miss rows of the
Gram as sparse sums (the default below kMissSparseRate) and once as dense tiles (RG_B200_GRAM=dense).  Prints the GPU
time per block of every kernel inside the `gram_wgmma` timer (missing lists, transpose, Gram tiles, sparse sums), the
other kernels as one line, and the timer itself.  Run it in a process of its own.
"""
import argparse
import collections
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["RG_B200_LANES"] = "1"

GRAM = ("bed_relayout", "miss_list", "miss_transpose", "gram_s8_wgmma", "miss_sparse", "Memset")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=20)
    ap.add_argument("--passes", type=int, default=2)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    from regenie_b200 import capi, hostprep

    c = bench.CFG
    N, bs, P, C, K, R = c["N"], c["bsize"], c["P"], c["C"], c["K"], c["R"]
    M = args.blocks * bs
    blocks = bench.blocks_of(M, bs)
    dev = torch.device("cuda", 0)
    Yr, cov, na = bench.gen_pheno(N, P, C, bench.SEED)
    X, Y, mask, in_an, neff = hostprep.prepare_qt(Yr, cov, na)
    h = hostprep.ridge_grid(R)
    lam = M * (1 - h) / h
    panel = bench.gen_panel_gpu(torch, N, M, bs, bench.SEED + 1000, dev, c["miss"])
    stride = panel.shape[1]
    print("# %s; %d blocks of %d SNPs, N = %d, %d traits, one lane: GPU time per block (us)"
          % (torch.cuda.get_device_name(0), args.passes * len(blocks), bs, N, P))
    for mode in ("auto", "dense"):
        if mode == "dense":
            os.environ["RG_B200_GRAM"] = "dense"
        st = capi.Step1(X, Y, mask, in_an, hostprep.fold_sizes(N, K), lam, neff, N, bs, len(blocks), device=0)
        os.environ.pop("RG_B200_GRAM", None)

        def one_pass():
            for b, (s, n) in enumerate(blocks):
                st.l0_block_bed(panel.data_ptr() + s * stride, n, b, row_stride=stride)
            st.sync()
            assert st.status() == 0, capi.lib().rg_last_error().decode()

        one_pass()                                   # warm-up: allocations, tensor maps, module load
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.passes):
                one_pass()
        per = collections.defaultdict(float)
        cnt = collections.Counter()
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                per[e.name] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
                cnt[e.name] += 1
        nb = args.passes * len(blocks)
        path = int(st.debug("gram_path", "int64", 3)[0])
        print("## RG_B200_GRAM=%s (Miss rows: %s)" % (mode, "sparse" if path else "dense tiles"))
        other = 0.0
        for name, us in sorted(per.items(), key=lambda kv: -kv[1]):
            short = name.split("(")[0].replace("void ", "").replace("rg::", "")
            if any(k in short for k in GRAM):
                print("%-28s %9.1f us  %5.2f launches" % (short[:28], us / nb, cnt[name] / nb))
            else:
                other += us / nb
        print("%-28s %9.1f us" % ("all other kernels", other))
        st.set_timing(True)
        one_pass()
        for timer in ("bed_relayout", "gram_wgmma"):
            ms, n = st.timing(timer)
            print("%-28s %9.1f us per block (CUDA events, %d blocks)" % (timer + " timer", 1e3 * ms / max(n, 1), n))
        st.set_timing(False)
        st.close()


if __name__ == "__main__":
    main()
