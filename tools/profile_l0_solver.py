"""Kernel times of the level-0 mixed-precision solver on the bench.py workload, one lane, next to the bytes its GEMM
launches move.

    python tools/profile_l0_solver.py [--blocks 20] [--passes 2]

Runs blocks of BASELINE.json configs[1] (N = 100k, bsize 1000, 10 traits, 5 folds x 5 ridge values) through a handle
with a single lane, so kernels do not share the GPU with other blocks, first under torch.profiler and then with the
library's CUDA-event timers on.  Prints the GPU time per block of every solver kernel; the 3xTF32 GEMM launches are
split into update launches (P_ik = A_ik - L_i,0:k L_k,0:k^T) and TRSM launches (L_ik = P_ik M_k^T) by their place in
the stream: the GEMM launch right behind a potrf128 launch is the TRSM of that panel step.  The operand and output
bytes of those launches are COUNTED from the tile lists of chol_mixed.cu's build_plan, not measured (DRAM counters
cannot be read here); bytes over time is therefore the rate the kernel asks of the memory system, to be set against
the H100 SXM data-sheet 3.35 TB/s of HBM3.  Run it in a process of its own.
"""
import argparse
import collections
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["RG_B200_LANES"] = "1"

SOLVER = ("tf32x3_gemm_nt", "potrf128", "mx_trisolve", "mx_residual_fused", "mx_residual_kernel", "mx_final_check",
          "l0_assemble_sym", "l0_rhs_sym")
TILE = 128 * 128 * 4          # one 128 x 128 FP32 tile
CHUNK = 128 * 32 * 4          # one operand tile of one K chunk (32 floats x 128 rows)


def gemm_bytes(n, nmat, first_col_ready=True):
    """(operand bytes, output bytes) of the update and the TRSM launches of one solve, from the tile lists."""
    nt = n // 128
    upd_in = upd_out = trsm_in = trsm_out = 0
    for k in range(nt):
        if not (k == 0 and first_col_ready):
            tiles = nt - k
            upd_in += tiles * (4 * CHUNK + 4 * k * 2 * CHUNK)      # 4 C chunks (the identity is built on chip) + A, B chunks
            upd_out += tiles * TILE
        tiles = nt - k - 1
        trsm_in += tiles * 4 * 2 * CHUNK
        trsm_out += tiles * 2 * TILE                               # the tile and its mirror image
    return {"update": (upd_in * nmat, upd_out * nmat), "trsm": (trsm_in * nmat, trsm_out * nmat)}


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
    st = capi.Step1(X, Y, mask, in_an, hostprep.fold_sizes(N, K), lam, neff, N, bs, len(blocks), device=0)

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
    evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    evs.sort(key=lambda e: e.time_range.start)
    after_potrf = False
    for e in evs:
        short = e.name.split("(")[0].replace("void ", "").replace("rg::", "")
        if "potrf128" in short:
            after_potrf = True
        elif "tf32x3_gemm_nt" in short:
            short = "tf32x3_gemm_nt [trsm]" if after_potrf else "tf32x3_gemm_nt [update]"
            after_potrf = False
        per[short] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        cnt[short] += 1
    nb = args.passes * len(blocks)
    n = 128
    while n < bs:
        n *= 2
    mixed, fallbacks = st.solver_stats()
    print("# %s; %d blocks of %d SNPs (n = %d, %d systems), N = %d, %d traits, one lane: GPU time per block (us)"
          % (torch.cuda.get_device_name(0), nb, bs, n, K * R, N, P))
    print("# blocks on the mixed solver: %d, re-solved in FP64: %d" % (mixed, fallbacks))
    solver_total = other = 0.0
    gemm_us = {}
    for name, us in sorted(per.items(), key=lambda kv: -kv[1]):
        if any(k in name for k in SOLVER):
            print("%-36s %9.1f us  %6.2f launches" % (name[:36], us / nb, cnt[name] / nb))
            solver_total += us / nb
            if "[update]" in name:
                gemm_us["update"] = us / nb
            if "[trsm]" in name:
                gemm_us["trsm"] = us / nb
        else:
            other += us / nb
    print("%-36s %9.1f us" % ("solver kernels", solver_total))
    print("%-36s %9.1f us" % ("all other kernels", other))
    print("# bytes per block counted from the tile lists (not measured), and the rate they imply over the kernel time")
    for kind, (b_in, b_out) in gemm_bytes(n, K * R).items():
        us = gemm_us.get(kind, 0.0)
        rate = (b_in + b_out) / (us * 1e-6) / 1e12 if us > 0 else float("nan")
        print("%-36s operands %7.1f MB  outputs %6.1f MB  -> %5.2f TB/s asked for (HBM3 data sheet: 3.35 TB/s)"
              % ("tf32x3_gemm_nt [%s]" % kind, b_in / 1e6, b_out / 1e6, rate))

    st.set_timing(True)
    one_pass()
    ms, nblk = st.timing("mx_solve")
    print("%-36s %9.3f ms per %d blocks (CUDA events around the phase, one lane)" % ("mx_solve timer", ms, nblk))
    st.set_timing(False)
    st.close()


if __name__ == "__main__":
    main()
