"""Time the GxE interaction routes (rg_s2_interaction, or with --bt rg_s2_interaction_bt / rg_s2_interaction_firth)
against the plain Step-2 block on the same data.

One block of `--bs` synthetic hard-call variants, P traits, C covariate columns, for each N in `--n`:
  plain    rg_s2_block_bed alone (no interaction state)
  hlm      rg_s2_block_bed + rg_s2_interaction, every variant on the HLM route (rare_mac above every MAC)
  robust   rg_s2_block_bed + rg_s2_interaction with --force-robust (HC3)
  cpu      the numpy restatement (tests/interaction_oracle.py) of the robust route on a few variants, per variant
With --bt, binary traits (about 20 % cases) and the basis of [1, covariates, E, E^2]:
  plain    rg_s2_block_bed_bt alone
  wald     rg_s2_block_bed_bt + rg_s2_interaction_bt (default routes: HC3 where MAC > 1000 and a Wald p < 0.05)
  robust   the same with --force-robust
  firth    rg_s2_block_bed_bt + rg_s2_interaction_bt + rg_s2_interaction_firth on the pairs whose GxE Wald p-value is at
           most --pthresh (the Firth time is also given per pair)
  cpu      tests/interaction_bt_oracle.py: the Wald route per variant and the Firth fits per pair
The block calls return with their results on the host, so a host clock around each call times the whole call.
Prints one JSON line; with --out also writes it to that file.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def best_of(fn, reps):
    fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return min(t) * 1e3


def one_size(N, bs, P, C, reps, cpu_variants):
    from regenie_b200 import capi
    import interaction_oracle as io
    rng = np.random.default_rng(1)
    X, _ = np.linalg.qr(np.column_stack([np.ones(N), rng.normal(size=(N, C - 1))]))
    mask = np.ones((N, P), dtype=np.uint8)
    res = rng.normal(size=(N, P))
    res -= X @ (X.T @ res)
    scf = np.ones(P)
    E = rng.normal(size=N)
    maf = rng.uniform(0.05, 0.5, bs)
    g = rng.binomial(2, maf[:, None], (bs, N))
    code = np.where(g == 2, 0, np.where(g == 1, 2, 3)).astype(np.uint8)     # ref-last .bed codes of the A1 count
    pad = (-N) % 4
    code = np.concatenate([code, np.zeros((bs, pad), dtype=np.uint8)], axis=1).reshape(bs, -1, 4)
    rows = (code[..., 0] | code[..., 1] << 2 | code[..., 2] << 4 | code[..., 3] << 6).astype(np.uint8)
    st = capi.Step2(X, mask, np.ones(N, dtype=np.uint8), N, bs)
    st.set_chr(res, scf)
    out = {"N": N, "bs": bs, "P": P, "C": C}
    out["plain_ms"] = best_of(lambda: st.block_bed(rows, min_mac=5.0), reps)
    K = C + 2
    d = np.exp(rng.normal(size=(N, P)) * 0.1)
    px = [np.linalg.qr(rng.normal(size=(N, K)) * d[:, [p]])[0] for p in range(P)]
    yres = rng.normal(size=(N, P))
    st.set_interaction(E, d, px, yres)

    def run(**kw):
        st.block_bed(rows, min_mac=5.0)
        return st.interaction(bs, min_mac=5.0, **kw)

    s_hlm = run(rare_mac=1e15)[0]
    s_rob = run(force_robust=True)[0]
    out["hlm_ms"] = best_of(lambda: run(rare_mac=1e15), reps)
    out["robust_ms"] = best_of(lambda: run(force_robust=True), reps)
    out["routes_ok"] = bool((s_hlm == 2).all() and (s_rob == 1).all())
    t0 = time.perf_counter()
    mac = np.full(P, 1e9)
    for v in range(cpu_variants):
        io.robust(g[v].astype(float), E, X, res, mask.astype(float), scf, N, mac)
    out["cpu_robust_ms_per_variant"] = (time.perf_counter() - t0) * 1e3 / cpu_variants
    out["cpu_robust_ms_per_block"] = out["cpu_robust_ms_per_variant"] * bs
    st.close()
    return out


def bed_rows(g):
    bs, N = g.shape
    code = np.where(g == 2, 0, np.where(g == 1, 2, 3)).astype(np.uint8)     # ref-last .bed codes of the A1 count
    code = np.concatenate([code, np.zeros((bs, (-N) % 4), dtype=np.uint8)], axis=1).reshape(bs, -1, 4)
    return (code[..., 0] | code[..., 1] << 2 | code[..., 2] << 4 | code[..., 3] << 6).astype(np.uint8)


def one_size_bt(N, bs, P, C, reps, cpu_variants, pthresh):
    from scipy.stats import chi2
    from regenie_b200 import capi
    from oracle import step2_bt
    from oracle.prep import get_basis
    import interaction_bt_oracle as ibo
    rng = np.random.default_rng(1)
    E = rng.normal(size=N)
    X, _ = get_basis(np.column_stack([np.ones(N), rng.normal(size=(N, C - 3)), E, E * E]))
    mask = np.ones((N, P), dtype=bool)
    y = (rng.random((N, P)) < 0.2).astype(float)
    blup = rng.normal(size=(N, P)) * 0.1
    sts = [step2_bt.BtChrom(y[:, p], X, blup[:, p], mask[:, p]) for p in range(P)]
    off = np.stack([blup[:, p] + X @ sts[p].beta0 for p in range(P)], 1)
    maf = rng.uniform(0.05, 0.5, bs)
    g = rng.binomial(2, maf[:, None], (bs, N))
    rows = bed_rows(g)
    st = capi.Step2(X, mask.astype(np.uint8), np.ones(N, dtype=np.uint8), N, bs)
    st.set_chr_bt(np.stack([s.gamma_sqrt_mask for s in sts], 1), np.stack([s.gamma_sqrt for s in sts], 1),
                  np.stack([s.yres for s in sts], 1), [s.Xg for s in sts], y, np.stack([s.cov_blup_offset for s in sts], 1))
    st.set_interaction_bt(E, off)
    out = {"N": N, "bs": bs, "P": P, "C": C}
    out["plain_ms"] = best_of(lambda: st.block_bed_bt(rows, min_mac=5.0), reps)

    def wald(**kw):
        o = st.block_bed_bt(rows, min_mac=5.0)
        return o, st.interaction_bt(min_mac=5.0, **kw)

    _, (s_def, coef, vcov) = wald()
    s_rob = wald(force_robust=True)[1][0]
    out["wald_ms"] = best_of(wald, reps)
    out["robust_ms"] = best_of(lambda: wald(force_robust=True), reps)
    out["routes"] = {"robust": int((s_def == 1).sum()), "model": int((s_def == 3).sum()),
                     "forced_robust": int((s_rob == 1).sum()), "pairs": bs * P}
    wald()
    sel = np.argwhere(np.isin(s_def, (1, 3)) & (coef[..., 1] ** 2 / vcov[..., 1, 1] >= chi2.isf(pthresh, 1)))
    vi, ti = sel[:, 0], sel[:, 1]

    def firth():
        o, _ = wald()
        return st.interaction_firth(vi, ti)

    fst = firth()[3]
    out["firth_pairs"] = int(len(vi))
    out["firth_ok"] = int((fst == 0).sum())
    out["firth_ms"] = best_of(firth, reps)
    out["firth_ms_per_pair"] = (out["firth_ms"] - out["wald_ms"]) / max(1, len(vi))
    t0 = time.perf_counter()
    flags = st.block_bed_bt(rows, min_mac=5.0)["flags"]
    for v in range(cpu_variants):
        gv = g[v].astype(float)
        if flags[v] & 8:
            gv = 2.0 - gv
        H, sf, scf = ibo.design(gv, E, X, N)
        for p in range(P):
            ibo.wald(H, y[:, p], off[:, p], mask[:, p], 1e9)
    out["cpu_wald_ms_per_variant"] = (time.perf_counter() - t0) * 1e3 / cpu_variants
    out["cpu_wald_ms_per_block"] = out["cpu_wald_ms_per_variant"] * bs
    nf = min(len(vi), cpu_variants)
    if nf:
        t0 = time.perf_counter()
        for k in range(nf):
            gv = g[vi[k]].astype(float)
            if flags[vi[k]] & 8:
                gv = 2.0 - gv
            H, sf, scf = ibo.design(gv, E, X, N)
            ibo.firth(H, y[:, ti[k]], sts[ti[k]].cov_blup_offset, mask[:, ti[k]])
        out["cpu_firth_ms_per_pair"] = (time.perf_counter() - t0) * 1e3 / nf
    st.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[100000, 500000])
    ap.add_argument("--bs", type=int, default=1000)
    ap.add_argument("--pheno", type=int, default=1)
    ap.add_argument("--cov", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-variants", type=int, default=5)
    ap.add_argument("--bt", action="store_true", help="binary traits: rg_s2_interaction_bt and the Firth fallback")
    ap.add_argument("--pthresh", type=float, default=0.05, help="--bt: Firth for GxE Wald p-values at most this")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from regenie_b200 import capi
    if capi.lib().rg_device_count() <= 0:
        sys.exit("interaction_bench.py needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    if a.bt:
        sizes = [one_size_bt(n, a.bs, a.pheno, max(a.cov, 4), a.reps, a.cpu_variants, a.pthresh) for n in a.n]
    else:
        sizes = [one_size(n, a.bs, a.pheno, a.cov, a.reps, a.cpu_variants) for n in a.n]
    r = {"gpu": gpu, "mode": "bt" if a.bt else "qt", "sizes": sizes, "cpu": "numpy restatement, one thread of the GPU host"}
    line = json.dumps(r)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
