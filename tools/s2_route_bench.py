"""Time the Step-2 block routes on 2-bit rows: rg_s2_block_bed (quantitative traits) and rg_s2_block_bed_bt (binary
traits), on one block of --bs synthetic hard-call variants at --n samples and --p traits, with the rows resident on the
device (staged once through rg_s2_stage, so no call copies them again).

A worker process times each route over one window of at least --window seconds after a warm-up, and reads the device
memory the handle holds after its first rg_s2_block_bed call.  The block calls return with their results on the host,
so a host clock around the calls times the whole calls.  With --tree given more than once (source trees that each
hold a built librg_b200.so, such as two versions of this project) the driver alternates worker processes between the
trees, --rounds times, so that every tree sees the same machine state, and reports the median and the range of each
route per tree.  bench.py's Step-2 figure covers a few milliseconds and is too short to compare such builds on.
Prints one JSON line; with --out also writes it to that file.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def window_ms(fn, seconds):
    """ms per call over a window of at least `seconds`, after three warm-up calls."""
    for _ in range(3):
        fn()
    n, t0 = 0, time.perf_counter()
    while True:
        fn()
        n += 1
        dt = time.perf_counter() - t0
        if dt >= seconds:
            return dt / n * 1e3


def worker(tree, N, bs, P, C_, seconds):
    sys.path.insert(0, tree)
    from regenie_b200 import capi, synth
    L = capi.lib()
    if L.rg_device_count() == 0:
        raise RuntimeError("no CUDA device")
    rt = C.CDLL("libcudart.so.12")            # the runtime the library loaded

    def used():
        free, total = C.c_size_t(), C.c_size_t()
        if rt.cudaMemGetInfo(C.byref(free), C.byref(total)) != 0:
            raise RuntimeError("cudaMemGetInfo failed")
        return total.value - free.value

    capi.check(L.rg_warmup(0))
    mem0 = used()
    rng = np.random.default_rng(1)
    X, _ = np.linalg.qr(np.column_stack([np.ones(N), rng.normal(size=(N, C_ - 1))]))
    mask = np.ones((N, P), dtype=np.uint8)
    ia = np.ones(N, dtype=np.uint8)
    st = capi.Step2(np.asfortranarray(X), mask, ia, N, bs)
    packed = synth.pack_bed(synth.genotypes(N, bs, seed=5, miss=0.01))
    stride = packed.shape[1]
    L.rg_host_alloc.argtypes = [C.c_void_p, C.c_int64]
    L.rg_host_free.argtypes = [C.c_void_p]
    L.rg_s2_block_bed_bt.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32,
                                     C.c_double, C.c_void_p]
    hp = C.c_void_p()
    capi.check(L.rg_host_alloc(C.byref(hp), packed.nbytes))
    try:
        C.memmove(hp, packed.ctypes.data, packed.nbytes)
        dev = st.stage(0, hp.value, packed.nbytes)
        st.set_chr(np.asfortranarray(rng.standard_normal((N, P))), np.ones(P))
        out = st._out(bs)
        st.block_bed_raw(dev, bs, stride, out)
        mem = used() - mem0
        qt = window_ms(lambda: st.block_bed_raw(dev, bs, stride, out), seconds)
        p = rng.uniform(0.2, 0.8, (N, P))
        gs = np.sqrt(p * (1 - p))
        y = (rng.random((N, P)) < p).astype(float)
        st.set_chr_bt(gs, gs, (y - p) / gs, [X * gs[:, [j]] for j in range(P)], y)
        so = out[1]
        bt = window_ms(lambda: capi.check(L.rg_s2_block_bed_bt(st.h, C.c_void_p(dev), stride, bs, None, 0, 5.0,
                                                              C.byref(so))), seconds)
    finally:
        capi.check(L.rg_host_free(hp))
    st.close()
    return {"tree": tree, "qt_ms": qt, "bt_ms": bt, "mem_after_first_block_MB": mem / 1e6}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--tree", action="append", help="source tree with a built library (default: this one)")
    ap.add_argument("--n", type=int, default=100000)
    ap.add_argument("--bs", type=int, default=1000)
    ap.add_argument("--p", type=int, default=10)
    ap.add_argument("--c", type=int, default=4, help="covariate columns, intercept included")
    ap.add_argument("--window", type=float, default=0.5, help="seconds per timed window")
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--out")
    a = ap.parse_args()
    trees = [os.path.abspath(t) for t in (a.tree or [ROOT])]
    if a.worker:
        print(json.dumps(worker(trees[0], a.n, a.bs, a.p, a.c, a.window)))
        return
    runs = {t: [] for t in trees}
    for _ in range(a.rounds):
        for t in trees:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--tree", t, "--n", str(a.n),
                                "--bs", str(a.bs), "--p", str(a.p), "--c", str(a.c), "--window", str(a.window)],
                               capture_output=True, text=True)
            if r.returncode != 0:
                sys.stderr.write(r.stderr)
                raise SystemExit("worker failed for " + t)
            runs[t].append(json.loads(r.stdout.strip().splitlines()[-1]))
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"gpu": gpu[0] if gpu else "unknown", "n": a.n, "bs": a.bs, "p": a.p, "c": a.c, "window_s": a.window,
           "rounds": a.rounds, "trees": {}}
    for t, rs in runs.items():
        e = {"mem_after_first_block_MB": rs[0]["mem_after_first_block_MB"]}
        for k in ("qt_ms", "bt_ms"):
            v = [r[k] for r in rs]
            e[k] = {"median": statistics.median(v), "min": min(v), "max": max(v), "all": v}
        res["trees"][t] = e
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
