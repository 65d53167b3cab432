"""In-tree build of librg_b200.so (CUDA kernels + C ABI) and the rgb200 host driver.

nvcc cross-compiles for sm_90a (H100) without a GPU; the .so and the objects are build products (git-ignored).
Rebuilds only when a source is newer than its object.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "librg_b200.so")
DRIVER = os.path.join(HERE, "rgb200")
PROBE = os.path.join(HERE, "rgb200_hostprobe")     # CPU-only test hook for the host logic (host/probe/)

NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    ARCH[0], ARCH[1], "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3,-Wall,-Wno-unused-function", "--expt-relaxed-constexpr",
    "-I", os.path.join(ROOT, "include"),
]


def _newer(src_list, target):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in src_list)


def _run(cmd, verbose):
    if verbose:
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("build failed: " + " ".join(cmd))
    if verbose and (r.stdout or r.stderr):
        print(r.stdout + r.stderr)


def cuda_sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h", ".hpp"))]
    hs.append(os.path.join(ROOT, "include", "rg_b200.h"))
    return hs


def build_lib(verbose=False, force=False, extra_flags=()):
    if not os.path.exists(NVCC):
        if os.path.exists(LIB):
            return LIB          # no toolchain here: use the library built earlier
        raise RuntimeError("nvcc not found and no prebuilt librg_b200.so")
    os.makedirs(OBJ, exist_ok=True)
    objs = []
    hdrs = headers()
    for src in cuda_sources():
        obj = os.path.join(OBJ, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if force or _newer([src] + hdrs, obj):
            _run([NVCC] + NVCC_FLAGS + list(extra_flags) + ["-c", src, "-o", obj], verbose)
    if force or _newer(objs, LIB):
        _run([NVCC, "-shared", "-o", LIB] + objs + ARCH + ["-lcudart"], verbose)
    return LIB


def host_sources():
    d = os.path.join(HERE, "host")
    if not os.path.isdir(d):
        return []
    return sorted(os.path.join(d, f) for f in os.listdir(d) if f.endswith(".cpp"))


def build_driver(verbose=False, force=False):
    srcs = host_sources()
    if not srcs:
        return None
    gxx = shutil.which("g++")
    if gxx is None:
        if os.path.exists(DRIVER):
            return DRIVER
        raise RuntimeError("g++ not found and no prebuilt rgb200")
    hdrs = [os.path.join(HERE, "host", f) for f in os.listdir(os.path.join(HERE, "host")) if f.endswith(".hpp")]
    if force or _newer(srcs + hdrs + [LIB], DRIVER):
        _run([gxx, "-O2", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), "-o", DRIVER] + srcs +
             ["-L", HERE, "-lrg_b200", "-Wl,-rpath,$ORIGIN", "-lz", "-lpthread", "-ldl"], verbose)
    return DRIVER


def build_probe(verbose=False, force=False):
    """Host sources minus main.cpp plus host/probe/probe_main.cpp; no CUDA library on the link line."""
    srcs = [s for s in host_sources() if os.path.basename(s) != "main.cpp"]
    probe_src = os.path.join(HERE, "host", "probe", "probe_main.cpp")
    gxx = shutil.which("g++")
    if gxx is None or not os.path.exists(probe_src):
        return PROBE if os.path.exists(PROBE) else None
    hdrs = [os.path.join(HERE, "host", f) for f in os.listdir(os.path.join(HERE, "host")) if f.endswith(".hpp")]
    hdrs.append(os.path.join(CSRC, "inflate_core.h"))          # the device decoders, compiled for the host with one lane
    hdrs.append(os.path.join(CSRC, "pgen_core.h"))
    if force or _newer(srcs + hdrs + [probe_src], PROBE):
        _run([gxx, "-O2", "-std=c++17", "-Wall", "-o", PROBE, probe_src] + srcs + ["-lz", "-lpthread", "-ldl"], verbose)
    return PROBE


def build_all(verbose=False, force=False):
    build_lib(verbose, force)
    build_driver(verbose, force)
    build_probe(verbose, force)


if __name__ == "__main__":
    build_all(verbose=True, force="--force" in sys.argv)
