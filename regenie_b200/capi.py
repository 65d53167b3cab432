"""ctypes binding of librg_b200.so -- the C ABI declared in include/rg_b200.h.

This is plumbing for tests / bench.py; the product boundary is the C header.  There is no
CPU fallback: importing works anywhere (so CPU-only checks can verify the exported symbols),
but every compute entry point raises RgError when no sm_90 device is present.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "librg_b200.so")


class RgError(RuntimeError):
    pass


class Step1Config(C.Structure):
    _fields_ = [
        ("device", C.c_int32), ("n_samples", C.c_int64), ("n_cov", C.c_int32), ("n_pheno", C.c_int32),
        ("n_folds", C.c_int32), ("n_ridge_l0", C.c_int32), ("n_ridge_l1", C.c_int32), ("loocv", C.c_int32),
        ("max_block_size", C.c_int32), ("total_blocks", C.c_int32), ("n_analyzed", C.c_int64),
    ]


class Step2Config(C.Structure):
    _fields_ = [
        ("device", C.c_int32), ("n_samples", C.c_int64), ("n_cov", C.c_int32), ("n_pheno", C.c_int32),
        ("max_block_size", C.c_int32), ("n_analyzed", C.c_int64), ("strict_mode", C.c_int32),
    ]


class S2BtChr(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("gamma_sqrt_mask", "gamma_sqrt", "yres", "x_gamma", "y_raw", "firth_offset",
                                           "y_hat_p")]


class S2Out(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("af", "ns", "mac", "af_all", "ns_all", "mac_all", "flags", "scale_fac",
                                           "stat", "beta", "se", "chisq")]


class PgenBlock(C.Structure):
    _fields_ = [("bytes", C.c_void_p), ("n_bytes", C.c_int64), ("rec_off", C.c_void_p), ("rec_len", C.c_void_p),
                ("rec_type", C.c_void_p), ("n_rec", C.c_int32), ("own", C.c_void_p), ("base", C.c_void_p),
                ("bs", C.c_int32), ("n_file", C.c_int64), ("block_id", C.c_int32)]


def pgen_decode(handle, data, rec_off, rec_len, rec_type, own, base, n_file, block_id=0):
    """rg_pgen_decode on a Step1 / Step2 object: record bytes + tables (see include/rg_b200.h) -> (device pointer of the
    PLINK 1 rows, row stride).  Mirrors what host/pgen.cpp PgenFile::gather + the rgb200 driver pass."""
    L = lib()
    L.rg_pgen_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    keep = [np.ascontiguousarray(data, dtype=np.uint8), np.ascontiguousarray(rec_off, dtype=np.uint64),
            np.ascontiguousarray(rec_len, dtype=np.uint32), np.ascontiguousarray(rec_type, dtype=np.uint8),
            np.ascontiguousarray(own, dtype=np.int32), np.ascontiguousarray(base, dtype=np.int32)]
    blk = PgenBlock(keep[0].ctypes.data, keep[0].size, keep[1].ctypes.data, keep[2].ctypes.data, keep[3].ctypes.data,
                    keep[1].size, keep[4].ctypes.data, keep[5].ctypes.data, keep[4].size, int(n_file), int(block_id))
    rows, stride = C.c_void_p(0), C.c_int64(0)
    check(L.rg_pgen_decode(handle.h, C.byref(blk), C.byref(rows), C.byref(stride)))
    return int(rows.value), int(stride.value)


def debug_fetch(handle, name, dtype, count):
    """rg_debug_fetch for either handle kind (test hook)."""
    out = np.empty(count, dtype=dtype)
    n = lib().rg_debug_fetch(handle.h, name.encode(), _ptr(out), out.nbytes)
    if n < 0:
        raise RgError("debug fetch failed for %s: %s" % (name, lib().rg_last_error().decode()))
    return out[: n // out.itemsize]


# every symbol include/rg_b200.h declares (checked by tests/test_abi.py)
EXPORTS = [
    "rg_last_error", "rg_version", "rg_device_count", "rg_step1_create", "rg_destroy", "rg_sync",
    "rg_l0_block_bed", "rg_l0_status", "rg_l0_fetch_W", "rg_l1_fit", "rg_loco", "rg_step2_create",
    "rg_s2_set_chr", "rg_s2_block_bed", "rg_W_info", "rg_debug_fetch", "rg_launch_count", "rg_stream",
    "rg_set_timing", "rg_get_timing", "rg_fence", "rg_s2_set_chr_bt", "rg_s2_block_bgen8_bt", "rg_s2_block_bgen8", "rg_s2_firth", "rg_l1_fit_bt", "rg_W_set_owned", "rg_W_export", "rg_W_attach_peer", "rg_l1_select", "rg_s2_set_sex", "rg_s2_set_non_par", "rg_l0_load_W", "rg_s2_spa", "rg_s2_block_bed_bt", "rg_prs", "rg_bgen_inflate", "rg_s2_set_interaction", "rg_s2_interaction", "rg_s2_set_interaction_bt", "rg_s2_interaction_bt", "rg_s2_interaction_firth",
    "rg_l0_solver_stats", "rg_dbg_mixed_solve", "rg_l0_wait_input", "rg_l0_block_dosage_u8", "rg_l0_block_f64", "rg_W_attach_local",
    "rg_s2_stage", "rg_host_alloc", "rg_host_free", "rg_pgen_decode", "rg_warmup", "rg_l0_poll_status",
]

_lib = None


def lib():
    """Load librg_b200.so (fails loudly if it was never built)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RgError("librg_b200.so not built: run `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(LIB_PATH)
        L.rg_last_error.restype = C.c_char_p
        L.rg_version.restype = C.c_char_p
        L.rg_l0_status.restype = C.c_int64
        L.rg_l0_poll_status.restype = C.c_int64
        L.rg_l0_poll_status.argtypes = [C.c_void_p]
        L.rg_debug_fetch.restype = C.c_int64
        L.rg_launch_count.restype = C.c_int64
        L.rg_stream.restype = C.c_void_p
        L.rg_destroy.restype = None
        for name in ("rg_destroy", "rg_sync", "rg_l0_status", "rg_launch_count", "rg_stream", "rg_fence"):
            getattr(L, name).argtypes = [C.c_void_p]
        L.rg_l0_block_bed.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_int32]
        L.rg_l0_fetch_W.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
        L.rg_debug_fetch.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64]
        L.rg_set_timing.argtypes = [C.c_void_p, C.c_int32]
        L.rg_get_timing.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_void_p]
        L.rg_l1_fit.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.rg_loco.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.rg_prs.argtypes = [C.c_void_p, C.c_void_p]
        L.rg_W_info.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def check(rc):
    if rc != 0:
        raise RgError(lib().rg_last_error().decode())


def _ptr(a):
    """numpy array -> void* (host), int -> raw (device) pointer, None -> NULL."""
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    return a.ctypes.data_as(C.c_void_p)


def _f64(a, order="F"):
    return np.require(a, dtype=np.float64, requirements=["F" if order == "F" else "C", "A"])


class Step1:
    """Host-side mirror of the Step-1 call sequence of Data::run_step1 (src/Data.cpp:95-133)."""

    def __init__(self, X, Y, mask, in_analysis, fold_sizes, lam, neff, n_analyzed, max_block_size,
                 total_blocks, n_ridge_l1=5, loocv=False, device=0):
        L = lib()
        X = _f64(X); Y = _f64(Y)
        mask = np.require(np.asarray(mask, dtype=np.uint8), requirements=["F", "A"])
        ia = np.ascontiguousarray(in_analysis, dtype=np.uint8)
        fs = np.ascontiguousarray(fold_sizes, dtype=np.int64)
        lam = np.ascontiguousarray(lam, dtype=np.float64)
        neff = np.ascontiguousarray(neff, dtype=np.float64)
        self.N, self.C = X.shape
        self.P = Y.shape[1]
        self.R = len(lam)
        self.R1 = n_ridge_l1
        self.total_blocks = total_blocks
        cfg = Step1Config(device, self.N, self.C, self.P, len(fs), self.R, n_ridge_l1, int(loocv),
                          max_block_size, total_blocks, int(n_analyzed))
        h = C.c_void_p()
        check(L.rg_step1_create(C.byref(cfg), _ptr(X), _ptr(Y), _ptr(mask), _ptr(ia), _ptr(fs), _ptr(lam),
                                _ptr(neff), C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            lib().rg_destroy(self.h)
            self.h = None

    __del__ = close

    def l0_block_bed(self, packed, bs, block_id, row_stride=None, sample_idx=None, ref_first=False):
        """packed: uint8 ndarray [bs, stride] (host) or an int device pointer (+ row_stride)."""
        if not isinstance(packed, int):
            packed = np.ascontiguousarray(packed, dtype=np.uint8)
            row_stride = packed.shape[1]
        if sample_idx is not None and not isinstance(sample_idx, int):
            sample_idx = np.ascontiguousarray(sample_idx, dtype=np.int32)
            self._keep_idx = sample_idx
        check(lib().rg_l0_block_bed(self.h, _ptr(packed), row_stride, bs, _ptr(sample_idx), int(ref_first),
                                    block_id))

    def status(self):
        return lib().rg_l0_status(self.h)

    def poll_status(self):
        """The sticky error word as the finished blocks left it; does not wait for the lanes."""
        return lib().rg_l0_poll_status(self.h)

    def sync(self):
        check(lib().rg_sync(self.h))

    def fence(self):
        check(lib().rg_fence(self.h))

    def fetch_W(self, block_id, ph):
        out = np.empty((self.N, self.R), dtype=np.float64, order="F")
        check(lib().rg_l0_fetch_W(self.h, block_id, ph, _ptr(out)))
        return out

    def load_W(self, block_id, ph, slab):
        L = lib(); L.rg_l0_load_W.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
        a = _f64(slab)
        check(L.rg_l0_load_W(self.h, block_id, ph, _ptr(a)))

    def l1_fit(self, tau):
        tau = np.ascontiguousarray(tau, dtype=np.float64).reshape(self.P, self.R1)
        cs = np.zeros((5, self.P, self.R1))
        best = np.zeros(self.P, dtype=np.int32)
        check(lib().rg_l1_fit(self.h, _ptr(tau), _ptr(cs), _ptr(best)))
        return cs, best

    def W_set_owned(self, owned):
        L = lib(); L.rg_W_set_owned.argtypes = [C.c_void_p, C.c_void_p]
        ob = np.ascontiguousarray(owned, dtype=np.uint8)
        check(L.rg_W_set_owned(self.h, _ptr(ob)))

    def W_export(self):
        """64-byte CUDA IPC handle of this rank's W allocation."""
        buf = (C.c_ubyte * 64)()
        L = lib(); L.rg_W_export.argtypes = [C.c_void_p, C.c_void_p]
        check(L.rg_W_export(self.h, buf))
        return bytes(buf)

    def W_attach_peer(self, handle, owned_by_peer):
        L = lib(); L.rg_W_attach_peer.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p]
        ob = np.ascontiguousarray(owned_by_peer, dtype=np.uint8)
        check(L.rg_W_attach_peer(self.h, handle, _ptr(ob)))

    def l1_select(self, sel):
        L = lib(); L.rg_l1_select.argtypes = [C.c_void_p, C.c_void_p]
        sb = np.ascontiguousarray(sel, dtype=np.uint8)
        check(L.rg_l1_select(self.h, _ptr(sb)))

    def l1_fit_bt(self, y_raw, offset, tau):
        """Binary traits: logistic level 1 (LOOCV).  Returns cumsums [6, P, R1] and argmin -logLik/N."""
        L = lib()
        L.rg_l1_fit_bt.argtypes = [C.c_void_p] * 6
        tau = np.ascontiguousarray(tau, dtype=np.float64).reshape(self.P, self.R1)
        y_raw = _f64(y_raw); offset = _f64(offset)
        cs = np.zeros((6, self.P, self.R1))
        best = np.zeros(self.P, dtype=np.int32)
        check(L.rg_l1_fit_bt(self.h, _ptr(y_raw), _ptr(offset), _ptr(tau), _ptr(cs), _ptr(best)))
        return cs, best

    def loco(self, chr_of_block):
        cb = np.ascontiguousarray(chr_of_block, dtype=np.int32)
        out = np.zeros((self.P, 23, self.N))          # [P][N x 23] column-major
        check(lib().rg_loco(self.h, _ptr(cb), _ptr(out)))
        return out.transpose(0, 2, 1)                 # -> [P, N, 23]

    def prs(self):
        """Whole-genome predictions [P, N] of the last loco() call (--print-prs)."""
        out = np.zeros((self.P, self.N))
        check(lib().rg_prs(self.h, _ptr(out)))
        return out

    def debug(self, name, dtype, count):
        """rg_debug_fetch: level-0 intermediates of the last block, or of the last level-1 fit: "l1_dims" (int64 x 8:
        B, nC, R1, K, systems, rows per system, chunks, chunk length), "l1_chunks" (int32 x 4 per chunk), "l1_beta"
        ([P][K R1][nC], k-fold), "l1_sums" ([P][3 kMaxRidge + 2]), "l1_bvec" ([P][nC]) and "l1_hvec" ([P][Npad]) (LOOCV)."""
        return debug_fetch(self, name, dtype, count)

    def launch_count(self):
        return lib().rg_launch_count(self.h)

    def l0_block_dosage_u8(self, probs, missing, block_id, sample_idx=None, ref_first=False):
        """probs u8 [bs][n_file][2], missing u8 [bs][n_file] (bit 7) or None."""
        L = lib()
        L.rg_l0_block_dosage_u8.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_int32]
        probs = np.ascontiguousarray(probs, dtype=np.uint8)
        if missing is not None:
            missing = np.ascontiguousarray(missing, dtype=np.uint8)
        if sample_idx is not None:
            sample_idx = np.ascontiguousarray(sample_idx, dtype=np.int32)
        check(L.rg_l0_block_dosage_u8(self.h, _ptr(probs), _ptr(missing), probs.shape[1], probs.shape[0], _ptr(sample_idx),
                                      int(ref_first), int(block_id)))

    def l0_block_f64(self, G, block_id, sample_idx=None):
        L = lib()
        L.rg_l0_block_f64.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32]
        G = np.ascontiguousarray(G, dtype=np.float64)
        if sample_idx is not None:
            sample_idx = np.ascontiguousarray(sample_idx, dtype=np.int32)
        check(L.rg_l0_block_f64(self.h, _ptr(G), G.shape[1], G.shape[0], _ptr(sample_idx), int(block_id)))

    def solver_stats(self):
        """(blocks solved by the tensor-core + refinement path, of which re-solved by the FP64 Cholesky)."""
        L = lib(); L.rg_l0_solver_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        a, b = C.c_int64(0), C.c_int64(0)
        check(L.rg_l0_solver_stats(self.h, C.byref(a), C.byref(b)))
        return int(a.value), int(b.value)

    def stream(self):
        return lib().rg_stream(self.h)

    def set_timing(self, on=True):
        check(lib().rg_set_timing(self.h, int(on)))

    def timing(self, name):
        ms = C.c_double(); n = C.c_int64()
        check(lib().rg_get_timing(self.h, name.encode(), C.byref(ms), C.byref(n)))
        return ms.value, n.value


class S2IntChr(C.Structure):
    _fields_ = [("E", C.c_void_p), ("n_px", C.c_int32), ("dinv_sqrt", C.c_void_p), ("px", C.c_void_p), ("yres", C.c_void_p)]


class S2IntOpts(C.Structure):
    _fields_ = [("rare_mac", C.c_double), ("min_mac", C.c_double), ("force_robust", C.c_int32),
                ("force_hc4", C.c_int32), ("no_robust", C.c_int32)]


class S2IntBtChr(C.Structure):
    _fields_ = [("E", C.c_void_p), ("offset", C.c_void_p)]


class Step2:
    """Host-side mirror of the Step-2 QT call sequence of Data::test_snps_fast (src/Data.cpp:2230-2383)."""

    def __init__(self, X, mask, in_analysis, n_analyzed, max_block_size, strict=False, device=0):
        L = lib()
        L.rg_s2_set_chr.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.rg_s2_block_bed.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32,
                                      C.c_double, C.c_void_p]
        X = _f64(X)
        mask = np.require(np.asarray(mask, dtype=np.uint8), requirements=["F", "A"])
        ia = np.ascontiguousarray(in_analysis, dtype=np.uint8)
        self.N, self.C = X.shape
        self.P = mask.shape[1]
        cfg = Step2Config(device, self.N, self.C, self.P, max_block_size, int(n_analyzed), int(strict))
        h = C.c_void_p()
        check(L.rg_step2_create(C.byref(cfg), _ptr(X), _ptr(mask), _ptr(ia), C.byref(h)))
        self.h = h
        self.last_bs = None                 # variants of the last block call that succeeded (what interaction() reads)

    def close(self):
        if getattr(self, "h", None):
            lib().rg_destroy(self.h)
            self.h = None

    __del__ = close

    def set_sex(self, male):
        L = lib(); L.rg_s2_set_sex.argtypes = [C.c_void_p, C.c_void_p]
        m = None if male is None else np.ascontiguousarray(male, dtype=np.uint8)
        check(L.rg_s2_set_sex(self.h, _ptr(m)))

    def set_non_par(self, flags):
        L = lib(); L.rg_s2_set_non_par.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
        f = np.ascontiguousarray(flags, dtype=np.uint8)
        check(L.rg_s2_set_non_par(self.h, _ptr(f), len(f)))

    def set_chr(self, res, scf_sv):
        res = _f64(res)
        scf = np.ascontiguousarray(scf_sv, dtype=np.float64)
        check(lib().rg_s2_set_chr(self.h, _ptr(res), _ptr(scf)))

    def block_bed(self, packed, sample_idx=None, ref_first=False, min_mac=5.0, row_stride=None, bs=None):
        """packed: uint8 ndarray [bs, stride] (host), or an int device pointer with row_stride and bs."""
        if isinstance(packed, int):
            P = self.P
        else:
            packed = np.ascontiguousarray(packed, dtype=np.uint8)
            bs, P, row_stride = packed.shape[0], self.P, packed.shape[1]
        o = dict(af=np.empty((bs, P)), ns=np.empty((bs, P), dtype=np.int32), mac=np.empty((bs, P)),
                 af_all=np.empty(bs), ns_all=np.empty(bs, dtype=np.int32), mac_all=np.empty(bs),
                 flags=np.empty(bs, dtype=np.int32), scale_fac=np.empty(bs), stat=np.empty((bs, P)),
                 beta=np.empty((bs, P)), se=np.empty((bs, P)), chisq=np.empty((bs, P)))
        so = S2Out(*[o[k].ctypes.data for k in ("af", "ns", "mac", "af_all", "ns_all", "mac_all", "flags",
                                                "scale_fac", "stat", "beta", "se", "chisq")])
        if sample_idx is not None:
            sample_idx = np.ascontiguousarray(sample_idx, dtype=np.int32)
        check(lib().rg_s2_block_bed(self.h, _ptr(packed), row_stride, bs, _ptr(sample_idx), int(ref_first),
                                    float(min_mac), C.byref(so)))
        self.last_bs = int(bs)
        return o

    def _out(self, bs, with_info=False):
        P = self.P
        o = dict(af=np.empty((bs, P)), ns=np.empty((bs, P), dtype=np.int32), mac=np.empty((bs, P)),
                 af_all=np.empty(bs), ns_all=np.empty(bs, dtype=np.int32), mac_all=np.empty(bs),
                 flags=np.empty(bs, dtype=np.int32), scale_fac=np.empty(bs), stat=np.empty((bs, P)),
                 beta=np.empty((bs, P)), se=np.empty((bs, P)), chisq=np.empty((bs, P)))
        if with_info:
            o["info"] = np.empty((bs, P))
        so = S2Out(*[o[k].ctypes.data for k in ("af", "ns", "mac", "af_all", "ns_all", "mac_all", "flags",
                                                "scale_fac", "stat", "beta", "se", "chisq")])
        return o, so

    def stage(self, slot, host_ptr, nbytes):
        """rg_s2_stage: start the H2D copy of a later block's input (raw host address, ideally pinned); returns the device
        address to hand to the *_raw block call of that block."""
        L = lib()
        L.rg_s2_stage.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p]
        dev = C.c_void_p()
        check(L.rg_s2_stage(self.h, int(slot), C.c_void_p(host_ptr), int(nbytes), C.byref(dev)))
        return dev.value

    def block_bed_raw(self, ptr, bs, row_stride, out=None, min_mac=5.0):
        """rg_s2_block_bed on a raw (host or DEVICE) address; `out` = a (dict, S2Out) pair from _out() to reuse."""
        o, so = out or self._out(bs)
        check(lib().rg_s2_block_bed(self.h, C.c_void_p(ptr), int(row_stride), int(bs), None, 0, float(min_mac), C.byref(so)))
        self.last_bs = int(bs)
        return o

    def block_bgen8_bt_raw(self, probs_ptr, miss_ptr, n_file, bs, out=None, min_mac=5.0):
        """rg_s2_block_bgen8_bt on raw (host or DEVICE) addresses, e.g. the pair rg_bgen_inflate returned."""
        L = lib()
        L.rg_s2_block_bgen8_bt.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p,
                                           C.c_int32, C.c_double, C.c_void_p, C.c_void_p]
        o, so = out or self._out(bs, with_info=True)
        check(L.rg_s2_block_bgen8_bt(self.h, C.c_void_p(probs_ptr), C.c_void_p(miss_ptr), int(n_file), int(bs), None, 0,
                                     float(min_mac), C.byref(so), _ptr(o["info"])))
        self.last_bs = int(bs)
        return o

    # ---- binary traits on BGEN 8-bit dosages
    def set_chr_bt(self, gamma_sqrt_mask, gamma_sqrt, yres, x_gamma, y_raw, firth_offset=None, y_hat_p=None):
        """Arrays are [N x P] (x_gamma: list of P arrays [N x C]); see rg_s2_bt_chr."""
        L = lib()
        L.rg_s2_set_chr_bt.argtypes = [C.c_void_p, C.c_void_p]
        keep = [_f64(gamma_sqrt_mask), _f64(gamma_sqrt), _f64(yres),
                np.ascontiguousarray(np.stack([_f64(x) for x in x_gamma]).transpose(0, 2, 1), dtype=np.float64),
                _f64(y_raw), None if firth_offset is None else _f64(firth_offset),
                None if y_hat_p is None else _f64(y_hat_p)]
        st = S2BtChr(*[None if a is None else a.ctypes.data for a in keep])
        check(L.rg_s2_set_chr_bt(self.h, C.byref(st)))

    def block_bed_bt(self, packed, sample_idx=None, ref_first=False, min_mac=5.0):
        """Binary traits on 2-bit rows (after set_chr_bt)."""
        L = lib()
        L.rg_s2_block_bed_bt.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32,
                                         C.c_double, C.c_void_p]
        packed = np.ascontiguousarray(packed, dtype=np.uint8)
        bs, P = packed.shape[0], self.P
        o = dict(af=np.empty((bs, P)), ns=np.empty((bs, P), dtype=np.int32), mac=np.empty((bs, P)),
                 af_all=np.empty(bs), ns_all=np.empty(bs, dtype=np.int32), mac_all=np.empty(bs),
                 flags=np.empty(bs, dtype=np.int32), scale_fac=np.empty(bs), stat=np.empty((bs, P)),
                 beta=np.empty((bs, P)), se=np.empty((bs, P)), chisq=np.empty((bs, P)))
        so = S2Out(*[o[k].ctypes.data for k in ("af", "ns", "mac", "af_all", "ns_all", "mac_all", "flags",
                                                "scale_fac", "stat", "beta", "se", "chisq")])
        if sample_idx is not None:
            sample_idx = np.ascontiguousarray(sample_idx, dtype=np.int32)
        check(L.rg_s2_block_bed_bt(self.h, _ptr(packed), packed.shape[1], bs, _ptr(sample_idx), int(ref_first),
                                   float(min_mac), C.byref(so)))
        self.last_bs = int(bs)
        return o

    def block_bgen8(self, probs, missing=None, sample_idx=None, ref_first=False, min_mac=5.0):
        """Quantitative traits on dosages (after set_chr)."""
        return self.block_bgen8_bt(probs, missing, sample_idx, ref_first, min_mac, _fn="rg_s2_block_bgen8")

    def block_bgen8_bt(self, probs, missing=None, sample_idx=None, ref_first=False, min_mac=5.0,
                       _fn="rg_s2_block_bgen8_bt"):
        """probs u8 [bs][n_file][2]; missing u8 [bs][n_file] (bit 7 = missing) or None."""
        L = lib()
        getattr(L, _fn).argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p,
                                           C.c_int32, C.c_double, C.c_void_p, C.c_void_p]
        probs = np.ascontiguousarray(probs, dtype=np.uint8)
        bs, n_file, P = probs.shape[0], probs.shape[1], self.P
        if missing is not None:
            missing = np.ascontiguousarray(missing, dtype=np.uint8)
        o = dict(af=np.empty((bs, P)), ns=np.empty((bs, P), dtype=np.int32), mac=np.empty((bs, P)),
                 af_all=np.empty(bs), ns_all=np.empty(bs, dtype=np.int32), mac_all=np.empty(bs),
                 flags=np.empty(bs, dtype=np.int32), scale_fac=np.empty(bs), stat=np.empty((bs, P)),
                 beta=np.empty((bs, P)), se=np.empty((bs, P)), chisq=np.empty((bs, P)), info=np.empty((bs, P)))
        so = S2Out(*[o[k].ctypes.data for k in ("af", "ns", "mac", "af_all", "ns_all", "mac_all", "flags",
                                                "scale_fac", "stat", "beta", "se", "chisq")])
        if sample_idx is not None:
            sample_idx = np.ascontiguousarray(sample_idx, dtype=np.int32)
        check(getattr(L, _fn)(self.h, _ptr(probs), _ptr(missing), n_file, bs, _ptr(sample_idx),
                                     int(ref_first), float(min_mac), C.byref(so), _ptr(o["info"])))
        self.last_bs = int(bs)
        return o

    def bgen_inflate(self, comp, comp_offs, n_file):
        """Inflate the zlib payloads of a block on the device (rg_bgen_inflate).  comp: u8 bytes, comp_offs: [bs+1].
        Returns the two DEVICE addresses (probs, ploidy_missing) to hand to block_bgen8*_dev."""
        L = lib()
        L.rg_bgen_inflate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_void_p]
        comp = np.ascontiguousarray(comp, dtype=np.uint8)
        offs = np.ascontiguousarray(comp_offs, dtype=np.uint64)
        pd, md = C.c_void_p(), C.c_void_p()
        check(L.rg_bgen_inflate(self.h, _ptr(comp), _ptr(offs), int(n_file), len(offs) - 1, C.byref(pd), C.byref(md)))
        return pd.value, md.value

    def spa(self, variant_idx, trait_idx):
        L = lib()
        L.rg_s2_spa.argtypes = [C.c_void_p, C.c_int32] + [C.c_void_p] * 4
        vi = np.ascontiguousarray(variant_idx, dtype=np.int32)
        ti = np.ascontiguousarray(trait_idx, dtype=np.int32)
        pv, status = np.empty(len(vi)), np.empty(len(vi), dtype=np.int32)
        check(L.rg_s2_spa(self.h, len(vi), _ptr(vi), _ptr(ti), _ptr(pv), _ptr(status)))
        return pv, status

    # ---- GxE interaction tests (quantitative traits)
    def set_interaction(self, E, dinv_sqrt=None, px=None, yres=None):
        """rg_s2_set_interaction after set_chr.  E [N]; HLM state (or None): dinv_sqrt, yres [N x P], px list of P [N x K]."""
        L = lib()
        L.rg_s2_set_interaction.argtypes = [C.c_void_p, C.c_void_p]
        E = np.ascontiguousarray(E, dtype=np.float64)
        K = 0 if px is None else px[0].shape[1]
        keep = [E]
        if K:
            keep += [_f64(dinv_sqrt), np.ascontiguousarray(np.stack([_f64(x) for x in px]).transpose(0, 2, 1)), _f64(yres)]
        st = S2IntChr(E.ctypes.data, K, *[keep[k].ctypes.data if K else None for k in (1, 2, 3)])
        check(L.rg_s2_set_interaction(self.h, C.byref(st)))

    def interaction(self, bs=None, rare_mac=1000.0, min_mac=5.0, force_robust=False, force_hc4=False, no_robust=False):
        """rg_s2_interaction on the resident block: (status [bs, P], coef [bs, P, 2], vcov [bs, P, 2, 2]).

        The library writes one row per variant of the last block call, so the outputs are sized for that block; `bs`, when
        given, must equal its size.  Raises ValueError, without calling the library, when no block call has succeeded on
        this handle or when `bs` differs."""
        if self.last_bs is None:
            raise ValueError("interaction() needs a block call first")
        if bs is None:
            bs = self.last_bs
        elif int(bs) != self.last_bs:
            raise ValueError("interaction(bs=%d): the last block had %d variants" % (int(bs), self.last_bs))
        L = lib()
        L.rg_s2_interaction.argtypes = [C.c_void_p] * 5
        P = self.P
        status = np.empty((bs, P), dtype=np.int32)
        coef, vcov = np.empty((bs, P, 2)), np.empty((bs, P, 2, 2))
        o = S2IntOpts(float(rare_mac), float(min_mac), int(force_robust), int(force_hc4), int(no_robust))
        check(L.rg_s2_interaction(self.h, C.byref(o), _ptr(status), _ptr(coef), _ptr(vcov)))
        return status, coef, vcov

    # ---- GxE interaction tests (binary traits)
    def set_interaction_bt(self, E, offset):
        """rg_s2_set_interaction_bt after set_chr_bt.  E [N]; offset [N x P], the linear predictor of each trait's null
        logistic fit (offset_nullreg)."""
        L = lib()
        L.rg_s2_set_interaction_bt.argtypes = [C.c_void_p, C.c_void_p]
        E = np.ascontiguousarray(E, dtype=np.float64)
        off = _f64(offset)
        if E.shape != (self.N,) or off.shape != (self.N, self.P):
            raise ValueError("set_interaction_bt: E must have %d entries and offset shape (%d, %d)" % (self.N, self.N, self.P))
        st = S2IntBtChr(E.ctypes.data, off.ctypes.data)
        check(L.rg_s2_set_interaction_bt(self.h, C.byref(st)))

    def interaction_bt(self, rare_mac=1000.0, min_mac=5.0, force_robust=False, no_robust=False):
        """rg_s2_interaction_bt on the resident binary-trait block: (status [bs, P], coef [bs, P, 2], vcov [bs, P, 2, 2]).
        Raises ValueError, without calling the library, when no block call has succeeded on this handle."""
        if self.last_bs is None:
            raise ValueError("interaction_bt() needs a block call first")
        L = lib()
        L.rg_s2_interaction_bt.argtypes = [C.c_void_p] * 5
        bs, P = self.last_bs, self.P
        status = np.empty((bs, P), dtype=np.int32)
        coef, vcov = np.empty((bs, P, 2)), np.empty((bs, P, 2, 2))
        o = S2IntOpts(float(rare_mac), float(min_mac), int(force_robust), 0, int(no_robust))
        check(L.rg_s2_interaction_bt(self.h, C.byref(o), _ptr(status), _ptr(coef), _ptr(vcov)))
        return status, coef, vcov

    def interaction_firth(self, variant_idx, trait_idx):
        """rg_s2_interaction_firth for the pairs (variant_idx[k], trait_idx[k]) of the resident block: (coef [n, 2],
        se [n, 2], lrt [n, 3] = (2DF, SNP, SNPxVAR), status [n])."""
        L = lib()
        L.rg_s2_interaction_firth.argtypes = [C.c_void_p, C.c_int32] + [C.c_void_p] * 6
        vi = np.ascontiguousarray(variant_idx, dtype=np.int32).reshape(-1)
        ti = np.ascontiguousarray(trait_idx, dtype=np.int32).reshape(-1)
        if len(vi) != len(ti):
            raise ValueError("interaction_firth: %d variant indices, %d trait indices" % (len(vi), len(ti)))
        n = len(vi)
        coef, se, lrt = np.empty((n, 2)), np.empty((n, 2)), np.empty((n, 3))
        status = np.empty(n, dtype=np.int32)
        check(L.rg_s2_interaction_firth(self.h, n, _ptr(vi), _ptr(ti), _ptr(coef), _ptr(se), _ptr(lrt), _ptr(status)))
        return coef, se, lrt, status

    def debug(self, name, dtype, count):
        """rg_debug_fetch: "s2_paths" (int64 x 8), "s2_sums", "bt_sums", "bt_nnz", "bt_n510" of the resident block; "s2_gp"
        (uint32 [rows_p][Npad/16]), "s2_T" (float32 [chunk][3 rows_p][drows]) and "s2_FD" (int8 [drows][Npad]): the 2-bit
        rows, tensor sums and digit rows of F of the last 2-bit block.  GxE interaction: "int_F" (float64 [Npad][nf]),
        the feature rows rg_s2_set_interaction built; of the last interaction() call since then, "int_paths" (int64 x 8:
        sample chunks, Npad, nf, robust columns nr, HLM columns per trait K, trait groups of the meat kernel, host slabs
        of the feature rows, bs), "int_route" (int8 [bs]: 0 none, 1 robust, 2 HLM) and "int_sums" (float64 [bs][nf],
        defined at the columns the variant's route reads)."""
        return debug_fetch(self, name, dtype, count)

    def firth(self, variant_idx, trait_idx):
        L = lib()
        L.rg_s2_firth.argtypes = [C.c_void_p, C.c_int32] + [C.c_void_p] * 6
        vi = np.ascontiguousarray(variant_idx, dtype=np.int32)
        ti = np.ascontiguousarray(trait_idx, dtype=np.int32)
        n = len(vi)
        beta, se, lrt, status = np.empty(n), np.empty(n), np.empty(n), np.empty(n, dtype=np.int32)
        check(L.rg_s2_firth(self.h, n, _ptr(vi), _ptr(ti), _ptr(beta), _ptr(se), _ptr(lrt), _ptr(status)))
        return beta, se, lrt, status


def mixed_solve(Af, lam, b, steps=3, tol=1e-9, device=0, want_inverse=False):
    """Test hook (rg_dbg_mixed_solve): solve (Af[f] + lam[r] I) x = b[f] for every (f, r) with the mixed-precision solver.
    Af [K, n, n] symmetric, lam [R], b [K, P, n].  Returns (x [K*R, P, n], fail flag, X [K*R, n, n] float32 or None)."""
    Af = np.ascontiguousarray(Af, dtype=np.float64); lam = np.ascontiguousarray(lam, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    K, n, _ = Af.shape
    R, P = len(lam), b.shape[1]
    x = np.zeros((K * R, P, n))
    X = np.zeros((K * R, n, n), dtype=np.float32) if want_inverse else None
    fail = C.c_uint32(0)
    L = lib()
    L.rg_dbg_mixed_solve.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_int32, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
    check(L.rg_dbg_mixed_solve(device, n, K, R, P, _ptr(Af), _ptr(lam), _ptr(b), steps, tol, _ptr(x),
                               _ptr(X) if X is not None else None, C.byref(fail)))
    return x, int(fail.value), X
