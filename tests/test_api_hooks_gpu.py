"""rg_debug_fetch failures, and the sample index of the Step-2 block calls in device memory.

rg_debug_fetch resolves a name in one of four families (the decoded .pgen rows, Step 2, level 1, level 0); every failure
returns -1 and names the buffer in rg_last_error.  "pgen_rows" alone cuts its copy to the caller's buffer instead of
failing.  rg_s2_block_bgen8_bt and rg_s2_block_bed_bt take sample_idx in host or device memory, like rg_l0_block_bed, and
give the same bits either way.
"""
import ctypes as C

import numpy as np
import pytest

from regenie_b200 import capi
from test_l1_paths_gpu import L1Case

pytestmark = pytest.mark.gpu


def _fetch(st, name, nbytes):
    out = np.zeros(max(nbytes, 8), dtype=np.uint8)
    n = capi.lib().rg_debug_fetch(st.h, name.encode(), out.ctypes.data_as(C.c_void_p), nbytes)
    return n, capi.lib().rg_last_error().decode()


def _fails(st, name, nbytes, words):
    n, msg = _fetch(st, name, nbytes)
    assert n == -1, (name, n)
    for w in (name,) + words:
        assert w in msg, (name, msg)


def _bt_problem(N=3000, n_file=3100, P=2, C=3, bs=40, seed=5):
    rng = np.random.default_rng(seed)
    X = np.asfortranarray(np.linalg.qr(np.hstack([np.ones((N, 1)), rng.standard_normal((N, C - 1))]))[0])
    mask = rng.random((N, P)) > 0.03
    p = rng.uniform(0.2, 0.8, (N, P))
    gs = np.sqrt(p * (1 - p))
    y = (rng.random((N, P)) < p) * mask
    chr_bt = (gs * mask, gs, (y - p) / gs * mask, [X * gs[:, [j]] for j in range(P)], y.astype(float))
    sample_idx = np.sort(rng.choice(n_file, N, replace=False)).astype(np.int32)
    g = rng.integers(0, 3, (bs, n_file))
    probs = np.stack([(g == 2) * 255, (g == 1) * 255], axis=2).astype(np.uint8)
    miss = np.where(rng.random((bs, n_file)) < 0.02, 0x82, 0x02).astype(np.uint8)
    packed = rng.integers(0, 256, (bs, (n_file + 3) // 4), dtype=np.uint8)
    return X, mask, chr_bt, sample_idx, probs, miss, packed


def _s2_handle(X, mask, chr_bt, bs):
    s2 = capi.Step2(X, mask, np.ones(len(X), np.uint8), len(X), bs)
    s2.set_chr_bt(*chr_bt)
    return s2


def _bgen8_bt(s2, probs, miss, idx_ptr):
    L = capi.lib()
    L.rg_s2_block_bgen8_bt.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32,
                                       C.c_double, C.c_void_p, C.c_void_p]
    o, so = s2._out(probs.shape[0], with_info=True)
    capi.check(L.rg_s2_block_bgen8_bt(s2.h, probs.ctypes.data, miss.ctypes.data, probs.shape[1], probs.shape[0], idx_ptr,
                                      0, 5.0, C.byref(so), o["info"].ctypes.data))
    return o


def _bed_bt(s2, packed, idx_ptr):
    L = capi.lib()
    L.rg_s2_block_bed_bt.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_double,
                                     C.c_void_p]
    o, so = s2._out(packed.shape[0])
    capi.check(L.rg_s2_block_bed_bt(s2.h, packed.ctypes.data, packed.shape[1], packed.shape[0], idx_ptr, 0, 5.0,
                                    C.byref(so)))
    return o


def _same_bits(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k


def test_debug_fetch_failures_name_the_buffer():
    case = L1Case(N=2000, nblocks=3)
    st = case.st
    _fails(st, "l1_dims", 64, ("no level-1 fit",))
    _fails(st, "gp", 1 << 20, ("not filled",))                     # no level-0 block has run
    _fails(st, "dims", 8, ("too small",))
    _fails(st, "no_such_buffer", 1 << 20, ("unknown",))
    case.fit()
    assert _fetch(st, "l1_dims", 64)[0] == 64
    _fails(st, "l1_dims", 8, ("too small",))
    _fails(st, "l1_chunks", 4, ("too small",))
    _fails(st, "l1_no_such_buffer", 1 << 20, ("no level-1 debug buffer",))
    _fails(st, "pgen_rows", 1 << 20, ("no rg_pgen_decode",))

    X, mask, chr_bt, idx, probs, miss, packed = _bt_problem()
    s2 = _s2_handle(X, mask, chr_bt, probs.shape[0])
    _fails(s2, "pgen_rows", 1 << 20, ("no rg_pgen_decode",))
    _fails(s2, "bt_sums", 1 << 20, ("not filled",))
    _bed_bt(s2, packed, idx.ctypes.data)
    n, _ = _fetch(s2, "bt_sums", 1 << 24)
    assert n > 0
    _fails(s2, "bt_sums", n - 8, ("too small",))
    _fails(s2, "s2_paths", 32, ("too small",))
    _fails(s2, "gp", 1 << 20, ("unknown Step-2",))
    s2.close()
    st.close()


def test_s2_bt_blocks_take_sample_idx_on_the_device():
    import torch
    X, mask, chr_bt, idx, probs, miss, packed = _bt_problem()
    idx_dev = torch.from_numpy(idx).to("cuda:0")
    bs = probs.shape[0]
    host, dev = _s2_handle(X, mask, chr_bt, bs), _s2_handle(X, mask, chr_bt, bs)
    # the device handle first maps the identity, so its index map is rebuilt from the device array
    _bgen8_bt(dev, np.ascontiguousarray(probs[:, :len(X)]), np.ascontiguousarray(miss[:, :len(X)]), None)
    _same_bits(_bgen8_bt(host, probs, miss, idx.ctypes.data), _bgen8_bt(dev, probs, miss, idx_dev.data_ptr()))
    _same_bits(_bed_bt(host, packed, idx.ctypes.data), _bed_bt(dev, packed, idx_dev.data_ptr()))
    host.close()
    dev.close()
