"""A handle is a Step-1 or a Step-2 handle, and each holds only its own kind's state.

Every entry point that serves one kind refuses a handle of the other kind with return code 1 (-1 for
rg_l0_poll_status) and, where it sets rg_last_error, the message that names the kind it needs; the handle stays usable,
and the next block on it is bit-identical to one on a fresh handle.  The entry points that serve both kinds keep
working on either.  A Step-1 create that fails inside its fold layout returns its message and leaves the device usable,
and handles destroyed with work and lazily made resources in flight (staging copies, the poll stream, timing events,
lane copy streams) leave the next handle's results unchanged.
"""
import ctypes as C

import numpy as np
import pytest

import helpers
from regenie_b200 import capi

pytestmark = pytest.mark.gpu

NOT_S1 = "handle is not a Step-1 handle"
NOT_S2 = "handle is not a Step-2 handle"
VP = C.c_void_p


@pytest.fixture(scope="module")
def pb(tmp_path_factory):
    return helpers.synthetic_problem(tmp_path_factory.mktemp("kinds"), N=640, M=256, P=2, C=3, bsize=128)


def _step2(pb):
    pr = pb.prep
    return capi.Step2(pr.X, pr.mask, pr.in_analysis, pr.n_analyzed, pb.bsize)


def _s2_block(pb, st):
    pr = pb.prep
    rng = np.random.default_rng(3)
    st.set_chr(np.asfortranarray(rng.standard_normal(pr.mask.shape) * pr.mask), np.ones(pr.mask.shape[1]))
    c, s, bs = pb.blocks[0]
    return st.block_bed(pb.packed[s:s + bs], sample_idx=None if pb.keep.all() else pb.sample_idx)


def _s1_W(pb, st):
    pb.gpu_l0_block(st, 0)
    assert st.status() == 0, capi.lib().rg_last_error().decode()
    return [st.fetch_W(0, ph) for ph in range(st.P)]


def _own_lib():
    """A CDLL of its own, so the prototypes set here leave those of capi.lib() alone."""
    L = C.CDLL(capi.LIB_PATH)
    L.rg_last_error.restype = C.c_char_p
    for name in ("rg_l0_status", "rg_l0_poll_status", "rg_debug_fetch", "rg_launch_count"):
        getattr(L, name).restype = C.c_int64
    L.rg_stream.restype = VP
    return L


def _refused(rc, message, expect_rc=1):
    assert rc == expect_rc
    assert capi.lib().rg_last_error().decode() == message


def test_single_kind_entry_points_refuse_the_other_kind(pb):
    L = _own_lib()
    s1, s2 = pb.gpu_step1(), _step2(pb)
    h1, h2 = s1.h, s2.h
    buf = np.zeros(1 << 20, dtype=np.float64)                    # room for whatever a call might (wrongly) write
    p = buf.ctypes.data_as(VP)
    i64 = C.c_int64
    out = capi.S2Out(*([buf.ctypes.data] * 12))
    bt = capi.S2BtChr(*([buf.ctypes.data] * 7))
    ic = capi.S2IntChr(buf.ctypes.data, 0, None, None, None)
    io = capi.S2IntOpts(1000.0, 5.0, 0, 0, 0)
    offs = np.zeros(8, dtype=np.uint64)

    def call(name, argtypes, *args):
        fn = getattr(L, name)
        fn.argtypes = argtypes
        return fn(*args)

    # Step-1 entry points on the Step-2 handle
    _refused(call("rg_l0_block_bed", [VP, VP, i64, C.c_int32, VP, C.c_int32, C.c_int32], h2, p, 160, 8, None, 0, 0),
             NOT_S1)
    _refused(call("rg_l0_block_dosage_u8", [VP, VP, VP, i64, C.c_int32, VP, C.c_int32, C.c_int32],
                  h2, p, p, 640, 8, None, 0, 0), NOT_S1)
    _refused(call("rg_l0_block_f64", [VP, VP, i64, C.c_int32, VP, C.c_int32], h2, p, 640, 8, None, 0), NOT_S1)
    _refused(call("rg_l0_wait_input", [VP], h2), NOT_S1)
    _refused(call("rg_l0_poll_status", [VP], h2), NOT_S1, -1)
    _refused(call("rg_l0_fetch_W", [VP, C.c_int32, C.c_int32, VP], h2, 0, 0, p), NOT_S1)
    _refused(call("rg_l0_load_W", [VP, C.c_int32, C.c_int32, VP], h2, 0, 0, p), NOT_S1)
    _refused(call("rg_l1_fit", [VP] * 4, h2, p, p, p), NOT_S1)
    _refused(call("rg_l1_fit_bt", [VP] * 6, h2, p, p, p, p, p), NOT_S1)
    _refused(call("rg_loco", [VP] * 3, h2, p, p), NOT_S1)
    _refused(call("rg_prs", [VP] * 2, h2, p), NOT_S1)
    _refused(call("rg_W_set_owned", [VP] * 2, h2, p), NOT_S1)
    _refused(call("rg_W_export", [VP] * 2, h2, p), NOT_S1)
    _refused(call("rg_W_attach_peer", [VP] * 3, h2, p, p), NOT_S1)
    _refused(call("rg_l1_select", [VP] * 2, h2, p), NOT_S1)
    _refused(call("rg_W_info", [VP, C.c_int32, VP, VP, VP], h2, 0, p, p, p), NOT_S1)
    _refused(call("rg_W_attach_local", [VP] * 3, h1, h2, p), NOT_S1)
    _refused(call("rg_W_attach_local", [VP] * 3, h2, h1, p), NOT_S1)
    _refused(call("rg_l0_solver_stats", [VP] * 3, h2, p, p), NOT_S1)
    _refused(call("rg_l0_wait_input", [VP], None), "not a Step-1 handle")                 # a null handle
    _refused(call("rg_l0_solver_stats", [VP] * 3, None, p, p), "not a Step-1 handle")

    # Step-2 entry points on the Step-1 handle
    _refused(call("rg_s2_set_chr", [VP] * 3, h1, p, p), NOT_S2)
    _refused(call("rg_s2_set_sex", [VP] * 2, h1, p), NOT_S2)
    _refused(call("rg_s2_set_non_par", [VP, VP, C.c_int32], h1, p, 8), NOT_S2)
    dev = VP()
    _refused(call("rg_s2_stage", [VP, C.c_int32, VP, i64, VP], h1, 0, p, 64, C.byref(dev)), NOT_S2)
    _refused(call("rg_s2_block_bed", [VP, VP, i64, C.c_int32, VP, C.c_int32, C.c_double, VP],
                  h1, p, 160, 8, None, 0, 5.0, C.byref(out)), NOT_S2)
    _refused(call("rg_s2_set_chr_bt", [VP] * 2, h1, C.byref(bt)), NOT_S2)
    for name in ("rg_s2_block_bgen8_bt", "rg_s2_block_bgen8"):
        _refused(call(name, [VP, VP, VP, i64, C.c_int32, VP, C.c_int32, C.c_double, VP, VP],
                      h1, p, p, 640, 8, None, 0, 5.0, C.byref(out), p), NOT_S2)
    _refused(call("rg_s2_block_bed_bt", [VP, VP, i64, C.c_int32, VP, C.c_int32, C.c_double, VP],
                  h1, p, 160, 8, None, 0, 5.0, C.byref(out)), NOT_S2)
    _refused(call("rg_bgen_inflate", [VP, VP, VP, i64, C.c_int32, VP, VP],
                  h1, p, offs.ctypes.data_as(VP), 640, 4, C.byref(dev), C.byref(dev)), NOT_S2)
    _refused(call("rg_s2_spa", [VP, C.c_int32] + [VP] * 4, h1, 1, p, p, p, p), NOT_S2)
    _refused(call("rg_s2_firth", [VP, C.c_int32] + [VP] * 6, h1, 1, p, p, p, p, p, p), NOT_S2)
    _refused(call("rg_s2_set_interaction", [VP] * 2, h1, C.byref(ic)), NOT_S2)
    _refused(call("rg_s2_interaction", [VP] * 5, h1, C.byref(io), p, p, p), NOT_S2)

    # the entry points that serve both kinds
    assert call("rg_l0_status", [VP], h2) == 0
    L.rg_get_timing.argtypes = [VP, C.c_char_p, VP, VP]
    L.rg_debug_fetch.argtypes = [VP, C.c_char_p, VP, i64]
    for name in ("rg_sync", "rg_fence", "rg_stream", "rg_launch_count", "rg_timing_reset"):
        getattr(L, name).argtypes = [VP]
    L.rg_set_timing.argtypes = [VP, C.c_int32]
    for h in (h1, h2):
        assert L.rg_sync(h) == 0 and L.rg_fence(h) == 0
        assert L.rg_stream(h)
        assert L.rg_launch_count(h) >= 0
        assert L.rg_set_timing(h, 1) == 0 and L.rg_timing_reset(h) == 0 and L.rg_set_timing(h, 0) == 0
        tot, n = C.c_double(-1.0), C.c_int64(-1)
        assert L.rg_get_timing(h, b"l0_predict", C.byref(tot), C.byref(n)) == 0 and n.value == 0
        _refused(L.rg_debug_fetch(h, b"pgen_rows", p, 8), "pgen_rows: no rg_pgen_decode has filled it", -1)
    assert s2.debug("s2_paths", np.int64, 8)[5] == 640                               # Npad

    # both handles still work, bit for bit like fresh ones
    W, W_fresh = _s1_W(pb, s1), _s1_W(pb, pb.gpu_step1())
    for a, b in zip(W, W_fresh):
        np.testing.assert_array_equal(a, b)
    o, o_fresh = _s2_block(pb, s2), _s2_block(pb, _step2(pb))
    for k in o:
        np.testing.assert_array_equal(o[k], o_fresh[k])
    s1.close(); s2.close()


def test_failed_create_then_valid_create(pb):
    pr = pb.prep
    bad = np.array(pb.fold_sizes, dtype=np.int64).copy()
    bad[0] += 1
    with pytest.raises(capi.RgError, match="fold sizes must sum to n_samples"):
        capi.Step1(pr.X, pr.Y, pr.mask, pr.in_analysis, bad, pb.lam, pr.neff, pr.n_analyzed, pb.bsize, len(pb.blocks))
    W = _s1_W(pb, pb.gpu_step1())
    W_o, _, _, _ = pb.oracle_l0(0)
    for ph in range(len(W)):
        assert np.abs(W[ph] - W_o[ph]).max() <= 1e-9 * np.abs(W_o[ph]).max()


def test_destroy_with_work_in_flight(pb):
    W_ref = _s1_W(pb, pb.gpu_step1())
    o_ref = _s2_block(pb, _step2(pb))
    # Step 1: host rows (lane copy streams), timing events never read, the poll stream; destroyed without a sync
    st = pb.gpu_step1()
    st.set_timing(True)
    for b in range(len(pb.blocks)):
        pb.gpu_l0_block(st, b)
    assert st.poll_status() >= 0
    st.close()
    # Step 2: every staging slot with a copy in flight
    s2 = _step2(pb)
    _s2_block(pb, s2)
    host = np.ones(1 << 22, dtype=np.uint8)
    for slot in range(4):
        s2.stage(slot, host.ctypes.data, host.size)
    s2.close()
    W = _s1_W(pb, pb.gpu_step1())
    for a, b in zip(W, W_ref):
        np.testing.assert_array_equal(a, b)
    o = _s2_block(pb, _step2(pb))
    for k in o:
        np.testing.assert_array_equal(o[k], o_ref[k])
