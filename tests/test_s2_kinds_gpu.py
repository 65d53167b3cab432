"""One Step-2 handle that holds both trait kinds.

rg_s2_set_chr builds the quantitative-trait state of a chromosome and rg_s2_set_chr_bt the binary-trait one, each with
its own feature rows and its own digit rows for the tensor-core statistics.  In whatever order one handle receives the
chromosome calls of both kinds and blocks of all four routes, each block must give bit for bit what the same block gives
on a fresh handle that holds only its own kind: every rg_s2_out field, the INFO scores, the sums hooks and the shape
"s2_paths" reports.  Firth and SPA read the resident block, so they are refused unless the last block call was a
binary-trait one and no rg_s2_set_chr_bt came after it; rg_s2_interaction is refused after a binary-trait block.
"""
import numpy as np
import pytest

from oracle import step2_bt
from regenie_b200 import capi, synth
from test_s2_paths_gpu import _bt_problem, _probs

pytestmark = pytest.mark.gpu
N, P, C, BS = 1500, 2, 3, 160
KIND = {"bed": "qt", "bgen8": "qt", "bed_bt": "bt", "bgen8_bt": "bt"}
NOT_BT = "needs a resident binary-trait block"


@pytest.fixture(scope="module")
def pb():
    b = _bt_problem(N, P, C, seed=5)
    rng = np.random.default_rng(5)
    chrs = []
    for _ in range(2):                            # two chromosomes: new residuals, new LOCO offsets
        blup = 0.3 * rng.standard_normal((N, P)) * b["mask"]
        sts = [step2_bt.BtChrom(b["Y"][:, j], b["X"], blup[:, j], b["mask"][:, j]) for j in range(P)]
        bt = (np.stack([s.gamma_sqrt_mask for s in sts], 1), np.stack([s.gamma_sqrt for s in sts], 1),
              np.stack([s.yres for s in sts], 1), [s.Xg for s in sts], b["Y"],
              np.stack([s.cov_blup_offset for s in sts], 1), np.stack([s.phat for s in sts], 1))
        qt = (np.asfortranarray(rng.standard_normal((N, P)) * b["mask"]), rng.uniform(0.5, 2.0, P))
        chrs.append(dict(qt=qt, bt=bt))
    probs, miss = _probs(rng, BS, N)
    return dict(b=b, chrs=chrs, packed=synth.pack_bed(synth.genotypes(N, BS, seed=5, miss=0.02)), probs=probs,
                miss=miss, fresh={})


def _handle(pb):
    b = pb["b"]
    return capi.Step2(b["X"], b["mask"], b["ia"], b["n_an"], BS)


def _set_chr(st, pb, kind, chrom):
    if kind == "qt":
        st.set_chr(*pb["chrs"][chrom]["qt"])
    else:
        st.set_chr_bt(*pb["chrs"][chrom]["bt"])


def _block(st, pb, route):
    """The outputs of one block, the sums hooks its route fills and the shape "s2_paths" reports for it."""
    if route in ("bed", "bed_bt"):
        o = getattr(st, "block_" + route)(pb["packed"])
    else:
        o = getattr(st, "block_" + route)(pb["probs"], pb["miss"])
    o["s2_paths"] = st.debug("s2_paths", np.int64, 8)[:6]
    hooks = (["s2_sums"] if KIND[route] == "qt" else []) + (["bt_sums", "bt_nnz", "bt_n510"] if route != "bed" else [])
    for n in hooks:
        o[n] = st.debug(n, np.float64, 1 << 20)
    return o


def _fresh(pb, route, chrom):
    """_block on a handle that has seen only the chromosome call of the route's kind."""
    key = (route, chrom)
    if key not in pb["fresh"]:
        st = _handle(pb)
        _set_chr(st, pb, KIND[route], chrom)
        pb["fresh"][key] = _block(st, pb, route), st
    return pb["fresh"][key]


def _same(got, want, what):
    assert got.keys() == want.keys(), what
    for k in want:
        np.testing.assert_array_equal(got[k], want[k], err_msg="%s: %s" % (what, k))


ORDERS = [
    [("qt", 0), ("bt", 0), "bed", "bed_bt", "bgen8", "bgen8_bt"],
    [("bt", 0), ("qt", 0), "bed_bt", "bed", "bgen8_bt", "bgen8"],
    [("qt", 0), "bed", ("bt", 0), "bed", "bgen8_bt", ("qt", 1), "bed_bt", "bed", ("bt", 1), "bgen8", "bed_bt", "bed"],
]


@pytest.mark.parametrize("order", range(len(ORDERS)))
def test_interleaved_kinds_match_single_kind_handles(pb, order):
    st = _handle(pb)
    chrom = {}
    for step in ORDERS[order]:
        if isinstance(step, tuple):
            _set_chr(st, pb, *step)
            chrom[step[0]] = step[1]
        else:
            _same(_block(st, pb, step), _fresh(pb, step, chrom[KIND[step]])[0], step)
    st.close()


def _selections(o):
    return np.nonzero(((o["flags"] & 17) == 0)[:, None] & (o["mac"] >= 5.0) & (np.abs(o["stat"]) > 0.5))


def _firth_spa(st, v, t):
    beta, se, lrt, fst = st.firth(v, t)
    pv, sst = st.spa(v, t)
    return dict(beta=beta, se=se, lrt=lrt, firth_status=fst, pval=pv, spa_status=sst)


def test_firth_spa_need_a_resident_binary_trait_block(pb):
    st = _handle(pb)
    _set_chr(st, pb, "qt", 0)
    _set_chr(st, pb, "bt", 0)

    def like_fresh(route, chrom):
        o, fresh = _fresh(pb, route, chrom)
        v, t = _selections(o)
        assert len(v) > 20
        _same(_firth_spa(st, v, t), _firth_spa(fresh, v, t), route)

    def refused():
        for call in (st.firth, st.spa):
            with pytest.raises(capi.RgError, match=NOT_BT):
                call([0], [0])

    _block(st, pb, "bgen8_bt")
    like_fresh("bgen8_bt", 0)
    _block(st, pb, "bed")                         # a quantitative-trait block replaces the binary-trait one
    refused()
    _block(st, pb, "bgen8")
    refused()
    _block(st, pb, "bed_bt")                      # the next binary-trait block
    like_fresh("bed_bt", 0)
    _set_chr(st, pb, "qt", 1)                     # a chromosome call of the other kind leaves it resident
    like_fresh("bed_bt", 0)
    _set_chr(st, pb, "bt", 1)                     # one of its own kind ends it
    refused()
    _block(st, pb, "bgen8_bt")
    like_fresh("bgen8_bt", 1)
    st.close()


def test_interaction_refused_after_a_binary_trait_block(pb):
    E = np.random.default_rng(9).standard_normal(N)
    st = _handle(pb)
    _set_chr(st, pb, "bt", 0)
    _set_chr(st, pb, "qt", 0)
    st.set_interaction(E)
    fresh = _handle(pb)
    _set_chr(fresh, pb, "qt", 0)
    fresh.set_interaction(E)
    for route in ("bgen8", "bed"):
        _block(st, pb, route)
        _block(fresh, pb, route)
        for a, b in zip(st.interaction(), fresh.interaction()):
            np.testing.assert_array_equal(a, b, err_msg=route)
    for route in ("bgen8_bt", "bed_bt"):
        _block(st, pb, route)
        with pytest.raises(capi.RgError, match="rg_s2_interaction needs the block of the last"):
            st.interaction()
    st.close()
    fresh.close()
