"""The persistent INT8 prediction kernel: a grid of min(items, SMs) CTAs, each walking (sample tile, output group) items
b, b + grid, ... with its epilogue warpgroup one item behind its MMA warpgroups.  Each shape's raw predictions against
the long-double recomputation from the kernel's own coefficients and digits (test_l0_paths_gpu), and W against the
oracle:
  * fewer items than SMs: 1500 samples (12 sample tiles) x 2 output groups, blocks of 2048 (2 rows_p = 4096, the last
    INT8 shape), 1000 and 129 SNPs, C = 64 covariate columns (kMaxCov);
  * more items than SMs, not a multiple of the grid: 20000 samples x 2 output groups, so every CTA runs several items
    and crosses fold boundaries (five folds) inside its walk, blocks of 100 and 1 SNPs (rows_p = 128, two k-blocks per
    item: the stage ring runs two items ahead).
P = 11 traits x R = 5 ridge values = 55 outputs: the second group of 50 holds 5.  Samples without a phenotype are
masked."""
import numpy as np
import pytest

from test_l0_paths_gpu import _calls, _check_W, _fileset, _run_block, check_raw_predictions

pytestmark = pytest.mark.gpu
P, R = 11, 5


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("N, chrom, C, bsize, many", [
    (1500, [2048, 1000, 129], 64, 2048, False),
    (20000, [100, 1], 3, 100, True),
], ids=["fewer-items-than-sms", "more-items-than-sms"])
def test_persistent_walk_within_the_error_bound(tmp_path, monkeypatch, N, chrom, C, bsize, many):
    monkeypatch.setenv("RG_B200_LANES", "2")
    pb = _fileset(tmp_path, N, chrom, P, C, 0.02, 7 + len(chrom), bsize=bsize)
    assert [b[2] for b in pb.blocks] == chrom
    assert pb.prep.ncov == C
    assert (pb.prep.mask == 0).any()
    st = pb.gpu_step1()
    sms = _sm_count()
    for b in range(len(chrom)):
        hk = _run_block(pb, st, b)
        assert hk["paths"][1] == 1, hk["paths"]
        items = (hk["Npad"] // 128) * 2               # 55 outputs: two groups
        if many:
            assert items > 2 * sms and items % sms != 0, (items, sms)
        else:
            assert items < sms, (items, sms)
        check_raw_predictions(hk, *_calls(pb, b), pb.prep.X, pb.prep.mask, pb.fold_sizes, power=chrom[b] > 1)
    for b in range(len(chrom)):
        _check_W(pb, st, b)
    st.close()
