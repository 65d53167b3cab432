"""Step 1 sharded over ranks (SURVEY 8(e)): level-0 blocks per rank, W tiles stored into the owner's HBM over
CUDA IPC, level 1 per phenotype owner; sharded == unsharded bit for bit (test/test_bash.sh:127-137 analogue)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ngpu():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=30).stdout
        return sum(1 for l in out.splitlines() if l.startswith("GPU "))
    except Exception:
        return 0


@pytest.mark.parametrize("world", [2, 3])
def test_step1_sharded_equals_unsharded(world):
    if _ngpu() < world:
        pytest.skip("needs %d GPUs" % world)
    env = dict(os.environ, MASTER_ADDR="127.0.0.1")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
           "127.0.0.1", "--master-port", str(29500 + world), os.path.join(ROOT, "tests", "mgpu_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("MGPU_OK") == world, r.stdout[-2000:]


@pytest.mark.parametrize("loocv", [False, True])
def test_driver_gpus_n_writes_the_single_gpu_files(tmp_path, golden_dir, loocv):
    """`rgb200 --gpus 2` (one host thread per GPU, level-0 blocks sharded, level 1 by phenotype, tiles stored into the
    owner's HBM through peer access) writes .loco / _pred.list files byte-identical to the single-GPU run - the
    reference's own invariant for its multi-job mode (test/test_bash.sh:127-137)."""
    if _ngpu() < 2:
        pytest.skip("needs two GPUs")
    rgb = os.path.join(ROOT, "regenie_b200", "rgb200")
    base = ["--step", "1", "--bed", golden_dir + "/example", "--phenoFile", golden_dir + "/phenotype.txt", "--covarFile",
            golden_dir + "/covariates.txt", "--bsize", "100"] + (["--loocv"] if loocv else [])
    outs = []
    for g in (1, 2):
        out = str(tmp_path / ("g%d" % g))
        r = subprocess.run([rgb] + base + ["--gpus", str(g), "--out", out], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        outs.append(out)
    for k in (1, 2):
        a = open(outs[0] + "_%d.loco" % k, "rb").read()
        b = open(outs[1] + "_%d.loco" % k, "rb").read()
        assert a == b
