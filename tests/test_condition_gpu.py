"""Conditional analysis through the real library: `rgb200` Step 1 then Step 2 conditioned on variants of the main file
or of an external fileset gives the .loco / .regenie files of the unconditioned runs whose covariate file carries the
conditioning genotypes (tests/condition_oracle.py), byte for byte."""
import os
import subprocess

import pytest

import condition_oracle as co

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RGB = os.path.join(ROOT, "regenie_b200", "rgb200")


def run(args):
    r = subprocess.run([RGB] + [str(a) for a in args], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    return r.stdout


def read(path):
    return open(path).read()


@pytest.mark.parametrize("main,bt,source", [("bed", False, None), ("bed", True, None), ("bed", False, "bgen"),
                                            ("pgen", True, "bed"), ("bgen", False, None), ("bgen", True, "pgen")])
def test_conditioned_steps_equal_covariate_runs(tmp_path, golden_dir, main, bt, source):
    co.check_equivalence(run, read, tmp_path, golden_dir, main, bt, source, step1=True)
