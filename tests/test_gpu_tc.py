"""GPU: the wgmma (TF32 hi/lo split) Linear forward and weight gradient vs fp64, each in a subprocess (a descriptor
mistake would fault the kernel and poison this process's CUDA context)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_tensor_core_linear_matches_fp64():
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "tc_check.py")], capture_output=True, text=True,
                         timeout=300)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    assert "tc linear ok" in res.stdout


def test_tensor_core_weight_gradient_matches_fp64():
    res = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "tc_dw_check.py")], capture_output=True, text=True,
                         timeout=300)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    assert "tc dw ok" in res.stdout
