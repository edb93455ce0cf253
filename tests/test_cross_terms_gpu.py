"""Accuracy of the f16f8 cross-term accumulation: E5M2 wgmma (both operands K-major) against fp16 wgmma on widened
tiles, each against the fp64 sum of the same E5M2 products at reduction lengths 512, 4096 and 16384
(tests/csrc/cross_term_selftest.cu)."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu


def test_cross_term_accumulation(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "cross_term_selftest")
    subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-o", exe,
                    os.path.join(root, "tests", "csrc", "cross_term_selftest.cu")], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0 and "ALL PASS" in r.stdout, r.stdout[-4000:] + r.stderr[-2000:]
