"""The f16f8 weight-gradient GEMM on native E5M2 wgmma with mixed operand layouts (fp16 planes MN-major, 8-bit planes
K-major from batch-major copies), two operand sets with a flagged all-zero residual plane, ragged K and partial tiles:
against the fp64 value of the same planes and against the widened instantiation (tests/csrc/native_dw_selftest.cu)."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu


def test_native_weight_gradient(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "native_dw_selftest")
    subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-o", exe,
                    os.path.join(root, "tests", "csrc", "native_dw_selftest.cu")], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    print(r.stdout)
    assert r.returncode == 0 and "ALL PASS" in r.stdout, r.stdout[-4000:] + r.stderr[-2000:]
