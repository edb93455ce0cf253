"""The split-operand GEMM on 192-row output tiles (BM = kBMTall in sce_gemm.cuh), which dense f16f8 training plans take
for decode and the native weight gradient.

A tall tile changes how many rows each CTA covers and runs its epilogue in two rounds, but not the K sweep of any output
element, and every epilogue share keeps the 128-row tiling's coordinates. So its outputs must be bitwise those of the
128-row tiles:

  - the standalone check (tests/csrc/gemm_tall_selftest.cu): decode with every output EpiDecodeT has (g planes, x^,
    loss partials, column sums of g, per-row partials of r^2, batch-major copies of g's 8-bit planes) and the weight
    gradient with set 0's residual flag on and off, at cluster sizes 1 and 2, at 4096, 1210, 1037, 33 and 5 rows, d = 64
    and 256, and at config 2's shapes, bitwise equal to the 128-row tiles, slots no share writes included;
  - training steps of tied, untied, learned-centre and non-negative tied plans, whose decode and weight gradient run on
    tall tiles, checked per (model, 128 x 128 tile) against fp64 with the bars of tests/test_tile_bounds_gpu.py, at a
    batch whose last 192-row tile is ragged.
"""
import os
import subprocess

import pytest

import engine_cases as EC

pytestmark = pytest.mark.gpu


def test_gemm_tall_selftest(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "build", "gemm_tall_selftest")
    if not os.path.exists(exe):   # build() makes it; a tree built with `make` alone may not have it
        exe = str(tmp_path / "gemm_tall_selftest")
        subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-o", exe,
                        os.path.join(root, "tests", "csrc", "gemm_tall_selftest.cu")], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1800)
    print(r.stdout)
    assert r.returncode == 0 and "ALL PASS" in r.stdout, r.stdout[-4000:] + r.stderr[-2000:]
    # every case ran both tile heights; the d = 256 cases (two column tiles) at cluster size 2 as well
    assert r.stdout.count("PASS decode") == 11 and r.stdout.count("PASS dw") == 21
    assert r.stdout.count("128/1, 192/1, 128/2, 192/2") == 5 + 10 + 2


# M, d, n, B: not launch-bound (the plan takes dw_native, hence tall tiles); decode over 8001 rows (the last 192-row tile
# ragged), the weight gradient over n = 1040 rows (a partial 128-row tile, covered by 192-row tiles to 1152)
SHAPE = (4, 400, 1040, 8001)


@pytest.mark.parametrize("variant", ["tied", "untied", "learned_center", "positive_tied"])
def test_tall_tile_plans_every_tile(variant):
    M, d, n, B = SHAPE
    assert 30.0 * M * B * n * d >= 3e11   # not launch-bound (plan_config)
    models, sig = EC.make_models(variant, M, d, n, 7)
    # (the learned-centre plan holds one centred batch per model; it is fed one, as its own tests do)
    per_model = variant == "learned_center"
    EC.run_case(f"tall tiles {variant}", variant, models, sig, "f16f8", SHAPE, per_model, True, seed=700)
