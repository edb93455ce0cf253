"""The split-operand GEMM in clusters of two CTAs that share each A tile by TMA multicast, and in clusters of one.

launch_gemm (sce_gemm.cuh) groups the CTAs in pairs along N where a model's column-tile count is even and each tile's
K loop runs at least 64 K blocks over its operand sets (K block 64 under f16f8, 32 under bf16x3), and runs them singly
otherwise. The pair splits the loads of every A tile between its two CTAs and frees a stage only once the consumers of
both are done with it; none of that may change a value. These tests check it:

  - the standalone check (tests/csrc/gemm_cluster_selftest.cu): every configuration libsce launches, at cluster sizes 1
    and 2, bitwise equal across runs and sizes and against the fp64 product of the planes; odd and even column-tile
    counts, ragged edges, two operand sets, tile counts around twice the SM count and a pair-indexed schedule;
  - training steps at shapes where the decode and weight-gradient GEMMs take clusters of two (`even`), where every GEMM
    takes clusters of one (`odd`: one column tile of d), or some of each (`mixed`), checked per (model, 128 x 128
    tile) against fp64 with the bars of tests/test_tile_bounds_gpu.py, and two runs on fresh ensembles bitwise equal.

  even   M = 2, d = 256, n = 4096, B = 2048   decode K = 4096, weight gradient 2 x 2048: both pairs under either arith
  odd    M = 2, d = 128, n = 640,  B = 2048   one column tile of d: singles throughout
  mixed  M = 3, d = 256, n = 640,  B = 2049   decode singles (K = 640), weight gradient pairs (2 x 2049)
"""
import os
import subprocess

import pytest

import engine_cases as EC

pytestmark = pytest.mark.gpu

SHAPES = {"even": (2, 256, 4096, 2048), "odd": (2, 128, 640, 2048), "mixed": (3, 256, 640, 2049)}


def cluster_sizes(shape, bk=64):
    """Cluster size launch_gemm takes for each GEMM of a training step at `shape` (M, d, n, B) and K block `bk`."""
    _, d, n, B = shape
    gemms = {"encode": (n, d, 1), "decode": (d, n, 1), "dcode": (n, d, 1), "dw": (d, B, 2)}   # N, K, sets
    return {g: 2 if -(-N // 128) % 2 == 0 and sets * -(-K // bk) >= 64 else 1 for g, (N, K, sets) in gemms.items()}


def test_shapes_cover_both_cluster_sizes():
    for bk in (64, 32):
        assert cluster_sizes(SHAPES["even"], bk) == {"encode": 1, "decode": 2, "dcode": 1, "dw": 2}
        assert set(cluster_sizes(SHAPES["odd"], bk).values()) == {1}
        assert cluster_sizes(SHAPES["mixed"], bk)["dw"] == 2
    assert cluster_sizes(SHAPES["mixed"], 64)["decode"] == 1


def test_gemm_cluster_selftest(tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "build", "gemm_cluster_selftest")
    if not os.path.exists(exe):   # build() makes it; a tree built with `make` alone may not have it
        exe = str(tmp_path / "gemm_cluster_selftest")
        subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-o", exe,
                        os.path.join(root, "tests", "csrc", "gemm_cluster_selftest.cu")], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1800)
    print(r.stdout)
    assert r.returncode == 0 and "ALL PASS" in r.stdout, r.stdout[-4000:] + r.stderr[-2000:]
    assert r.stdout.count("cluster sizes 1, 1, 2, 2") >= 20 and r.stdout.count("cluster sizes 1, 1 ") >= 12


@pytest.mark.parametrize("arith", EC.ARITHS)
@pytest.mark.parametrize("case", sorted(SHAPES))
def test_every_tile_against_fp64(case, arith):
    shp = SHAPES[case]
    M, d, n, _ = shp
    models, sig = EC.make_models("tied", M, d, n, 21)
    EC.run_case(f"cluster {case}", "tied", models, sig, arith, shp, False, True, steps=1, seed=710)


@pytest.mark.parametrize("arith", EC.ARITHS)
@pytest.mark.parametrize("case", sorted(SHAPES))
def test_two_runs_bitwise_equal(case, arith):
    shp = SHAPES[case]
    M, d, n, _ = shp
    models, sig = EC.make_models("tied", M, d, n, 22)
    EC.bitwise_reruns(models, sig, arith, shp, (910, 995))
