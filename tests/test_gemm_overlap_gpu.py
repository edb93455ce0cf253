"""The split-operand GEMM with its epilogue in a warpgroup of its own, at tile counts around the SM count.

The epilogue warpgroup runs tile t's epilogue while the consumers run tile t + 1's main loop, handing the accumulator
tile over through two mbarriers. What can go wrong there depends on how many tiles each persistent CTA runs: none
after the first (fewer tiles than SMs), exactly one (one tile per SM), a second one on a single CTA (one tile more than
SMs), or many, where the hand-off's phases wrap. The encode and dcode GEMMs of a training step run ceil(B / 128) x
ceil(n / 128) tiles per model, and these shapes put them in each of those cases:

  fewer      M = 1, B = 1000, n = 1024      64 tiles
  one_each   M = 1, rows x columns = SMs    one tile per SM (H100 SXM, 132 SMs: B = 1403, n = 1536)
  one_more   M = 1, rows x columns = SMs+1  one CTA runs a second tile (133: B = 2427, n = 896)
  many       M = 2, B = 4001, n = 1040       576 tiles, ragged in every dimension

The last row tile is partial in every case; d = 256 keeps every reduction inside the lengths the bars were set at.

Each is checked against fp64 per (model, 128 x 128 tile) with the bars of tests/test_tile_bounds_gpu.py
(oracle/tile_bounds.py), at initialisation and after a step, in both arithmetics; and two runs of the same steps on
fresh ensembles must return bitwise equal tensors, since the hand-off changes when an epilogue runs, never what it sums.
"""
import pytest
import torch

import engine_cases as EC

pytestmark = pytest.mark.gpu

D = 256
CASES = ["fewer", "one_each", "one_more", "many"]


def grid_shape(tiles):
    """(n, B) whose encode GEMM has exactly `tiles` tiles: the column count the largest divisor of `tiles` up to 16
    (a prime count gets one row tile), the last row tile partial."""
    cols = max([c for c in range(1, 17) if tiles % c == 0 and tiles // c > 1] or [tiles])
    return 128 * cols, 128 * (tiles // cols) - 5


def shape(case):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if case in ("one_each", "one_more"):
        return (1, D) + grid_shape(sms if case == "one_each" else sms + 1)
    return {"fewer": (1, D, 1024, 1000), "many": (2, D, 1040, 4001)}[case]


def encode_tiles(M, n, B):
    return M * ((B + 127) // 128) * ((n + 127) // 128)


def test_tile_counts_around_the_sm_count():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = {c: encode_tiles(shape(c)[0], shape(c)[2], shape(c)[3]) for c in CASES}
    assert tiles["fewer"] < sms and tiles["one_each"] == sms and tiles["one_more"] == sms + 1
    assert tiles["many"] > 4 * sms, tiles


@pytest.mark.parametrize("arith", EC.ARITHS)
@pytest.mark.parametrize("case", CASES)
def test_every_tile_against_fp64(case, arith):
    shp = shape(case)
    M, d, n, _ = shp
    models, sig = EC.make_models("tied", M, d, n, 11)
    EC.run_case(f"overlap {case}", "tied", models, sig, arith, shp, False, True, steps=1, seed=700)


@pytest.mark.parametrize("arith", EC.ARITHS)
@pytest.mark.parametrize("case", CASES)
def test_two_runs_bitwise_equal(case, arith):
    shp = shape(case)
    M, d, n, _ = shp
    models, sig = EC.make_models("tied", M, d, n, 12)
    la, lb = EC.bitwise_reruns(models, sig, arith, shp, (900, 990))
    assert la == lb
