"""The batch-major copies of the code's and g's 8-bit planes, written by the encode and decode epilogues of an f16f8
training step whose weight gradient runs on native E5M2 wgmma (dw_native: a dense plan that is not launch-bound).

The copies are stored straight from the epilogues' registers, clipped at the batch's B rows and at the matrix's columns.
Each case builds a plan with batch_max = 1210 (a padded pitch of 1216), runs a full batch to leave stale rows, then a
batch of B rows:
  - the code read back after grads_batch takes its residual plane from the batch-major copy; it must be bitwise equal to
    the code read back after forward_batch on the same parameters and rows, which takes it from the row-major plane;
  - the weight gradients and the code of the same calls are checked per (model, 128 x 128 tile) against fp64 with the
    bars of tests/test_tile_bounds_gpu.py (oracle/tile_bounds.py).
Tied plans run every B in {1210, 1037, 33, 5} with fp16-exact and fp32 inputs; the other dense signatures on this path
(untied: c^T g is a GEMM of its own; masked; learned centre: the decode epilogue with column sums of g; non-negative
tied: a shifted batch) run one ragged B each.
"""
import pytest

import engine_cases as EC
from oracle.plan_paths import launch_bound

pytestmark = pytest.mark.gpu

M, D, N, BMAX = 4, 512, 4096, 1210


def run(variant, B, fp16_values, seed):
    assert not launch_bound(M, BMAX, N, D)
    models, sig = EC.make_models(variant, M, D, N, seed)
    ens = EC.ensemble(models, sig, "f16f8")
    ens.forward_batch(EC.batch(M, BMAX, D, seed + 1, False, fp16_values))   # batch_max = BMAX; stale rows behind B
    assert ens.resolved_arith() == "f16f8"
    X = EC.batch(M, B, D, seed + 2, False, fp16_values)
    _, (_, aux) = ens.grads_batch(X)
    code_bwd = aux["c"].dense().clone()
    _, aux = ens.forward_batch(X)
    code_fwd = aux["c"].dense().clone()
    assert code_bwd.shape == (M, B, N)
    assert EC.raw(code_bwd) == EC.raw(code_fwd), (variant, B, "code from the batch-major copy differs from the row-major one")
    EC.check(f"batch-major {variant} B={B} {'fp16' if fp16_values else 'fp32'}", variant, ens, X, False, "f16f8")


@pytest.mark.parametrize("inputs", ["fp16", "fp32"])
@pytest.mark.parametrize("B", [BMAX, 1037, 33, 5])
def test_tied_ragged_batches(B, inputs):
    run("tied", B, inputs == "fp16", 31)


@pytest.mark.parametrize("variant", ["untied", "masked_tied", "learned_center", "positive_tied"])
def test_other_dense_signatures(variant):
    run(variant, 1037, False, 41)
