"""Per-tile error bounds of the engine's row passes against fp64.

*** TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT PATH. *** (as oracle/tile_bounds.py)

The row passes (sce_second_moments, sce_ica_pass, sce_nmf_project, sce_nmf_grams, sce_nmf_residual; include/sce.h) write
their matrix outputs in 128 x 128 tiles, reduce their rows in slices and their vectors per row block. One norm-relative
number per output dilutes an error confined to one tile or one run of a vector by about 1/sqrt(tiles), so each output
is measured per tile with oracle/tile_bounds.py's tile_ratios against its absolute-product scale S: the fp64 formula with
every operand replaced by its absolute value, the size the rounding of a split-operand product can reach whatever the
cancellation in the product. Vectors are tiled in runs of 128.

For the B rows x_b, v_b = x_b - s (the NMF passes: v_b = max(x_b - s, 0)), V = [v_b] in fp64:
  second moments   gram = V^T V                  S = |V|^T |V|
                   col_sum = sum_b v_b           S = sum_b |v_b|
  FastICA          U = V unmix^T, T = tanh(a U)
                   gx = T^T V                    S = |T|^T |V| + a (|V| |unmix|^T)^T |V|
                       The first term is GEMM 2's own rounding. GEMM 1's error in u, at most eps |V| |unmix|^T, reaches t
                       through tanh' = a (1 - t^2) <= a, and gx through |v|: the second term.
                   g_sum = sum_b a (1 - t^2)     S = sum_b a (1 + 2 a |t| (|V| |unmix|^T))
                       The first term bounds a (1 - t^2) itself; d/du a (1 - t^2) = -2 a^2 t (1 - t^2), at most 2 a^2 |t|
                       in size, carries GEMM 1's error into g'.
  NMF projection   P = V M^T                     S_P = |V| |M|^T
                   norms = [sum_b max(P, 0)^2, sum_b min(P, 0)^2]
                                                 S = sum_b (2 |P| S_P + S_P^2) (both halves)
                       An element off by at most e S_P has its square within 2 e |P| S_P + e^2 S_P^2 of the true one,
                       at most e (2 |P| S_P + S_P^2) for e <= 1. (|P| + S_P)^2 would also count P^2, which no
                       rounding of P reaches: with it, a run of the norms scaled by 1 + 4 bar could stay within its bar.
  NMF Grams        wtw = W^T W                   S = |W|^T |W|
                   wtv = W^T V                   S = |W|^T V        (V >= 0)
  NMF residual     r = ||V - W H||^2 (one scalar), judged as |got - r| / (||V||^2 + || |W| |H| ||^2): the residual is a
                   sum of squares of differences that cancel at a good fit, so its own size is no measure of the rounding
                   of W H; the fp32 product's error in each element is at most a few ulps of (|W| |H|), and the square
                   of the difference moves by at most twice that times |V - W H| <= |V| + |W| |H|.

Everything is computed in fp64 on the device of the inputs, so that the largest cases (2^21 rows, d = 8192) stay fast.
"""
from __future__ import annotations

from typing import Dict

import torch

from oracle import tile_bounds as T

Tensor = torch.Tensor

ALPHA = 1.5        # the FastICA pass's tanh gain in the tests
# the outputs a row pass adds to instead of overwriting
ACCUMULATED = ("gram", "col_sum", "gx", "g_sum", "norms", "wtw", "wtv")
# (tile ratio, element maximum) per pass, output and arithmetic: max(twice the worst value measured, 2^-24) rounded up,
# set from measurement in tests/test_row_pass_tiles_gpu.py (see its docstring); "residual" is one relative error per call
BARS = {
    "moments": {"gram": {"bf16x3": (9.2e-6, 4.0e-5), "f16f8": (4.5e-5, 2.6e-4)},
                "col_sum": {"bf16x3": (6.0e-8, 1.1e-7), "f16f8": (6.0e-8, 1.1e-7)}},
    "ica": {"gx": {"bf16x3": (9.3e-7, 3.9e-6), "f16f8": (3.4e-6, 1.6e-5)},
            "g_sum": {"bf16x3": (4.3e-7, 2.8e-6), "f16f8": (1.5e-6, 7.7e-6)}},
    "project": {"p": {"bf16x3": (1.9e-6, 1.1e-5), "f16f8": (8.4e-6, 4.7e-5)},
                "norms": {"bf16x3": (3.4e-7, 1.5e-6), "f16f8": (1.7e-6, 6.4e-6)}},
    "grams": {"wtw": {"bf16x3": (5.4e-6, 2.7e-5), "f16f8": (4.2e-5, 1.9e-4)},
              "wtv": {"bf16x3": (6.5e-6, 2.8e-5), "f16f8": (4.1e-5, 1.9e-4)}},
    "residual": 6.0e-8,
}


def shifted(x: Tensor, shift: Tensor, clamp: bool = False) -> Tensor:
    """V = x - shift in fp64 (clamp: max(x - shift, 0), the NMF passes)."""
    v = x.double() - shift.double()[None, :]
    return v.clamp(min=0.0) if clamp else v


def moments(V: Tensor) -> Dict[str, tuple]:
    """{output: (reference, scale)} of sce_second_moments."""
    A = V.abs()
    return {"gram": (V.T @ V, A.T @ A), "col_sum": (V.sum(0), A.sum(0))}


def ica(V: Tensor, unmix: Tensor, alpha: float) -> Dict[str, tuple]:
    """{output: (reference, scale)} of sce_ica_pass."""
    U = unmix.double()
    A = V.abs()
    t = torch.tanh(alpha * (V @ U.T))
    SU = A @ U.abs().T
    gx = (t.T @ V, t.abs().T @ A + alpha * (SU.T @ A))
    g_sum = ((alpha * (1.0 - t * t)).sum(0), (alpha * (1.0 + 2.0 * alpha * t.abs() * SU)).sum(0))
    return {"gx": gx, "g_sum": g_sum}


def nmf_project(V: Tensor, M: Tensor) -> Dict[str, tuple]:
    """{output: (reference, scale)} of sce_nmf_project: P [B, k] and the norms [2k]."""
    M = M.double()
    P = V @ M.T
    SP = V.abs() @ M.abs().T
    sn = (2.0 * P.abs() * SP + SP * SP).sum(0)
    norms = torch.cat(((P.clamp(min=0.0) ** 2).sum(0), (P.clamp(max=0.0) ** 2).sum(0)))
    return {"p": (P, SP), "norms": (norms, torch.cat((sn, sn)))}


def nmf_grams(V: Tensor, W: Tensor) -> Dict[str, tuple]:
    """{output: (reference, scale)} of sce_nmf_grams."""
    W = W.double()
    A = W.abs()
    return {"wtw": (W.T @ W, A.T @ A), "wtv": (W.T @ V, A.T @ V.abs())}


def nmf_residual(V: Tensor, W: Tensor, H: Tensor) -> tuple:
    """(reference, scale) of sce_nmf_residual's sum ||V - W H||^2."""
    W, H = W.double(), H.double()
    want = float(((V - W @ H) ** 2).sum())
    scale = float((V * V).sum()) + float(((W.abs() @ H.abs()) ** 2).sum())
    return want, scale


def reference(kind: str, x: Tensor, shift: Tensor, mat: Tensor = None, alpha: float = 1.0) -> Dict[str, tuple]:
    """{output: (reference, scale)} of the row pass `kind` ("moments", "ica", "project", "grams") over the rows x, with
    its matrix (unmix, M or W)."""
    V = shifted(x, shift, clamp=kind in ("project", "grams"))
    if kind == "moments":
        return moments(V)
    if kind == "ica":
        return ica(V, mat, alpha)
    return nmf_project(V, mat) if kind == "project" else nmf_grams(V, mat)


# ---- the engine's slicing and cluster rules, restated (sce_rowpass.cu mom_slices, sce_gemm.cuh gemm_cluster_size)
ROWS_MAX, TARGET_TILES, SLICE_MIN, BLOCK_ROWS = 2048, 528, 256, 64


def mom_slices(d: int, B: int) -> tuple:
    """(S, R): a sliced pass's B rows of width d as S slices of R rows."""
    tiles = (-(-d // T.TILE)) ** 2
    s = min(-(-TARGET_TILES // tiles), -(-B // SLICE_MIN))
    s = max(s, -(-B // ROWS_MAX))
    R = -(-(-(-B // s)) // BLOCK_ROWS) * BLOCK_ROWS
    return -(-B // R), R


def cluster_size(n_cols: int, k: int, arith: str) -> int:
    """CTAs per cluster of a GEMM with n_cols output columns and reduction length k (one operand set; libsce's row
    passes run f16f8 on native E5M2 wgmma, never widened)."""
    bk = 64 if arith == "f16f8" else 32
    return 2 if -(-n_cols // T.TILE) % 2 == 0 and -(-k // bk) >= 64 else 1


def pass_clusters(kind: str, d: int, n: int, B: int, arith: str) -> Dict[str, int]:
    """Cluster size of each GEMM of a row pass: "gemm1" (U = V unmix^T, P = V M^T: K = d, N = n) and the sliced
    reductions (K = R): "sliced" (gram, gx: N = d), "wtw" (N = k), "wtv" (N = d)."""
    if kind == "project":
        return {"gemm1": cluster_size(n, d, arith)}
    _, R = mom_slices(d, B)
    if kind == "moments":
        return {"sliced": cluster_size(d, R, arith)}
    if kind == "ica":
        return {"gemm1": cluster_size(n, d, arith), "sliced": cluster_size(d, R, arith)}
    return {"wtw": cluster_size(n, R, arith), "wtv": cluster_size(d, R, arith)}
