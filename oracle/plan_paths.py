"""The engine's path choices, restated from plan_config and sce_prepare (sparse_coding_b200/csrc/sce_plan.cu).

*** TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT PATH. *** (as oracle/sae_oracle.py)

Tests compute from a shape which path a plan should take and pin it by the launch count of each call, so that a case
meant for one branch (the top-k gather decode and its k classes, the graph-replayed step) cannot drift to another.
"""
from __future__ import annotations


def launch_bound(M, batch_max, n, d):
    """plan_config's rule for replaying the step as a CUDA graph: ~30 M B n d tensor FLOPs below 3e11."""
    return 30.0 * M * batch_max * n * d < 3e11


def gather_slices(d, kmax):
    """Slices of the activation width topk_sparse_kernel runs per row for list capacity ``kmax`` (a multiple of 8):
    the fewest of 2, 4, 8 with 16-byte aligned slices of at most 512 columns whose shared memory fits 112 KiB; 0 if
    none does."""
    for s in (2, 4, 8):
        ds = d // s
        if d % (4 * s) or ds > 512:
            continue
        if kmax * ds * 4 + 9 * ds * 4 + kmax * 8 + 128 <= 112 * 1024:
            return s
    return 0


def gather_classes(d, n, ks):
    """Gather launches per call: non-empty k classes where the plan takes the gather path, else 0."""
    kmax = max(ks)
    if kmax > 256:
        return 0
    kr = (kmax + 7) // 8 * 8
    if not gather_slices(d, kr) or n < 96 * kr:
        return 0
    caps, lo, used = [16, 32, 64, kr], 0, 0
    for g, cap in enumerate(caps):
        cap = min(cap, kr)
        if g > 0 and cap <= lo:
            continue
        used += any(lo < k <= cap for k in ks)
        lo = cap
        if cap == kr:
            break
    return used


def launches(kind, classes, xm, arith):
    """Kernel launches of one top-k call: split of x per batch, l1/B, scores GEMM, selection, decode (gather classes or
    one GEMM), finalize; backward adds the code-gradient scatter or GEMM and the weight-gradient GEMM; a step adds the
    dictionary-row Adam kernel and, on the dense f16f8 path, the three transposes of the decoder planes."""
    fwd = xm + 4 + (classes or 1)
    if kind == "forward":
        return fwd
    if kind == "grads":
        return fwd + 2
    return fwd + 3 + (3 if arith == "f16f8" and not classes else 0)
