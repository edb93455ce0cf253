"""fp64 references and error bounds of the fused evaluation pass (libsce sce_forward_stats) per feature.

*** TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT PATH. *** (as oracle/tile_bounds.py)

sce_forward_stats adds, per model m, feature j and power p = 1..4, sum_b c[b, j]^p to moment_sums[m, j, p - 1] (fp64),
and the segments of `seg` rows that end in the call and in which feature j fired to seg_counts[m, j], carrying the
flag of a segment still open in seg_open[m, j]. A defect there (a 32-row partial never written, a warp past the batch
adding rows that do not exist, a carry flag dropped or never cleared) moves single features by a whole row's or
segment's worth, which a bar relative to the largest value of the vector does not see. So every feature is held to a
bound of its own.

Moment bound. The engine sums the exact fp32 code c' = relu(z') of its fp32 pre-activation z' (top-k: relu of the fp32
score where the selection kept it). ReLU is 1-Lipschitz, so |c' - c| <= |z' - z| <= e S_b with c the fp64 code, S_b the
code's absolute-product scale (tile_bounds.code_scale; top-k: |x| |W|^T on the support) and e the element bar of the
code in that arithmetic (tile_bounds.BARS / TOPK_BARS). By the mean value theorem |c'^p - c^p| <= p (c + e S_b)^(p-1) e S_b.
The powers and sums are then rounded in fp32, u = 2^-24 (first order, over the absolute values, which are the values):
  c2 = c * c                     1 rounding
  c3 = c2 * c, c4 = c2 * c2      2 and 3 roundings
  32-row partial                 SAE variants: the 5-level pairwise tree of warp_column_sum, 5 roundings on each term;
                                 top-k (topk_moment_kernel): a running sum over the 32 rows, up to 31 roundings
  fp64 sum of the partials       about 2^-53 per partial, and one rounding of the accumulator (2^-53 |result|)
so the arithmetic adds at most K sum_b c_b^p with K = 8 u (SAE) or 34 u (top-k), and the caller's fp64 start value one
rounding of 2^-53 (|start| + |result|). Per feature j and power p:

  bound_p[j] = e sum_b p (c_b + e S_b)^(p-1) S_b  +  K sum_b c_b^p  +  2^-52 (|start| + |got|)

The check is |(got - start) - want| <= bound per element (ratio <= 1), and the same ratio over runs of 128 features
(tile_bounds.tile_ratios on a vector). No new bar is measured: the bound follows from the code's element bar, which
tests/test_tile_bounds_gpu.py and tests/test_topk_tile_bounds_gpu.py hold every code element to. For the SAE variants
it needs no support pinned; top-k pins the fp64 code to the engine's support (topk_pinned_code), as the top-k tile test
does.

Segment counts are exact, on the engine's own activity: segment_counts restates the header's definition call by call.
"""
from __future__ import annotations

from typing import Iterable, List, Tuple

import torch

from . import tile_bounds as T

Tensor = torch.Tensor
U = 2.0 ** -24
K_TREE = 8 * U          # SAE variants: c4's 3 roundings and the 5 levels of warp_column_sum
K_RUNNING = 34 * U      # top-k: c4's 3 roundings and a running sum over 32 rows
ROWS = 32               # rows per fp32 partial


def moment_sums(c: Tensor) -> Tensor:
    """[..., B, n] code -> [..., n, 4]: sum over the rows of c, c^2, c^3, c^4 (in c's dtype)."""
    return torch.stack([c.pow(p).sum(-2) for p in (1, 2, 3, 4)], dim=-1)


def moment_bound(c: Tensor, S: Tensor, e: float, K: float, weight: Tensor = None) -> Tensor:
    """[B, n] fp64 code and its scale -> [n, 4]: e sum_b p (c_b + e S_b)^(p-1) S_b + K sum_b c_b^p (module docstring).
    ``weight`` ([B], optional): each row's weight in a weighted sum (a streaming average's). The caller adds the
    accumulator's rounding (accumulator_slack)."""
    c, S = c.double().abs(), S.double().abs()
    hi = c + e * S
    w = weight.double()[:, None] if weight is not None else 1.0
    out = [(w * (e * p * hi.pow(p - 1) * S + K * c.pow(p))).sum(0) for p in (1, 2, 3, 4)]
    return torch.stack(out, dim=-1)


def accumulator_slack(start: Tensor, got: Tensor) -> Tensor:
    """One fp64 rounding of the accumulated sum start + result: 2^-52 (|start| + |got|), from the finite values only (a
    non-finite sum is an error of its own, not a reason for slack)."""
    fin = lambda t: torch.nan_to_num(t.double().abs(), nan=0.0, posinf=0.0, neginf=0.0)
    return 2.0 ** -52 * (fin(start) + fin(got))


def moment_ratios(got: Tensor, start: Tensor, want: Tensor, bound: Tensor) -> Tensor:
    """|(got - start) - want| / bound per feature and power ([n, 4], fp64): inf wherever the accumulator after the call
    is not finite (a NaN partial, say) or the error is not 0 where the bound is. got and start are the accumulator after
    and before the call; the result is never NaN."""
    err = ((got.double() - start.double()) - want.double()).abs()
    bad = ~torch.isfinite(got.double()) | torch.isnan(err)
    err = torch.where(bad, torch.full_like(err, float("inf")), err)
    b = bound.double() + accumulator_slack(start, got)
    return torch.where(err == 0, torch.zeros_like(err), err / b)


def moment_run_ratios(got: Tensor, start: Tensor, want: Tensor, bound: Tensor) -> Tensor:
    """The same error over runs of 128 features per power, ||err||_run / ||bound + slack||_run ([4, runs], fp64), inf
    for a run holding a non-finite accumulator."""
    err = ((got.double() - start.double()) - want.double()).abs()
    err = torch.where(~torch.isfinite(got.double()) | torch.isnan(err), torch.full_like(err, float("inf")), err)
    scale = bound.double() + accumulator_slack(start, got)
    return T.tile_ratios(err.T, torch.zeros_like(err.T), scale.T, tile=(1, T.TILE))["ratio"][0]


def fp32_partial_moments(c: Tensor, tree: bool = True) -> Tensor:
    """What the engine computes from a code c ([B, n], taken as fp32): the powers in fp32, summed over 32-row blocks
    in fp32 (tree: pairwise in 5 levels as warp_column_sum; else a running sum in row order as topk_moment_kernel),
    the partials added in fp64 in row-block order. [n, 4] fp64."""
    c = c.float()
    B, n = c.shape
    rb = -(-B // ROWS)
    c = torch.nn.functional.pad(c, (0, 0, 0, rb * ROWS - B)).reshape(rb, ROWS, n)
    c2 = c * c
    powers = (c, c2, c2 * c, c2 * c2)
    out = []
    for v in powers:
        if tree:
            while v.shape[1] > 1:
                v = v[:, 0::2] + v[:, 1::2]
            part = v[:, 0]
        else:
            part = v[:, 0]
            for r in range(1, ROWS):
                part = part + v[:, r]
        acc = torch.zeros(n, dtype=torch.float64)
        for i in range(rb):
            acc = acc + part[i].double()
        out.append(acc)
    return torch.stack(out, dim=-1)


# ----------------------------------------------------------------------------------------------------------------------
# segment counts (sce_forward_stats' seg_counts / seg_open, sce_forward_fragments' n_active)
# ----------------------------------------------------------------------------------------------------------------------
def segment_call(active: Tensor, seg: int, phase: int, open_: Tensor) -> Tuple[Tensor, Tensor]:
    """One call as include/sce.h defines it. ``active`` bool [M, B, n]: the activity of the call's rows; ``phase``:
    rows of the first segment that earlier calls saw; ``open_`` int [M, n]: 1 where the feature fired in the segment
    still open before the call. Returns (increments of seg_counts: the segments that END in this call in which the
    feature fired, the open flags after the call). seg = 1 counts rows and leaves ``open_`` as it was."""
    M, B, n = active.shape
    if seg == 1:
        return active.sum(1).long(), open_.clone()
    assert 0 <= phase < seg
    counts = torch.zeros(M, n, dtype=torch.long, device=active.device)
    new_open = open_.clone().long()
    k = 0
    while True:
        lo, end = max(0, k * seg - phase), (k + 1) * seg - phase
        fired = active[:, lo:min(end, B)].any(1).long()
        if k == 0:
            fired = fired | open_.long()
        if end <= B:
            counts += fired
            new_open = torch.zeros_like(new_open)
            if end == B:
                break
        else:
            new_open = fired
            break
        k += 1
    return counts, new_open


def segment_sequence(calls: Iterable[Tuple[Tensor, int, int]], open_: Tensor) -> Tuple[Tensor, Tensor]:
    """segment_call over a sequence of calls (activity, seg, phase): (summed increments, open flags at the end)."""
    total = torch.zeros_like(open_, dtype=torch.long)
    for active, seg, phase in calls:
        inc, open_ = segment_call(active, seg, phase, open_)
        total += inc
    return total, open_


def stream_segments(active: Tensor, seg: int, phase: int, open_: Tensor) -> Tuple[Tensor, Tensor]:
    """The same quantities computed on the whole stream at once ([M, N, n]): the rows, preceded by ``phase`` rows seen
    earlier (whose activity is ``open_``), cut into segments of ``seg``; the completed ones counted, the last one's flag
    open if it is incomplete. An independent restatement for tests/test_eval_bounds_cpu.py."""
    M, N, n = active.shape
    total = phase + N
    n_seg = -(-total // seg)
    rows = torch.zeros(M, n_seg * seg, n, dtype=torch.bool, device=active.device)
    rows[:, phase:phase + N] = active
    if phase:
        rows[:, 0] |= open_.bool()
    fired = rows.reshape(M, n_seg, seg, n).any(2)
    done = total // seg
    if seg == 1:
        return fired[:, phase:].sum(1).long(), open_.clone()
    counts = fired[:, :done].sum(1).long()
    left = fired[:, done].long() if done < n_seg else torch.zeros(M, n, dtype=torch.long, device=active.device)
    return counts, left


# ----------------------------------------------------------------------------------------------------------------------
# top-k: the fp64 code on the engine's support
# ----------------------------------------------------------------------------------------------------------------------
def topk_pinned_code(X: Tensor, W: Tensor, code: Tensor, counts: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
    """Scores Z = X W^T (W the unit rows), the engine's support (the code read back plus the f16f8 codes too small to
    read back, tile_bounds.engine_activity) and the fp64 code relu(Z) on it: (c, S_code, support). S_code is the code's
    scale |X| |W|^T on the support (0 elsewhere, where both sides are 0)."""
    Z = X @ W.T
    support = T.engine_activity(code, counts, Z.abs() < T.kink_window(Z), Z)
    on = support.to(X.dtype)
    return Z.clamp(min=0.0) * on, (X.abs() @ W.abs().T) * on, support


def padding_unchanged(before: Tensor, after: Tensor, pad: Tensor) -> List[int]:
    """Indices of padding features (``pad`` bool [n]) whose entries (any trailing dims) are not bitwise unchanged."""
    bits = {torch.float64: torch.int64, torch.float32: torch.int32}
    if before.dtype in bits:
        before, after = before.view(bits[before.dtype]), after.view(bits[after.dtype])
    diff = before != after
    while diff.dim() > 1:
        diff = diff.any(-1)
    return torch.nonzero(diff & pad.to(diff.device)).flatten().tolist()
