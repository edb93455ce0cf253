"""oracle/eval_bounds.py on small synthetic tensors: the segment reference over split call sequences against a whole-stream
computation, and planted defects of the evaluation pass that the per-feature checks of tests/test_eval_bounds_gpu.py
reject, beside the exact result rounded as the engine rounds it, which they accept."""
import pytest
import torch

from oracle import eval_bounds as EB
from oracle import tile_bounds as T

ARITHS = ("bf16x3", "f16f8")


def _random_calls(g, M, n, sizes, seg, density):
    """Activities of calls of ``sizes`` rows and their phases (rows seen so far mod seg)."""
    calls, seen = [], 0
    for B in sizes:
        calls.append((torch.rand(M, B, n, generator=g) < density, seg, seen % seg))
        seen += B
    return calls


def test_segment_reference_over_calls_equals_the_whole_stream():
    g = torch.Generator().manual_seed(0)
    for trial in range(60):
        M, n = 2, 7
        sizes = torch.randint(1, 90, (int(torch.randint(1, 6, (1,), generator=g)),), generator=g).tolist()
        seg = int(torch.randint(1, 120, (1,), generator=g))
        density = [0.002, 0.02, 0.3][trial % 3]
        calls = _random_calls(g, M, n, sizes, seg, density)
        open0 = torch.zeros(M, n, dtype=torch.long) if seg == 1 else (torch.rand(M, n, generator=g) < 0.5).long()
        phase0 = 0 if seg == 1 else int(torch.randint(0, seg, (1,), generator=g))
        calls = [(a, s, (p + phase0) % seg) for a, s, p in calls]
        got = EB.segment_sequence(calls, open0)
        want = EB.stream_segments(torch.cat([a for a, _, _ in calls], 1), seg, phase0, open0)
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), (trial, sizes, seg, phase0)
        if seg == 1:    # rows: exactly the activity counts
            assert torch.equal(got[0], torch.cat([a for a, _, _ in calls], 1).sum(1))


def test_segment_reference_counts_a_segment_that_ends_at_a_call_end():
    a = torch.zeros(1, 8, 1, dtype=torch.bool)
    a[0, 7, 0] = True
    counts, open_ = EB.segment_call(a, 4, 0, torch.zeros(1, 1, dtype=torch.long))
    assert int(counts) == 1 and int(open_) == 0
    counts, open_ = EB.segment_call(a[:, :6], 4, 0, torch.zeros(1, 1, dtype=torch.long))   # row 5 of segment 1: open
    assert int(counts) == 0 and int(open_) == 0
    counts, open_ = EB.segment_call(a, 5, 2, torch.ones(1, 1, dtype=torch.long))          # carried flag at phase 2
    assert int(counts) == 2 and int(open_) == 0
    counts, open_ = EB.segment_call(a[:, :7], 5, 2, torch.ones(1, 1, dtype=torch.long))   # rows 3..6 of 3..7: open
    assert int(counts) == 1 and int(open_) == 0


# ----------------------------------------------------------------------------------------------------------------------
# planted segment-count defects: the exact comparison rejects each on the call sequence of the GPU test
# ----------------------------------------------------------------------------------------------------------------------
def _defective_call(active, seg, phase, open_, defect):
    """segment_count_kernel's rule, restated segment by segment, with one defect planted: "left_open_at_call_end" takes
    a segment that ends exactly at the call's end for still open (end < B instead of end <= B), "carry_ignored" drops
    the carried flag of the first segment."""
    M, B, n = active.shape
    counts, new = torch.zeros(M, n, dtype=torch.long), open_.clone()
    K = -(-(B + phase) // seg)
    for k in range(K):
        lo, end = max(0, k * seg - phase), (k + 1) * seg - phase
        fired = active[:, lo:min(end, B)].any(1).long()
        if k == 0 and defect != "carry_ignored":
            fired = fired | open_
        if end < B or (end == B and defect != "left_open_at_call_end"):
            counts += fired
            if k == K - 1:
                new = torch.zeros_like(new)
        else:
            new = fired
    return counts, new


@pytest.mark.parametrize("defect,seg", [("left_open_at_call_end", 4001), ("carry_ignored", 37),
                                         ("carry_ignored", 4001)])
def test_planted_segment_defects_are_rejected(defect, seg):
    """The call sizes of the GPU test's sequence. At seg = 37 segments end inside calls and span them, but none ends
    exactly at a call's end; at seg = 4001 the first does, and the second spans the five calls after it."""
    g = torch.Generator().manual_seed(1)
    M, n = 3, 64
    sizes = (4001, 33, 1, 31, 129, 2048)
    calls = _random_calls(g, M, n, sizes, seg, 0.003)
    want = EB.segment_sequence(calls, torch.zeros(M, n, dtype=torch.long))
    total, open_ = torch.zeros(M, n, dtype=torch.long), torch.zeros(M, n, dtype=torch.long)
    for active, s, phase in calls:
        inc, open_ = _defective_call(active, s, phase, open_, defect)
        total += inc
    assert not (torch.equal(total, want[0]) and torch.equal(open_, want[1])), (defect, seg)


# ----------------------------------------------------------------------------------------------------------------------
# moments: the bound accepts the engine's rounding and rejects planted defects
# ----------------------------------------------------------------------------------------------------------------------
def _case(seed=2, B=4001, d=64, n=96, bias=-0.1):
    """A dense SAE code with a partial last row block (4001 = 125 * 32 + 1 rows), its scale and the fp64 sums."""
    g = torch.Generator().manual_seed(seed)
    X = torch.randn(B, d, generator=g, dtype=torch.float64)
    W = torch.nn.functional.normalize(torch.randn(n, d, generator=g, dtype=torch.float64), dim=-1)
    b = bias + 0.05 * torch.randn(n, generator=g, dtype=torch.float64)
    c = (X @ W.T + b).clamp(min=0.0)
    return c, T.code_scale(X, W, b), EB.moment_sums(c)


def _worst(got, want, bound, start=None):
    start = torch.zeros_like(got) if start is None else start
    return float(EB.moment_ratios(got + start, start, want, bound).max())


@pytest.mark.parametrize("arith", ARITHS)
def test_moment_bound_accepts_the_exact_code_rounded_to_fp32_in_32_row_partials(arith):
    c, S, want = _case()
    e = T.BARS[arith]["signed"]["code"][1]
    for tree, K in ((True, EB.K_TREE), (False, EB.K_RUNNING)):
        got = EB.fp32_partial_moments(c, tree=tree)
        assert _worst(got, want, EB.moment_bound(c, S, e, K)) <= 1.0, (arith, tree)
        # random fp64 start values: the accumulator's rounding is part of the bound
        start = 1e3 * torch.randn(want.shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
        assert _worst(got, want, EB.moment_bound(c, S, e, K), start) <= 1.0, (arith, tree)
    # a code error of e S_b on every coefficient with the same sign is the worst the bound allows
    moved = EB.moment_sums(c + e * S * (c > 0))
    assert _worst(moved, want, EB.moment_bound(c, S, e, EB.K_TREE)) <= 1.0


@pytest.mark.parametrize("arith", ARITHS)
def test_moment_bound_rejects_the_last_partial_row_block_dropped(arith):
    c, S, want = _case()
    e = T.BARS[arith]["signed"]["code"][1]
    got = EB.fp32_partial_moments(c[:4000])           # the one-row block 125 never added
    assert (c[4000] > 0).any()
    assert _worst(got, want, EB.moment_bound(c, S, e, EB.K_TREE)) > 1.0


def test_moment_bound_rejects_moments_of_a_one_pass_bf16x3_code():
    """The moments of the code rounded to bf16 (a single-pass bf16x3 code's leading plane). A single f16f8 pass keeps
    an fp16 plane, whose rounding summed over many rows stays under the f16f8 bound (tests/test_eval_bounds_gpu.py
    measures its 1-pass moments at about half of it): no claim is made there."""
    c, S, want = _case()
    e = T.BARS["bf16x3"]["signed"]["code"][1]
    one = c.to(torch.bfloat16).double()
    assert _worst(EB.fp32_partial_moments(one), want, EB.moment_bound(c, S, e, EB.K_TREE)) > 1.0


def test_moment_bound_rejects_a_warp_past_the_batch_adding_rows():
    """Rows beyond the batch in the last row block encoded from zero input rows: relu(bias) added 31 times (what the
    STATS epilogue would add without its row rule)."""
    c, S, want = _case(bias=0.02)
    b = torch.full((c.shape[1],), 0.02, dtype=torch.float64)
    ghost = torch.cat([c, b.clamp(min=0.0)[None].expand(31, -1)])
    assert _worst(EB.moment_sums(ghost), want, EB.moment_bound(c, S, T.BARS["bf16x3"]["signed"]["code"][1],
                                                                EB.K_TREE)) > 1.0


def test_padding_feature_with_a_nonzero_sum_is_rejected():
    start = torch.randn(2, 10, 4, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    pad = torch.arange(10) >= 7
    after = start.clone()
    after[:, ~pad] += 1.0
    assert EB.padding_unchanged(start[1], after[1], pad) == []
    after[1, 8, 2] += 2.0 ** -40
    assert EB.padding_unchanged(start[1], after[1], pad) == [8]
    counts = torch.zeros(10, dtype=torch.int32)
    assert EB.padding_unchanged(counts, counts + (torch.arange(10) == 9).int(), pad) == [9]


def test_a_nan_moment_sum_is_rejected():
    """A partial never written reads as NaN from the 0xFF-filled workspace: one feature's sum NaN (or inf) among
    correct ones must give an infinite ratio per feature and per run, and one that the worst-value record keeps."""
    c, S, want = _case()
    bound = EB.moment_bound(c, S, T.BARS["bf16x3"]["signed"]["code"][1], EB.K_TREE)
    start = torch.randn(want.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    good = start + EB.fp32_partial_moments(c)
    assert float(EB.moment_ratios(good, start, want, bound).max()) <= 1.0
    assert float(EB.moment_run_ratios(good, start, want, bound).max()) <= 1.0
    for bad_value in (float("nan"), float("inf")):
        got = good.clone()
        got[17, 2] = bad_value
        ratio = EB.moment_ratios(got, start, want, bound)
        runs = EB.moment_run_ratios(got, start, want, bound)
        assert not ratio.isnan().any() and not runs.isnan().any()
        assert float(ratio[17, 2]) == float("inf") and float(runs[2, 0]) == float("inf")
        assert float(ratio.max()) == float("inf") and float(runs.max()) == float("inf")
    w = T.Worst()
    w.add_scalar("moments", 0, 0.1)
    w.add_scalar("moments", 1, float("nan"))
    w.add_scalar("moments", 2, 0.2)
    assert w.tile["moments"][0] == float("inf") and w.elem["moments"] == float("inf")
