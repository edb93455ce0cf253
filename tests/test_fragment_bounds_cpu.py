"""The call-by-call fragment reference (oracle/interp_oracle.merge_call) and the per-element value bounds
(interp_oracle.value_bounds) on small tensors: any cut of a stream into calls at fragment boundaries, at any frag0
offsets, gives what select() gives on the whole stream, ties and all-zero features included; the bounds accept the
exact code rounded to fp32; and the checks of tests/test_fragment_bounds_gpu.py reject each planted defect of
fragment_max_kernel / fragment_merge_kernel, restated here row by row beside the correct rule, which they accept."""
import math

import pytest
import torch

from oracle import interp_oracle as IO
from oracle import tile_bounds as T

GARBAGE_KEY = (1 << 63) - 1     # what an empty random entry holds: above every priority if it were compared
SENTINEL = -7.25                # the rows of an empty entry


def _code(g, G, L, n, ties=True, zero=(3,)):
    """[G L, n] fp64 non-negative sparse code: fragment 2 a copy of 0, fragment G-1 a copy of 1 (exact ties), some
    features zero everywhere."""
    c = (torch.rand(G * L, n, generator=g, dtype=torch.float64) < 0.2) * torch.rand(G * L, n, generator=g,
                                                                                     dtype=torch.float64)
    if ties:
        c[2 * L:3 * L] = c[0:L]
        c[(G - 1) * L:] = c[L:2 * L]
    c[:, list(zero)] = 0.0
    return c


def _run(code, L, cuts, frag0s, n_top, n_random, seed, rows=True):
    """merge_call over the calls ``cuts`` (fragment ranges of ``code``) from empty lists."""
    n = code.shape[1]
    top = IO.empty_lists(n, n_top, L if rows else None)
    rnd = IO.empty_lists(n, n_random, L if rows else None, key_dtype=torch.int64)
    for (a, b), f0 in zip(cuts, frag0s):
        fmax, active = IO.fragment_tables(code[a * L:b * L], L)
        top, rnd = IO.merge_call(top, rnd, fmax, active, f0, seed, code[a * L:b * L], L)
    return top, rnd


def _random_cuts(g, G):
    """Fragment ranges covering 0 .. G in random pieces (single fragments among them)."""
    edges = sorted(set([0, G] + torch.randint(1, G, (int(torch.randint(1, 6, (1,), generator=g)),),
                                              generator=g).tolist()))
    return list(zip(edges[:-1], edges[1:]))


@pytest.mark.parametrize("n_top,n_random", [(8, 8), (64, 64), (1, 0), (0, 64), (20, 20)])
def test_calls_give_select_on_the_whole_stream(n_top, n_random):
    """select() encodes a tied dictionary over the whole stream; its code has exact ties (fragments 2 and 0, G - 1 and
    1 copy each other's rows) and a dead feature (bias -100)."""
    g = torch.Generator().manual_seed(0)
    d, n, L, G = 16, 24, 32, 30
    m = {"kind": "tied", "encoder": torch.randn(n, d, generator=g, dtype=torch.float64),
         "encoder_bias": 0.3 * torch.randn(n, generator=g, dtype=torch.float64) - 0.5}
    m["encoder_bias"][5] = -100.0
    x = torch.randn(G * L, d, generator=g, dtype=torch.float64)
    x[2 * L:3 * L], x[(G - 1) * L:] = x[:L], x[L:2 * L]
    for seed in (0, (1 << 63) + 12345):
        o = IO.select(m, x, L=L, n_top=n_top, n_random=n_random, seed=seed)
        assert bool((o["fmax"][:, 5] == 0).all()) and bool((o["fmax"][2] == o["fmax"][0]).all())
        for trial in range(4):
            cuts = _random_cuts(g, G)
            top, rnd = _run(o["code"], L, cuts, [a for a, _ in cuts], n_top, n_random, seed)
            assert torch.equal(top[1], o["top_fragments"]), (trial, cuts)
            want_v = o["fmax"].T.gather(1, o["top_fragments"].clamp(min=0))
            assert torch.equal(top[0], torch.where(o["top_fragments"] >= 0, want_v, torch.zeros_like(want_v)))
            assert torch.equal(top[2], IO.fragment_values(o["code"], o["top_fragments"], L))
            assert torch.equal(rnd[1], o["random_fragments"]), (trial, cuts)
            assert torch.equal(rnd[2], IO.fragment_values(o["code"], o["random_fragments"], L))
        if n_top:      # the dead feature: fragments 0 .. n_top - 1, all at 0
            want = torch.arange(n_top)
            assert torch.equal(top[1][5], torch.where(want < G, want, torch.full_like(want, -1)))


@pytest.mark.parametrize("n_top,n_random", [(8, 8), (64, 64)])
def test_calls_at_frag0_gaps_give_select_on_the_stream_with_the_gaps(n_top, n_random):
    """Calls at random frag0 gaps equal select_top / select_random over the whole numbering, the gap fragments holding
    a maximum of -1 (below every fragment) and no activity; select_top's gap picks are the reference's empty entries."""
    g = torch.Generator().manual_seed(1)
    L, G, n = 32, 26, 40
    code = _code(g, G, L, n)
    for trial in range(4):
        cuts = _random_cuts(g, G)
        frag0s, f = [], 0
        for a, b in cuts:
            f += int(torch.randint(0, 5, (1,), generator=g))
            frag0s.append(f)
            f += b - a
        fmax, active = IO.fragment_tables(code, L)
        F = frag0s[-1] + cuts[-1][1] - cuts[-1][0]
        full_max = torch.full((F, n), -1.0, dtype=torch.float64)
        full_act = torch.zeros(F, n, dtype=torch.bool)
        for (a, b), f0 in zip(cuts, frag0s):
            full_max[f0:f0 + b - a], full_act[f0:f0 + b - a] = fmax[a:b], active[a:b]
        top, rnd = _run(code, L, cuts, frag0s, n_top, n_random, 7)
        want_t = IO.select_top(full_max, n_top)
        want_t = torch.where(full_max.T.gather(1, want_t.clamp(min=0)) < 0, torch.full_like(want_t, -1), want_t)
        assert torch.equal(top[1], want_t), (trial, cuts, frag0s)
        assert torch.equal(rnd[1], IO.select_random(full_act, n_random, 7)), (trial, cuts, frag0s)


def test_frag0_beyond_2_32_against_a_plain_sort():
    """Calls at frag0 >= 2^32 and a seed >= 2^63, against Python's sort of (key, fragment) tuples per feature."""
    g = torch.Generator().manual_seed(2)
    L, G, n, k = 32, 12, 6, 5
    code = _code(g, G, L, n)
    cuts, frag0s = [(0, 3), (3, 4), (4, 12)], [0, 1 << 32, (1 << 32) + 7]
    seed = (1 << 64) - 3
    top, rnd = _run(code, L, cuts, frag0s, k, k, seed)
    fmax, active = IO.fragment_tables(code, L)
    ids = torch.cat([f0 + torch.arange(b - a) for (a, b), f0 in zip(cuts, frag0s)])
    p = IO.priority(seed, torch.arange(n), ids)
    for j in range(n):
        best = sorted((-float(fmax[i, j]), int(ids[i])) for i in range(G))[:k]
        assert top[1][j].tolist() == [f for _, f in best] and top[0][j].tolist() == [-v for v, _ in best]
        draw = sorted((-int(p[i, j]), int(ids[i])) for i in range(G) if active[i, j])[:k]
        assert rnd[1][j].tolist() == [f for _, f in draw] + [-1] * (k - len(draw)), j
    assert bool((rnd[1][3] == -1).all())       # the all-zero feature draws nothing


def test_list_order_never_compares_the_key_of_an_empty_entry():
    key = torch.tensor([[float("nan"), 1.0, float("inf"), 1.0, 2.0]])
    frag = torch.tensor([[-1, 9, -1, 4, 6]])
    assert IO.list_order(key, frag)[0, :3].tolist() == [4, 3, 1]


# ----------------------------------------------------------------------------------------------------------------------
# bounds
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arith", ["bf16x3", "f16f8"])
def test_bounds_accept_the_exact_code_rounded_to_fp32(arith):
    g = torch.Generator().manual_seed(3)
    L, G, n, d = 32, 10, 50, 24
    X = torch.randn(G * L, d, generator=g, dtype=torch.float64)
    W = torch.nn.functional.normalize(torch.randn(n, d, generator=g, dtype=torch.float64), dim=-1)
    b = 0.1 * torch.randn(n, generator=g, dtype=torch.float64) - 0.2
    c = (X @ W.T + b).clamp(min=0.0)
    S = T.code_scale(X, W, b)
    e = T.BARS[arith]["signed"]["code"][1]
    cb, fb = IO.value_bounds(S, e, L)
    c32 = c.float().double()
    assert bool(((c32 - c).abs() <= cb).all())
    assert bool(((IO.fragment_tables(c32, L)[0] - IO.fragment_tables(c, L)[0]).abs() <= fb).all())
    # a code error of e S on every element is the most the bounds allow; a maximum moved past its bound is rejected
    moved = c + e * S
    assert bool(((IO.fragment_tables(moved, L)[0] - IO.fragment_tables(c, L)[0]).abs() <= fb + 1e-12).all())      # (fp64 rounding of c + e S)
    assert not bool(((IO.fragment_tables(c + 2 * e * S, L)[0] - IO.fragment_tables(c, L)[0]).abs() <= fb).all())


# ----------------------------------------------------------------------------------------------------------------------
# planted defects: the engine's two kernels restated row by row, each defect switchable
# ----------------------------------------------------------------------------------------------------------------------
DEFECTS = ["tie_to_higher", "empty_key_compared", "lists_reset", "frag0_ignored", "rows_from_previous",
           "last_row_dropped", "partial_chunk_unwritten", "inactive_admitted"]


def _tables(code, L, defect):
    """fragment_max_kernel: maxima and activity (fp64 stand-in for fp32); the unwritten chunk keeps the 0xFF
    workspace: a NaN maximum and a non-zero flag."""
    G, n = code.shape[0] // L, code.shape[1]
    c = code.reshape(G, L, n)
    if defect == "last_row_dropped":
        c = c[:, :L - 1]
    fmax, active = c.amax(1), (c > 0).any(1)
    if defect == "partial_chunk_unwritten":
        last = (n - 1) // 32 * 32
        fmax[:, last:], active[:, last:] = float("nan"), True
    return fmax, active


def _above(k, f, k2, f2, defect):
    if defect == "empty_key_compared":
        return k > k2 or (k == k2 and f < f2)
    if f2 < 0:
        return True
    tie = f > f2 if defect == "tie_to_higher" else f < f2
    return f >= 0 and (k > k2 or (k == k2 and tie))


def _lowest(key, frag, defect):
    w = 0
    for i in range(1, len(key)):
        if _above(key[w], frag[w], key[i], frag[i], defect):
            w = i
    return w


def _fresh(n, n_top, n_random, L):
    """Lists as a caller may hand them over: every entry empty, with a NaN value or a garbage key and sentinel rows."""
    mk = lambda cap, key: [[[key] * cap, [-1] * cap, [[SENTINEL] * L for _ in range(cap)]] for _ in range(n)]
    return {"top": mk(n_top, float("nan")), "rnd": mk(n_random, GARBAGE_KEY)}


def _kernel_call(lists, code, L, frag0, seed, defect):
    """fragment_merge_kernel per feature, with ``defect`` planted."""
    fmax, active = _tables(code, L, defect)
    G, n = fmax.shape
    if defect == "lists_reset":
        lists.update(_fresh(n, len(lists["top"][0][0]), len(lists["rnd"][0][0]), L))
    base = 0 if defect == "frag0_ignored" else frag0
    p = IO.priority(seed, torch.arange(n), base + torch.arange(G))
    for which in ("top", "rnd"):
        for j in range(n):
            key, frag, rows = lists[which][j]
            if not key:
                continue
            low = _lowest(key, frag, defect)
            for gi in range(G):
                if which == "rnd" and not (active[gi, j] or defect == "inactive_admitted"):
                    continue
                k = float(fmax[gi, j]) if which == "top" else int(p[gi, j])
                if _above(k, base + gi, key[low], frag[low], defect):
                    src = max(gi - 1, 0) if defect == "rows_from_previous" else gi
                    key[low], frag[low], rows[low] = k, base + gi, code[src * L:(src + 1) * L, j].tolist()
                    low = _lowest(key, frag, defect)


def _judge(lists, ref, code_stream, frag_rows):
    """The GPU test's exact checks on one list kind: sorted keys and fragments equal to the reference's, every entry's
    rows equal to the code of its fragment (rows of empty entries keep their sentinel), and (top) each value the
    maximum of its rows. ``frag_rows``: fragment id -> first stream row."""
    key = torch.tensor([e[0] for e in lists], dtype=ref[0].dtype)
    frag = torch.tensor([e[1] for e in lists], dtype=torch.int64)
    rows = torch.tensor([e[2] for e in lists], dtype=torch.float64)
    o = IO.list_order(key, frag)
    frag_s, key_s, rows_s = frag.gather(1, o), key.gather(1, o), rows.gather(1, o[..., None].expand_as(rows))
    if not torch.equal(frag_s, ref[1]):
        return False
    full = frag_s >= 0
    if not torch.equal(key_s[full], ref[0][full]):
        return False
    if not bool((rows_s[~full] == SENTINEL).all()):
        return False
    for j, i in full.nonzero().tolist():
        r0 = frag_rows[int(frag_s[j, i])]
        if not torch.equal(rows_s[j, i], code_stream[r0:r0 + rows.shape[-1], j]):
            return False
    return True


def _sequence(n_top, n_random, defect):
    g = torch.Generator().manual_seed(4)
    L, G, n = 32, 24, 40           # two 32-column chunks, the second partial
    code = _code(g, G, L, n)
    cuts, frag0s = [(0, 1), (1, 9), (9, 11), (11, 20), (20, 24)], [0, 1, 15, 1 << 32, (1 << 32) + 9]
    seed = (1 << 63) + 5
    ref_top, ref_rnd = _run(code, L, cuts, frag0s, n_top, n_random, seed)
    lists = _fresh(n, n_top, n_random, L)
    frag_rows = {}
    for (a, b), f0 in zip(cuts, frag0s):
        _kernel_call(lists, code[a * L:b * L], L, f0, seed, defect)
        frag_rows.update({f0 + i: (a + i) * L for i in range(b - a)})
    ok_top = n_top == 0 or _judge(lists["top"], ref_top, code, frag_rows)
    ok_rnd = n_random == 0 or _judge(lists["rnd"], ref_rnd, code, frag_rows)
    return ok_top and ok_rnd, lists, code, frag_rows


@pytest.mark.parametrize("n_top,n_random", [(8, 8), (64, 64)])
def test_the_restated_kernels_pass(n_top, n_random):
    ok, lists, _, _ = _sequence(n_top, n_random, None)
    assert ok
    assert any(f < 0 for e in lists["top"] for f in e[1]) == (n_top > 24)


@pytest.mark.parametrize("defect", DEFECTS)
def test_planted_defect_is_rejected(defect):
    assert not _sequence(8, 8, defect)[0], defect


def test_last_row_dropped_fails_the_fp64_value_bound():
    """Where values are not the read-back planes (top-k) the fp64 layer alone must reject a maximum that misses its
    fragment's last row (top_ratios: each value against its fragment's fp64 maximum, and a fragment outside the fp64
    top set against the n_top-th maximum), here with an element bar of 2.5e-5 on a unit scale."""
    for defect, rejected in ((None, False), ("last_row_dropped", True)):
        _, lists, code, frag_rows = _sequence(8, 8, defect)
        _, fb = IO.value_bounds(torch.ones_like(code), 2.5e-5, 32)
        fmax = IO.fragment_tables(code, 32)[0]
        vals = torch.tensor([e[0] for e in lists["top"]], dtype=torch.float64)
        local = torch.tensor([[frag_rows[f] // 32 for f in e[1]] for e in lists["top"]])
        r = IO.top_ratios(vals, local, fmax, fb)
        worst = max(float(r["value"].max()), float(r["set"].max()))
        assert math.isfinite(worst) and (worst > 1.0) == rejected, (defect, worst)
