"""oracle/tile_bounds.py on small synthetic tensors: the absolute-product scales against brute-force loops, the tile grid
with its ragged edge tiles, and a perturbation confined to one tile that the per-model norm-relative bar accepts and the
per-tile check rejects."""
import itertools

import torch

from oracle import sae_oracle as O
from oracle import tile_bounds as T


def _loops(A, B):
    """sum_k |A[i, k]| |B[k, j]| by explicit loops."""
    out = torch.zeros(A.shape[0], B.shape[1], dtype=torch.float64)
    for i, j in itertools.product(range(A.shape[0]), range(B.shape[1])):
        out[i, j] = sum(abs(float(A[i, k])) * abs(float(B[k, j])) for k in range(A.shape[1]))
    return out


def test_scales_equal_brute_force_loops():
    g = torch.Generator().manual_seed(0)
    B, d, n = 7, 5, 6
    X, E, D = (torch.randn(r, c, generator=g, dtype=torch.float64) for r, c in ((B, d), (n, d), (n, d)))
    b = torch.randn(n, generator=g, dtype=torch.float64)
    f = O.tied_grads(E, b, X, 1e-2, 0.05)
    W, s, dZ, C, G = f["W"], f["s"], f["dZ"], f["c"], f["G"]

    code = _loops(X, W.T) + b.abs()
    assert torch.allclose(T.code_scale(X, W, b), code, rtol=1e-12, atol=0)
    assert torch.allclose(T.x_hat_scale(X, W, b, D), _loops(code, D), rtol=1e-12, atol=0)

    dw = _loops(dZ.T, X) + _loops(C.T, G)
    assert torch.allclose(T.weight_grad_scale(dZ, X, C, G), dw, rtol=1e-12, atol=0)
    assert torch.allclose(T.weight_grad_scale(dZ, X), _loops(dZ.T, X), rtol=1e-12, atol=0)
    assert torch.allclose(T.weight_grad_scale(None, None, C, G), _loops(C.T, G), rtol=1e-12, atol=0)
    jac = torch.zeros(n, d, dtype=torch.float64)
    for i, j in itertools.product(range(n), range(d)):
        dot = sum(abs(float(W[i, k])) * abs(float(dw[i, k])) for k in range(d))
        jac[i, j] = (abs(float(dw[i, j])) + abs(float(W[i, j])) * dot) / float(s[i])
    assert torch.allclose(T.row_norm_jacobian_scale(W, s, dw), jac, rtol=1e-12, atol=0)
    # it bounds what it scales: the Jacobian of dW, term by term
    assert bool((f["grads"]["encoder"].abs() <= T.row_norm_jacobian_scale(W, s, dw) * (1 + 1e-12)).all())

    # the pre-activation gradient's scale, (|g| |W|^T + alpha / B) on the gate, and it bounds dz
    gate = f["Z"] >= 0
    sdz = torch.zeros(B, n, dtype=torch.float64)
    for r, i in itertools.product(range(B), range(n)):
        if gate[r, i]:
            sdz[r, i] = sum(abs(float(G[r, k])) * abs(float(W[i, k])) for k in range(d)) + 1e-2 / B
    assert torch.allclose(T.pre_activation_grad_scale(G, W, 1e-2 / B, gate), sdz, rtol=1e-12, atol=0)
    assert bool((dZ.abs() <= sdz * (1 + 1e-12)).all())
    # the centred batch's scale, (|x - t| |R|^T) |s|, bounds the centred batch
    t, R, sc = torch.randn(d, generator=g, dtype=torch.float64), torch.randn(d, d, generator=g, dtype=torch.float64), \
        torch.randn(d, generator=g, dtype=torch.float64)
    xc = _loops(X - t, R.T) * sc.abs()
    assert torch.allclose(T.centered_input_scale(X, t, R, sc), xc, rtol=1e-12, atol=0)
    assert bool((O.center(X, t, R, sc).abs() <= xc * (1 + 1e-12)).all())

    decay = O._bias_decay_grad(b, 0.05)
    bias = torch.tensor([sum(abs(float(dZ[r, i])) for r in range(B)) + abs(float(decay[i])) for i in range(n)],
                        dtype=torch.float64)
    assert torch.allclose(T.bias_grad_scale(dZ, decay), bias, rtol=1e-12, atol=0)
    db = f["grads"]["encoder_bias"]
    centre = torch.tensor([sum(abs(float(G[r, j])) for r in range(B)) + sum(abs(float(db[i])) * abs(float(W[i, j]))
                                                                         for i in range(n)) for j in range(d)],
                          dtype=torch.float64)
    assert torch.allclose(T.center_grad_scale(G, db, W), centre, rtol=1e-12, atol=0)


def test_tile_grid_counts_ragged_edge_tiles():
    g = torch.Generator().manual_seed(1)
    M, R, C = 2, 130, 257                         # 2 x 3 tiles of 128 per model, the last row and column partial
    want = torch.randn(M, R, C, generator=g, dtype=torch.float64)
    scale = want.abs() + 1.0
    got = want.clone()
    got[1, 129, 256] += 0.5                       # the last element, in the 2 x 1 corner tile
    r = T.tile_ratios(got, want, scale)
    assert tuple(r["ratio"].shape) == (M, 2, 3)
    assert r["worst"][1] == (1, 1, 2)
    assert int((r["ratio"] > 0).sum()) == 1
    # the corner tile's ratio is over its own two elements, not over a whole padded tile
    corner = 0.5 / float(scale[1, 128:, 256].norm())
    assert abs(r["worst"][0] - corner) <= 1e-12 * corner, (r["worst"], corner)
    assert abs(r["elem"] - 0.5 / float(scale[1, 129, 256])) <= 1e-12 * r["elem"]
    # one model [R, C] and a vector [L] (runs of 128)
    assert tuple(T.tile_ratios(got[0], want[0], scale[0])["ratio"].shape) == (1, 2, 3)
    v = T.tile_ratios(got[1, 129], want[1, 129], scale[1, 129])
    assert tuple(v["ratio"].shape) == (1, 1, 3) and v["worst"][1] == (0, 0, 2)
    # a NaN is an infinite error
    got[0, 0, 0] = float("nan")
    assert T.tile_ratios(got, want, scale)["worst"] == (float("inf"), (0, 0, 0))


def test_one_tile_at_single_pass_accuracy_passes_the_norm_bar_and_fails_the_tile_bar():
    """An x_hat-like output at config 2's size per model ([8192, 512]: 256 tiles, K = 4096) computed from fp32 operands,
    except its last tile, computed from fp16-rounded operands (a tile that lost its cross terms). The per-model
    norm-relative error stays under the 1e-4 bar the dense-variant tests apply; the per-tile ratio of that tile is more
    than ten times that of every other tile."""
    g = torch.Generator().manual_seed(2)
    B, d, n = 8192, 512, 4096
    X = torch.randn(B, d, generator=g, dtype=torch.float64)
    W, _ = O.unit_rows(torch.randn(n, d, generator=g, dtype=torch.float64))
    b = 0.02 * torch.randn(n, generator=g, dtype=torch.float64)
    C = (X @ W.T + b).clamp(min=0)
    want = C @ W
    S = T.x_hat_scale(X, W, b, W)
    got = (C.float() @ W.float()).double()
    got[-128:, -128:] = C[-128:].half().double() @ W[:, -128:].half().double()
    rel = float((got - want).norm() / want.norm())
    r = T.tile_ratios(got, want, S)
    assert rel <= 1e-4, rel
    assert r["worst"][1] == (0, 63, 3)
    assert r["worst"][0] > 10 * float(r["ratio"][0].flatten()[:-1].max()), r["worst"]


# ----------------------------------------------------------------------------------------------------------------------
# top-k: planted defects against the bars of tests/test_topk_tile_bounds_gpu.py (oracle/tile_bounds.py: TOPK_BARS)
# ----------------------------------------------------------------------------------------------------------------------
def _topk(D, X, k):
    """fp64 TopKEncoder outputs and their scales on the oracle's own support."""
    f = O.topk_grads(D, X, k)
    support = f["sel"] & (f["Z"] > 0)
    return f, support, T.topk_scales(X, f["W"], f["s"], f["c"], f["G"], support)


def _topk_case(k=12, seed=3):
    """Ragged tiles in every output: B = 160, d = 200, n = 320; a previous batch X0 for the stale-state defects."""
    g = torch.Generator().manual_seed(seed)
    B, d, n = 160, 200, 320
    D = torch.randn(n, d, generator=g, dtype=torch.float64)
    X, X0 = (torch.randn(B, d, generator=g, dtype=torch.float64) for _ in range(2))
    return D, X, X0, k


def _dict_grad(f, X, dZ):
    return O._row_norm_jacobian(f["W"], f["s"], dZ.T @ X + f["c"].T @ f["G"])


def _verdict(name, got, want, S):
    """Per arithmetic: does the check fail (tile ratio or element maximum above its bar)?"""
    r = T.tile_ratios(got, want, S)
    return {a: r["worst"][0] > T.TOPK_BARS[a][name][0] or r["elem"] > T.TOPK_BARS[a][name][1] for a in T.TOPK_BARS}


def _plane_residual(v, arith):
    """What the residual planes hold of v: v minus its leading bf16 (bf16x3) or fp16 (f16f8) plane."""
    return v - v.to(torch.bfloat16 if arith == "bf16x3" else torch.float16).double()


def test_topk_bars_accept_the_exact_result_rounded_to_fp32():
    D, X, _, k = _topk_case()
    f, _, S = _topk(D, X, k)
    for name, want in (("code", f["c"]), ("x_hat", f["x_hat"]), ("dict", f["grads"]["dict"])):
        assert not any(_verdict(name, want.float(), want, S[name]).values()), name


def test_topk_bars_reject_a_stale_code_gradient_residual():
    """Code-gradient residual-plane entries left from the previous call, at columns that call selected and this one does
    not: stray lo x terms in the weight gradient. The entries a selection failed to clear are rejected under both
    arithmetics; so is a single one under bf16x3 (a bf16 residual, up to 2^-9 of its entry). A single f16f8 residual
    (up to 2^-12 of its entry) measures 3e-6 of its element's scale here, under the element bar of 2.1e-4."""
    D, X, X0, k = _topk_case()
    f, support, S = _topk(D, X, k)
    f0, support0, _ = _topk(D, X0, k)
    stale = support0 & ~support
    for arith in T.TOPK_BARS:
        resid = _plane_residual(f0["dZ"], arith) * stale.to(X.dtype)
        got = _dict_grad(f, X, f["dZ"] + resid)
        assert _verdict("dict", got, f["grads"]["dict"], S["dict"])[arith], arith
    r, j = (int(i) for i in torch.nonzero(stale)[0])
    one = f["dZ"].clone()
    one[r, j] += _plane_residual(f0["dZ"], "bf16x3")[r, j]
    assert _verdict("dict", _dict_grad(f, X, one), f["grads"]["dict"], S["dict"])["bf16x3"]


def test_topk_bars_reject_x_hat_from_the_dictionary_before_the_last_step():
    """x_hat gathered from the normalised dictionary as it was before the last Adam step (a stale fp32 copy): the
    scores see the new rows, the decode the old ones (an Adam step moves every entry by about lr = 1e-3)."""
    D, X, _, k = _topk_case()
    f, _, S = _topk(D, X, k)
    old, _ = O.unit_rows(D + 1e-3 * torch.sign(f["grads"]["dict"]), floor=None)
    assert all(_verdict("x_hat", f["c"] @ old, f["x_hat"], S["x_hat"]).values())


def test_topk_bars_reject_a_gather_sum_missing_one_entry():
    """x_hat of one row without one selected entry's contribution to one slice (the first half) of its columns."""
    D, X, _, k = _topk_case()
    f, support, S = _topk(D, X, k)
    r, j = (int(i) for i in torch.nonzero(support)[len(torch.nonzero(support)) // 2])
    got = f["x_hat"].clone()
    h = X.shape[1] // 2
    got[r, :h] -= f["c"][r, j] * f["W"][j, :h]
    assert all(_verdict("x_hat", got, f["x_hat"], S["x_hat"]).values())


def test_topk_bars_reject_a_gradient_through_a_nonpositive_selected_score():
    """k = 200 of n = 320 keeps non-positive scores in every row; one of them passes g w^T to the weight gradient,
    which the ReLU stops."""
    D, X, _, k = _topk_case(k=200)
    f, support, S = _topk(D, X, k)
    cand = f["sel"] & (f["Z"] < 0)
    dz = (f["G"] @ f["W"].T)[cand]
    at = torch.nonzero(cand)[int(dz.abs().argsort()[len(dz) // 2])]          # the median |g w^T| of them
    dZ = f["dZ"].clone()
    dZ[at[0], at[1]] = (f["G"][at[0]] @ f["W"][at[1]])
    assert all(_verdict("dict", _dict_grad(f, X, dZ), f["grads"]["dict"], S["dict"]).values())
