"""oracle/row_pass_bounds.py on the CPU: the absolute-product scales bound what they scale, the slicing restatement keeps
its invariants, and the per-tile check with its bars (measured in tests/test_row_pass_tiles_gpu.py) rejects each
planted defect of a row pass (one tile off by 4 bars, the last slice's padding rows added as 0 - shift, the last partial slice dropped,
g' counted over padding rows, an output stored instead of accumulated) while it accepts the exact result rounded to
fp32."""
import pytest
import torch

from engine_cases import ARITHS
from oracle import row_pass_bounds as RB
from oracle import tile_bounds as T

KINDS = ("moments", "ica", "project", "grams")
D, N, B = 200, 136, 700            # 2 x 2 tiles, the last ragged; 3 slices of 256 rows, 68 of them padding
ALPHA = RB.ALPHA


def data(kind, positive, seed=0):
    """x [B, D] fp32, shift [D] and the pass's matrix. positive: rows above the shift and non-negative matrices, so that
    no product cancels and every output equals its scale (up to tanh and the norms' square)."""
    g = torch.Generator().manual_seed(seed)
    if positive:
        x = 1.0 + torch.rand(B, D, generator=g)
        shift = 0.5 + 0.1 * torch.rand(D, generator=g)
        mat = {"ica": 0.05 * torch.rand(N, D, generator=g) / D ** 0.5, "project": torch.rand(N, D, generator=g),
               "grams": torch.rand(B, N, generator=g)}.get(kind)
    else:
        mu = 3.0 * torch.randn(D, generator=g)
        x = torch.randn(B, D, generator=g) + mu
        shift = mu + 0.1 * torch.randn(D, generator=g)
        mat = {"ica": torch.randn(N, D, generator=g) / D ** 0.5, "project": torch.randn(N, D, generator=g) / D ** 0.5,
               "grams": torch.rand(B, N, generator=g) * (torch.rand(B, N, generator=g) < 0.3)}.get(kind)
    return x, shift, mat


def worst(kind, name, got, want, scale):
    return T.tile_ratios(got, want, scale)["worst"][0]


def bar(kind, name, arith):
    return RB.BARS[kind][name][arith][0]


def test_slicing_restatement():
    assert RB.mom_slices(D, B) == (3, 256)
    for d in (64, 200, 512, 2048, 8192):
        for b in (1, 63, 64, 65, 700, 3841, 4096, 64000, 65536, 1 << 21):
            S, R = RB.mom_slices(d, b)
            assert R % 64 == 0 and R <= 2048 and (S - 1) * R < b <= S * R, (d, b, S, R)


@pytest.mark.parametrize("kind", KINDS)
def test_scales_bound_their_outputs(kind):
    x, shift, mat = data(kind, False)
    for name, (want, scale) in RB.reference(kind, x, shift, mat, ALPHA).items():
        assert bool((want.abs() <= scale * (1 + 1e-12)).all()), name
        assert bool((scale > 0).all()), name


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("kind", KINDS)
def test_bars_accept_the_exact_result_rounded_to_fp32(kind, arith):
    for positive in (False, True):
        x, shift, mat = data(kind, positive)
        for name, (want, scale) in RB.reference(kind, x, shift, mat, ALPHA).items():
            r = worst(kind, name, want.float().double(), want, scale)
            assert r <= bar(kind, name, arith), (name, r, bar(kind, name, arith))
    want, scale = RB.nmf_residual(RB.shifted(x, shift, clamp=True), torch.rand(B, 8), torch.rand(8, D))
    assert abs(float(torch.tensor(want).float()) - want) / scale <= RB.BARS["residual"]


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("kind", KINDS)
def test_one_tile_off_by_four_bars_fails(kind, arith):
    x, shift, mat = data(kind, True)
    for name, (want, scale) in RB.reference(kind, x, shift, mat, ALPHA).items():
        b = bar(kind, name, arith)
        got = want.clone()
        if got.dim() == 1:                                 # the first run of 128 (the norms' second half is 0 here)
            got[:128] *= 1 + 4 * b
        else:                                              # the last, ragged tile
            got[-(got.shape[0] % 128 or 128):, -(got.shape[1] % 128 or 128):] *= 1 + 4 * b
        r = T.tile_ratios(got, want, scale)
        assert r["worst"][0] > b, (name, r["worst"], b)


def padded(x, mat, kind):
    """x with the last slice's padding rows as zero rows (so v = 0 - shift), as a pass that did not zero them would see
    them; W gets zero rows too (the Grams pass zeroes its padding rows of W separately)."""
    S, R = RB.mom_slices(D, B)
    x = torch.cat((x, torch.zeros(S * R - B, D)))
    if kind == "grams":
        mat = torch.cat((mat, torch.zeros(S * R - B, N)))
    return x, mat


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("kind", ("moments", "ica"))
def test_padding_rows_as_minus_shift_fail(kind, arith):
    x, shift, mat = data(kind, False)
    ref = RB.reference(kind, x, shift, mat, ALPHA)
    bad = RB.reference(kind, padded(x, mat, kind)[0], shift, mat, ALPHA)
    name = "gram" if kind == "moments" else "gx"
    assert worst(kind, name, bad[name][0], *ref[name]) > bar(kind, name, arith)


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("kind", ("moments", "ica", "grams"))
def test_last_partial_slice_dropped_fails(kind, arith):
    x, shift, mat = data(kind, False)
    S, R = RB.mom_slices(D, B)
    keep = (S - 1) * R
    ref = RB.reference(kind, x, shift, mat, ALPHA)
    bad = RB.reference(kind, x[:keep], shift, mat[:keep] if kind == "grams" else mat, ALPHA)
    for name in ref:
        assert worst(kind, name, bad[name][0], *ref[name]) > bar(kind, name, arith), name


@pytest.mark.parametrize("arith", ARITHS)
def test_g_prime_over_padding_rows_fails(arith):
    """g' = alpha (1 - 0) on the rows of the last 32-row block past B (u = 0 on a zero padding row)."""
    x, shift, mat = data("ica", False)
    want, scale = RB.reference("ica", x, shift, mat, ALPHA)["g_sum"]
    got = want + ALPHA * (-(-B // 32) * 32 - B)
    assert worst("ica", "g_sum", got, want, scale) > bar("ica", "g_sum", arith)


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("kind", KINDS)
def test_stored_instead_of_accumulated_fails(kind, arith):
    """out - initial, where the pass wrote its result over the initial values instead of adding to them."""
    x, shift, mat = data(kind, False)
    for name, (want, scale) in RB.reference(kind, x, shift, mat, ALPHA).items():
        if name not in RB.ACCUMULATED:
            continue
        init = (float(scale.abs().mean()) + 1.0) * (torch.rand(want.shape, generator=torch.Generator().manual_seed(3),
                                                               dtype=torch.float64) + 0.5)
        assert worst(kind, name, want - init, want, scale) > bar(kind, name, arith), name
