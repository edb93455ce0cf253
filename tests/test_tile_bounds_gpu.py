"""Every dense training-step output of the engine per (model, 128 x 128 tile) and per element against fp64.

The GEMMs of a step write their outputs in 128 x 128 tiles per model, and a fused epilogue works on one tile at a time.
An error confined to one tile (the ragged last row or column tile, the K tail, one model's slab of a per-model batch,
one operand set of dW = dz^T x + c^T g, the second tile a persistent CTA runs) enters a norm-relative number per model
divided by about sqrt(tiles): the last tile of x_hat at 1-pass accuracy passes the 1e-4 bar of the other parity tests
(test_negative_control_single_pass_tile shows it). Here every output is measured per tile and per element against its
absolute-product scale (oracle/tile_bounds.py), over the whole output of every model:

  code, x_hat           tiles of [B, n] and [B, d]                losses   |got - want| / |want|
  encoder, decoder      tiles of [n, d] (after the row-norm Jacobian where the rows are normalised)
  encoder_bias, center  runs of 128 of [n] and [d]

Signatures: tied, tied with FunctionalTiedSAE's centring, untied, masked tied and untied (dictionary sizes that are not
multiples of 128), learned centre, positive tied; both arithmetics; a batch shared by the models and per-model batches;
fp16-exact inputs (the f16f8 residual-flag skip) and arbitrary fp32 ones. The ragged shape M = 4, d = 400, n = 1040,
B = 4001 gives every GEMM of the step more than 132 tiles (the H100's SM count) and a partial last tile in each output
dimension and in K, and replays the step as a CUDA graph; at B = 8001, above the launch-bound rule, tied and untied
run the step eagerly and, under f16f8, the native E5M2 weight gradient (dw_native) with those partial tiles; config 2
runs at full size with all 16 models, config 5's width tied and untied. Each case is checked at initialisation and again after 3 steps on the engine's own fp32 parameters as read back (which covers the
planes the dictionary-row kernel re-splits). Adam is not compared element by element. Gradients keep the kink rule of
the other parity tests: coefficients with |z| < kink_window are pinned to the engine's side, none outside it may be on
the other side, and their number is bounded.

The activity the oracle is pinned to is the engine's: the dense code read back from its planes can hold an f16f8 code
below ~4e-9 as 0 while the engine's mask has it active (engine_activity recovers those from the mask counts), and a
pre-activation the engine computes as exactly 0 passes the reconstruction gradient without the L1 term, which no call
reads back (regate_exact_zeros recognises the one coefficient that explains a feature's error; at most a couple per
model). Both were found by this file, as single coefficients whose gradient was off by alpha / B or by g w^T.

Bars (tile ratio, element maximum) per arithmetic, dictionary sign and output, set from measurement on an H100 SXM
(80 GB HBM3, 700 W limit): each is twice the worst 3-pass value this file observes at any shape, rounded up. The 1-pass
column is the smallest tile ratio over every tile of the single-pass runs (ragged shape, fp32 inputs; fwd_passes=1 for
code / x_hat, bwd_passes=1 for the gradients). Where it is at least twice the bar, the output is SEPARATED: a tile that
lost its cross terms fails its bar, and test_single_pass_tiles_clear_the_bars holds every such tile to it.

  arith   dict    output        3-pass worst tile   bar       1-pass smallest tile   separated
  bf16x3  signed  code          3.2e-7              6.5e-7    1.1e-4                 yes
                  x_hat         2.9e-8              5.8e-8    5.5e-6                 yes
                  encoder       5.2e-6              1.1e-5    6.8e-6                 no
                  decoder       3.2e-6              6.5e-6    4.2e-5                 yes
                  encoder_bias  2.6e-6              5.3e-6    1.6e-5                 yes
                  center        3.8e-8              7.6e-8    1.4e-6                 yes
          nonneg  code          1.8e-6              3.6e-6    1.1e-4                 yes
                  x_hat         2.7e-6              5.5e-6    7.8e-5                 yes
                  encoder       1.3e-5              2.7e-5    2.5e-5                 no
                  encoder_bias  7.0e-6              1.5e-5    6.2e-5                 yes
  f16f8   signed  code          1.4e-6              2.8e-6    1.3e-5                 yes
                  x_hat         8.0e-8              1.6e-7    7.2e-7                 yes
                  encoder       6.8e-6              1.4e-5    9.1e-7                 no
                  decoder       3.5e-5              7.0e-5    5.8e-6                 no
                  encoder_bias  7.8e-6              1.6e-5    3.2e-6                 no
                  center        5.7e-8              1.2e-7    2.3e-7                 no (4.0x)
          nonneg  code          8.5e-6              1.7e-5    1.5e-5                 no
                  x_hat         8.5e-6              1.7e-5    1.0e-5                 no
                  encoder       2.7e-5              5.4e-5    1.6e-5                 no
                  encoder_bias  1.9e-5              3.9e-5    1.5e-5                 no

Losses (relative error of each term): bf16x3 3.1e-5 signed, 1.1e-5 non-negative; f16f8 8.3e-5, 3.4e-5. Where no gap
exists the 3-pass worst and the 1-pass best tile overlap: the f16f8 gradients (their bwd_passes=1 error relative to
the pre-activation gradient's scale is as small as the 3-pass error of the features an L1 of 1e-2 keeps nearly
inactive), the non-negative dictionary in f16f8 (its one-signed sums accumulate fp32 rounding in the tensor cores as
large as a single pass's operand rounding), and the bf16x3 encoder gradient. For those outputs the bar still bounds
every tile and element at twice the worst value measured, but a tile at 1-pass accuracy is not guaranteed to fail it.
The whole file runs in about 30 s on an H100. The harness it runs is tests/engine_cases.py, shared with the other
step tests.
"""
import pytest
import torch

from engine_cases import (ARITHS, RAGGED, RAGGED_EAGER, VARIANTS, batch, ensemble, make_models, measure, oracle,
                          regate_exact_zeros, relnorm, report, run_case, scales, sign)
from oracle import tile_bounds as T
from oracle.plan_paths import launch_bound

pytestmark = pytest.mark.gpu

REL, GRAD_REL = 1e-4, 2e-4           # the per-model norm-relative bars of the other parity tests
BARS, SEPARATED = T.BARS, T.SEPARATED   # (tile ratio bar, element bar) and the separated outputs: see the docstring


@pytest.mark.parametrize("inputs", ["fp16", "fp32"])
@pytest.mark.parametrize("per_model", [False, True], ids=["shared", "per_model"])
@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("variant", VARIANTS)
def test_ragged_shape_every_tile(variant, arith, per_model, inputs):
    """Every signature at M = 4, d = 400, n = 1040, B = 4001: more than 132 tiles in every GEMM, a partial last tile in
    every output dimension and in K."""
    M, d, n, B = RAGGED
    models, sig = make_models(variant, M, d, n, 0)
    tag = f"ragged {variant} {'per-model' if per_model else 'shared'} {inputs}"
    run_case(tag, variant, models, sig, arith, RAGGED, per_model, inputs == "fp16")


@pytest.mark.parametrize("inputs", ["fp16", "fp32"])
@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("variant", ["tied", "untied"])
def test_ragged_eager_shape_every_tile(variant, arith, inputs):
    """M = 4, d = 400, n = 1040, B = 8001: ragged like the shape above but not launch-bound, so the step runs eagerly
    and, under f16f8, the weight gradient takes the native E5M2 path (dw_native) with a partial tile in n, in d and in
    K = B (Bp = 8016)."""
    M, d, n, B = RAGGED_EAGER
    assert not launch_bound(M, B, n, d)
    models, sig = make_models(variant, M, d, n, 0)
    tag = f"ragged eager {variant} {inputs}"
    print(f"{tag}: step eager, dw_native {'yes' if arith == 'f16f8' else 'no'}")
    run_case(tag, variant, models, sig, arith, RAGGED_EAGER, False, inputs == "fp16", seed=200)


@pytest.mark.parametrize("arith", ARITHS)
def test_config2_all_models_every_tile(arith):
    """BASELINE config 2 at full size (d = 512, n = 4096, B = 8192) with all 16 models across its L1 grid."""
    shape = (16, 512, 4096, 8192)
    models, sig = make_models("tied", shape[0], *shape[1:3], 2)
    run_case("cfg2 tied 16 models", "tied", models, sig, arith, shape, False, True, seed=300)


@pytest.mark.parametrize("variant", ["tied", "untied"])
def test_config5_width_every_tile(variant):
    """BASELINE config 5's width (d = 2048, n = 32768, B = 4096, one model): K = 32768 in decode, K = B in dW."""
    shape = (1, 2048, 32768, 4096)
    models, sig = make_models(variant, *shape[:3], 3)
    run_case(f"cfg5 {variant}", variant, models, sig, "f16f8", shape, False, True, seed=400, n_feats=4096)


def single_pass(variant, arith, seed=500):
    """The ragged shape with fwd_passes=1 (code, x_hat, losses) and with bwd_passes=1 (the gradients), arbitrary fp32
    inputs: what every tile of an output that lost its cross terms measures."""
    M, d, n, B = RAGGED
    models, sig = make_models(variant, M, d, n, 0)
    X = batch(M, B, d, seed, False, False)
    fwd, _ = measure(variant, ensemble(models, sig, arith, fwd_passes=1), X, False)
    bwd, _ = measure(variant, ensemble(models, sig, arith, bwd_passes=1), X, False)
    for name in ("encoder", "decoder", "encoder_bias", "center"):
        for attr in ("tile", "elem", "minimum"):
            table = getattr(bwd, attr)
            if name in table:
                getattr(fwd, attr)[name] = table[name]
    return fwd


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("variant", ["tied", "untied", "learned_center", "positive_tied"])
def test_single_pass_tiles_clear_the_bars(variant, arith):
    """Every tile of a single-pass output measures at least twice its bar, for each output the bar separates."""
    w = single_pass(variant, arith)
    report(f"1-pass {variant}", arith, variant, w)
    bars = BARS[arith][sign(variant)]
    for name in SEPARATED[arith][sign(variant)]:
        if name in w.minimum:
            assert w.minimum[name][0] >= 2 * bars[name][0], (name, w.minimum[name][0], bars[name][0])


def _splice_last_tile(dst, src):
    """dst with its last (ragged) tile replaced by src's."""
    out = dst.clone()
    r0, c0 = (dst.shape[0] - 1) // 128 * 128, (dst.shape[1] - 1) // 128 * 128
    out[r0:, c0:] = src[r0:, c0:]
    return out


@pytest.mark.parametrize("arith", ARITHS)
def test_negative_control_single_pass_tile(arith):
    """The last, ragged tile of the last model's x_hat (from a fwd_passes=1 plan) and of its encoder gradient (from a
    bwd_passes=1 plan) spliced into the 3-pass outputs: the per-model norm-relative bar still accepts each spliced
    tensor, the per-tile check rejects it at that tile. Asserted for the outputs whose bar separates 3-pass from 1-pass
    tiles (x_hat in both arithmetics); the encoder gradient's numbers are printed, its bar does not separate them."""
    M, d, n, B = RAGGED
    models, sig = make_models("tied", M, d, n, 0)
    X = batch(M, B, d, 600, False, False)
    full = ensemble(models, sig, arith)
    grads, (_, aux) = full.grads_batch(X)
    code = aux["c"].dense()
    counts = full.active_counts(B)
    _, _, x_hat = full.forward_batch(X, return_x_hat=True)
    _, _, x_hat1 = ensemble(models, sig, arith, fwd_passes=1).forward_batch(X, return_x_hat=True)
    grads1, _ = ensemble(models, sig, arith, bwd_passes=1).grads_batch(X)
    m = M - 1
    P = {k: v[m].double() for k, v in full.params.items()}
    buf = {k: v[m] for k, v in full.buffers.items()}
    f0 = oracle("tied", P, buf, X.double())
    near = f0["Z"].abs() < T.kink_window(f0["Z"])
    active = torch.where(near, T.engine_activity(code[m], counts[m], near, f0["Z"]), f0["Z"] > 0)
    f = oracle("tied", P, buf, X.double(), active)
    regate_exact_zeros("tied", f, grads["encoder_bias"][m], near & ~active & (code[m] == 0))
    S_x = T.x_hat_scale(f["Xabs"], f["W"], P["encoder_bias"], f["W"])
    S_e = scales("tied", f, P["encoder_bias"])["encoder"]
    last = lambda t: ((t.shape[0] - 1) // 128, (t.shape[1] - 1) // 128)
    results = []
    for name, got, got1, want, S, bar in (("x_hat", x_hat[m], x_hat1[m], f["x_hat"], S_x, REL),
                                          ("encoder", grads["encoder"][m], grads1["encoder"][m],
                                           f["grads"]["encoder"], S_e, GRAD_REL)):
        spliced = _splice_last_tile(got, got1)
        rel, rel3 = relnorm(spliced, want), relnorm(got, want)
        r = T.tile_ratios(spliced, want, S)
        tile_bar = BARS[arith]["signed"][name][0]
        print(f"negative control {arith:6s} {name:8s} spliced tile {last(want)}: norm-relative {rel:.2e} (3-pass "
              f"{rel3:.2e}, bar {bar:.0e}); worst tile {r['worst'][0]:.2e} at {r['worst'][1]}, tile bar {tile_bar:.1e}")
        results.append((name, rel, bar, r["worst"], tile_bar, (0,) + last(want)))
    for name, rel, bar, worst, tile_bar, at in results:
        if name not in SEPARATED[arith]["signed"]:
            continue                       # no gap between 3-pass and 1-pass tiles of this output: no claim
        assert rel <= bar, (name, rel, bar)                                  # the per-model norm misses the tile ...
        assert worst[0] > tile_bar and worst[1] == at, (name, worst, at)    # ... the per-tile check does not
    assert "x_hat" in SEPARATED[arith]["signed"]
