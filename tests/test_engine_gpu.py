"""Parity of the CUDA engine (through the C ABI, via sparse_coding_b200.FunctionalEnsemble) against
 (a) the golden vectors recorded from the reference's own loss functions (tests/golden, oracle/make_golden.py) and
 (b) the oracle (oracle/sae_oracle.py) on seeded inputs, single steps and multi-step trajectories.

Tolerances (BASELINE.json north_star: "within 1e-4 rel on reconstructed activations and loss"):
  x̂, code : ||a - b||_2 / ||b||_2 <= 1e-4          losses : |a - b| / |b| <= 1e-4
  gradients: norm-relative <= 2e-4 (3-pass backward)   trajectories: see test docstrings

Both operand arithmetics (include/sce.h sce_arith) are held to the same bars: "bf16x3" and "f16f8" (the default
where d and n are multiples of 16). The loss is not differentiable where a pre-activation is exactly at the ReLU
kink; a pre-activation within the engine's rounding of zero (|z| < kink_window) may land on either side, so
gradient checks pin the activity pattern of those (measure-zero) coefficients to the engine's side.
"""
import math
import os
import subprocess

import pytest
import torch

from engine_cases import clone_models, relnorm
from oracle import sae_oracle as O
from oracle.tile_bounds import kink_window

pytestmark = pytest.mark.gpu

REL = 1e-4
ARITHS = ["bf16x3", "f16f8"]


def tied_grads_engine_kinks(p, b, X, code, mask=None):
    """Oracle gradients of one tied model on batch X (fp64, centring applied here) with the activity pattern of the
    near-kink coefficients taken from the engine's code."""
    pd = {k: v.double() for k, v in p.items()}
    Xd = X.double()
    if "center_rot" in b:
        Xd = O.center(Xd, b["center_trans"].double(), b["center_rot"].double(), b["center_scale"].double())
    bd = float(b["bias_decay"]) if "bias_decay" in b else 0.0
    f0 = O.tied_forward(pd["encoder"], pd["encoder_bias"], Xd, float(b["l1_alpha"]), bd, mask)
    active = torch.where(f0["Z"].abs() < kink_window(f0["Z"]), code.cpu() > 0, f0["Z"] > 0)
    return O.tied_grads(pd["encoder"], pd["encoder_bias"], Xd, float(b["l1_alpha"]), bd, mask, active=active), f0


def _sigs():
    import sparse_coding_b200 as S
    return {"tied": S.FunctionalTiedSAE, "untied": S.FunctionalSAE, "masked_tied": S.FunctionalMaskedTiedSAE,
            "masked_untied": S.FunctionalMaskedSAE, "topk": S.TopKEncoder}


def _models(fx):
    M = next(iter(fx["params"].values())).shape[0]
    return [({k: v[i].float().clone() for k, v in fx["params"].items()},
             {k: (v[i].float().clone() if v.dtype.is_floating_point else v[i].clone()) for k, v in fx["buffers"].items()})
            for i in range(M)]


def _ensemble(fx, **kw):
    import sparse_coding_b200 as S
    return S.FunctionalEnsemble(_models(fx), _sigs()[fx["kind"]], S.adam, {"lr": 1e-3}, device="cuda", **kw)


GOLDEN = ["tied_small", "tied_bias", "tied_f64", "tied_centered", "untied_small", "masked_tied", "masked_untied",
          "topk_small"]


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("name", GOLDEN)
def test_golden_forward_and_grads(golden, name, arith):
    """Engine vs the reference's recorded loss_data / code / gradients on identical params and batch."""
    fx = golden(name)
    ens = _ensemble(fx, arith=arith)
    X = fx["batch"].float().cuda()
    grads, (loss, aux) = ens.grads_batch(X)
    for k, ref in fx["loss_data"].items():
        got = loss[k].cpu().double()
        assert torch.allclose(got, ref.double(), rtol=REL, atol=1e-9), (name, k, got, ref)
    c = aux["c"].dense()
    assert relnorm(c, fx["c"]) <= REL
    # sparsity pattern: identical wherever the reference activation is not within rounding of zero
    ref_c = fx["c"].float()
    big = ref_c.abs() > 1e-4 * ref_c.abs().max()
    assert torch.equal((c.cpu() != 0)[big], (ref_c != 0)[big])
    nnz_ref = fx["c"].count_nonzero(dim=-1).float().mean(dim=-1)
    assert torch.allclose(aux["c"].count_nonzero(dim=-1).float().mean(dim=-1).cpu(), nnz_ref, rtol=2e-2, atol=0.51)
    assert ens.resolved_arith() == arith
    for k, ref in fx["grads"].items():
        err = relnorm(grads[k], ref)
        if err > 2e-4 and fx["kind"] == "tied":
            # a recorded pre-activation sits within the engine's rounding of the kink (tied_centered has one at
            # |z| = 7.7e-6): compare against the oracle (itself pinned to these fixtures, tests/test_oracle.py) with
            # that coefficient on the engine's side
            near = 0
            for i, (p, b) in enumerate(_models(fx)):
                f, f0 = tied_grads_engine_kinks(p, b, fx["batch"], c[i])
                near += int((f0["Z"].abs() < kink_window(f0["Z"])).sum())
                assert relnorm(grads[k][i], f["grads"][k]) <= 2e-4, (name, k, i, relnorm(grads[k][i], f["grads"][k]))
            assert near > 0, (name, k, err)   # the only excuse for missing the recorded gradient
            continue
        assert err <= 2e-4, (name, k, err)


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("name", ["tied_small", "tied_centered", "untied_small", "masked_tied", "topk_small"])
def test_golden_reconstruction(golden, name, arith):
    """x̂ (centred space) against the oracle evaluated on the golden inputs."""
    fx = golden(name)
    ens = _ensemble(fx, arith=arith)
    X = fx["batch"].float().cuda()
    _, _, x_hat = ens.forward_batch(X, return_x_hat=True)
    for i, (p, b) in enumerate(_models(fx)):
        Xd = fx["batch"].double()
        pd = {k: v.double() for k, v in p.items()}
        if fx["kind"] == "tied":
            Xc = O.center(Xd, b["center_trans"].double(), b["center_rot"].double(), b["center_scale"].double())
            f = O.tied_forward(pd["encoder"], pd["encoder_bias"], Xc, float(b["l1_alpha"]))
        elif fx["kind"] == "untied":
            f = O.untied_forward(pd["encoder"], pd["encoder_bias"], pd["decoder"], Xd, float(b["l1_alpha"]))
        elif fx["kind"] == "masked_tied":
            f = O.tied_forward(pd["encoder"], pd["encoder_bias"], Xd, float(b["l1_alpha"]), 0.0, b["coef_mask"])
        else:
            f = O.topk_forward(pd["dict"], Xd, int(b["sparsity"]))
        assert relnorm(x_hat[i], f["x_hat"]) <= REL, (name, i, relnorm(x_hat[i], f["x_hat"]))


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("per_model", [False, True])
def test_device_side_centring(arith, per_model):
    """FunctionalTiedSAE.center (sae_ensemble.py:126-128) on the device — (x - trans) planes, rotation GEMM, scale — at a
    realistic width, for a batch shared by the models and for per-model batches (expand_dims=False): losses, centred
    reconstruction and gradients against the fp64 oracle on the fp64-centred batch, then three steps against the fp32
    reference step."""
    import sparse_coding_b200 as S
    M, d, n, B = 3, 512, 1024, 300
    gen = torch.Generator().manual_seed(11)
    torch.manual_seed(5)
    models = []
    for i in range(M):
        q, _ = torch.linalg.qr(torch.randn(d, d, generator=gen))
        p, b = S.FunctionalTiedSAE.init(d, n, 10 ** (-3 + 0.5 * i), translation=0.3 * torch.randn(d, generator=gen),
                                        rotation=q.contiguous(), scaling=0.5 + torch.rand(d, generator=gen))
        p["encoder_bias"] = 0.05 * torch.randn(n, generator=gen)
        models.append((p, b))
    ens = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda", arith=arith)
    X = torch.randn(M, B, d, generator=gen) if per_model else torch.randn(B, d, generator=gen)
    kw = dict(expand_dims=not per_model)
    grads, (loss, aux) = ens.grads_batch(X.cuda(), **kw)
    code = aux["c"].dense().cpu()
    _, _, x_hat = ens.forward_batch(X.cuda(), return_x_hat=True, **kw)
    for i, (p, b) in enumerate(models):
        Xi = X[i] if per_model else X
        f, f0 = tied_grads_engine_kinks(p, b, Xi, code[i])
        assert relnorm(x_hat[i], f0["x_hat"]) <= REL, (i, relnorm(x_hat[i], f0["x_hat"]))
        assert abs(float(loss["loss"][i]) - float(f0["loss"])) <= REL * float(f0["loss"])
        for k in ("encoder", "encoder_bias"):
            assert relnorm(grads[k][i], f["grads"][k]) <= 2e-4, (i, k, relnorm(grads[k][i], f["grads"][k]))
    ref = O.RefPortEnsemble(clone_models(models), O.SIG_LOSSES["tied"], lr=1e-3)
    for _ in range(3):
        le, _ = ens.step_batch(X.cuda(), **kw)
        lr_, _ = ref.step_batch(X, **kw)
    assert torch.allclose(le["loss"].cpu(), lr_["loss"], rtol=1e-3)
    assert relnorm(ens.params["encoder"], ref.params["encoder"]) <= 2e-3


@pytest.mark.parametrize("arith", ARITHS)
def test_cfg1_golden(golden, arith):
    """BASELINE config 1 (d=128, n=256, B=1024, L1=1e-3): losses, per-row nnz and gradients of the reference."""
    fx = golden("cfg1")
    ens = _ensemble(fx, arith=arith)
    grads, (loss, aux) = ens.grads_batch(fx["batch"].cuda())
    for k, ref in fx["loss_data"].items():
        assert torch.allclose(loss[k].cpu(), ref, rtol=REL, atol=0), (k, loss[k], ref)
    c = aux["c"].dense()[0].cpu()
    assert relnorm(c.double().sum(-1), fx["c_sum"][0]) <= REL
    assert (c.count_nonzero(dim=-1) - fx["c_nnz"][0]).abs().max() <= 1   # a score within rounding of 0 may flip
    p, b = _models(fx)[0]
    f, f0 = tied_grads_engine_kinks(p, b, fx["batch"], aux["c"].dense()[0])
    flipped = int(((c > 0) != (f0["c"] > 0)).sum())
    for k, ref in fx["grads"].items():
        if flipped == 0:
            assert relnorm(grads[k], ref) <= 2e-4, (k, relnorm(grads[k], ref))
        else:   # a score within rounding of 0 flipped: the recorded gradient is on the other side of that kink
            assert relnorm(grads[k][0], f["grads"][k]) <= 2e-4, (k, flipped, relnorm(grads[k][0], f["grads"][k]))


def _random_tied(M, d, n, seed, l1=(1e-4, 1e-2), bias=0.02):
    import sparse_coding_b200 as S
    torch.manual_seed(seed)
    models = []
    for a in torch.logspace(math.log10(l1[0]), math.log10(l1[1]), M).tolist():
        p, b = S.FunctionalTiedSAE.init(d, n, a)
        p["encoder_bias"] = bias * torch.randn(n)
        models.append((p, b))
    return models


@pytest.mark.parametrize("B", [1, 37, 128, 200, 300])
def test_ragged_batches_and_last_short_batch(B):
    """drop_last=False gives a short final batch (SURVEY.md Q7): any B <= batch_max must be exact, including after
    a larger batch left stale rows in the workspace."""
    import sparse_coding_b200 as S
    models = _random_tied(2, 64, 192, 0)
    ens = S.FunctionalEnsemble([({k: v.clone() for k, v in p.items()}, b) for p, b in models], S.FunctionalTiedSAE,
                               S.adam, {"lr": 1e-3}, device="cuda")
    gen = torch.Generator().manual_seed(B)
    big = torch.randn(300, 64, generator=gen)
    ens.forward_batch(big.cuda())                     # fill the workspace with 300 rows first
    X = torch.randn(B, 64, generator=gen)
    grads, (loss, aux) = ens.grads_batch(X.cuda())
    code = aux["c"].dense().cpu()
    for i, (p, b) in enumerate(models):
        # pre-activations within rounding of zero: take the engine's side of the kink (see tied_grads docstring)
        f, _ = tied_grads_engine_kinks(p, b, X, code[i])
        assert abs(float(loss["loss"][i]) - float(f["loss"])) <= REL * abs(float(f["loss"]))
        assert relnorm(grads["encoder"][i], f["grads"]["encoder"]) <= 2e-4
        assert relnorm(grads["encoder_bias"][i], f["grads"]["encoder_bias"]) <= 2e-4
        assert relnorm(aux["c"].dense()[i], f["c"]) <= REL


def test_exact_zero_rows_clamp_gradient():
    """Q4: all-zero input rows with zero bias give z == 0 exactly; clamp(min=0) passes the gradient there."""
    import sparse_coding_b200 as S
    torch.manual_seed(0)
    p, b = S.FunctionalTiedSAE.init(32, 64, 1e-2)
    X = torch.randn(40, 32)
    X[5] = 0.0
    X[17] = 0.0
    ens = S.FunctionalEnsemble([({k: v.clone() for k, v in p.items()}, b)], S.FunctionalTiedSAE, S.adam, {"lr": 1e-3},
                               device="cuda")
    grads, (loss, aux) = ens.grads_batch(X.cuda())
    f = O.tied_grads(p["encoder"].double(), p["encoder_bias"].double(), X.double(), 1e-2)
    assert relnorm(grads["encoder"][0], f["grads"]["encoder"]) <= 2e-4
    assert relnorm(grads["encoder_bias"][0], f["grads"]["encoder_bias"]) <= 2e-4
    assert int(aux["c"].dense()[0, 5].count_nonzero()) == 0


def test_input_range_monitor():
    """sce_input_absmax: the running maximum of |x| an f16f8 plan has been fed (train_loop warns outside [1e-3, 3e4])."""
    import sparse_coding_b200 as S
    torch.manual_seed(0)
    models = [S.FunctionalTiedSAE.init(32, 64, 1e-3)]
    ens = S.FunctionalEnsemble(models, S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda", arith="f16f8")
    assert ens.input_absmax() == 0.0
    X = torch.randn(40, 32)
    ens.step_batch(X.cuda())
    assert ens.input_absmax() == float(X.abs().max())
    Y = 0.5 * torch.randn(24, 32)
    Y[3, 7] = -123.5
    ens.step_batch(Y.cuda())
    assert ens.input_absmax() == 123.5
    ens.step_batch(X.cuda())
    assert ens.input_absmax() == 123.5
    ref = S.FunctionalEnsemble(models, S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda", arith="bf16x3")
    ref.step_batch(X.cuda())
    assert ref.input_absmax() == 0.0


@pytest.mark.parametrize("kind", ["tied", "untied"])
def test_fp16_exact_batches_skip_the_residual_term(kind):
    """Activation chunks are fp16 on disk (activation_dataset.py:404-412): such a batch has an all-zero residual
    plane, the batch-split kernel leaves the plan's flag at 0 and the encode / weight-gradient GEMMs skip the cross
    term (and the loads) that multiply it. The flag is per step: exact and inexact batches may alternate, and every
    step must match the oracle on ITS batch — a stale flag would drop a needed term (1e-3-level error) or keep a dead one."""
    import sparse_coding_b200 as S
    torch.manual_seed(3)
    d, n, B, M = 64, 256, 320, 2
    sig = S.FunctionalTiedSAE if kind == "tied" else S.FunctionalSAE
    models = []
    for a in (1e-3, 1e-2):
        p, b = sig.init(d, n, a) if kind == "tied" else sig.init(d, n, a, bias_decay=0.01)
        p["encoder_bias"] = 0.02 * torch.randn(n)
        models.append((p, b))
    ens = S.FunctionalEnsemble([({k: v.clone() for k, v in p.items()}, {k: v.clone() for k, v in b.items()})
                                for p, b in models], sig, S.adam, {"lr": 1e-3}, device="cuda", arith="f16f8")
    gen = torch.Generator().manual_seed(4)
    for step, exact in enumerate([True, False, True, True, False]):
        X = torch.randn(B, d, generator=gen)
        if exact:
            X = X.half().float()
        grads, (loss, aux) = ens.grads_batch(X.cuda())
        code = aux["c"].dense().cpu()
        for i, (p, b) in enumerate(models):
            pd = {k: v.double() for k, v in p.items()}
            if kind == "tied":
                f, _ = tied_grads_engine_kinks(p, b, X, code[i])
            else:
                f = O.untied_grads(pd["encoder"], pd["encoder_bias"], pd["decoder"], X.double(), float(b["l1_alpha"]),
                                   float(b["bias_decay"]))
            assert abs(float(loss["loss"][i]) - float(f["loss"])) <= REL * abs(float(f["loss"])), (step, exact, i)
            assert relnorm(code[i], f["c"]) <= REL, (step, exact, i)
            if kind == "tied":
                assert relnorm(grads["encoder"][i], f["grads"]["encoder"]) <= 2e-4, (step, exact, i)
                assert relnorm(grads["encoder_bias"][i], f["grads"]["encoder_bias"]) <= 2e-4, (step, exact, i)


@pytest.mark.parametrize("arith", ARITHS)
@pytest.mark.parametrize("mode", ["frozen_t1", "standard"])
@pytest.mark.parametrize("kind", ["tied", "untied"])
def test_training_trajectory_matches_oracle(kind, mode, arith):
    """30 optimiser steps, engine vs the restated reference step (RefPortEnsemble) from identical initial state on
    identical batches. Adam's update is sign-like where |g| is tiny, so parameters are compared in norm and the
    per-step losses to 1e-3. The Adam moments integrate 30 gradients whose near-kink coefficients cannot be pinned
    along a trajectory: with the activity pattern pinned the f16f8 gradient error is 1.2e-5 (bf16x3: 3e-6), the
    rest is coefficients with |z| <~ 2e-5 rms(z) landing on the other side of the kink — about four times as many
    as with bf16x3, hence the wider bound on the moments."""
    import sparse_coding_b200 as S
    torch.manual_seed(1)
    d, n, B, M = 64, 256, 256, 3
    sig = S.FunctionalTiedSAE if kind == "tied" else S.FunctionalSAE
    models = []
    for a in (1e-4, 1e-3, 1e-2):
        p, b = sig.init(d, n, a) if kind == "tied" else sig.init(d, n, a, bias_decay=0.01)
        models.append((p, b))
    ens = S.FunctionalEnsemble(clone_models(models), sig, S.adam, {"lr": 1e-3}, device="cuda", adam_count_mode=mode,
                               arith=arith)
    ref = O.RefPortEnsemble(clone_models(models), O.SIG_LOSSES[kind], lr=1e-3, count_mode=mode)
    gen = torch.Generator().manual_seed(2)
    feats = torch.randn(512, d, generator=gen)
    feats /= feats.norm(dim=-1, keepdim=True)
    for step in range(30):
        codes = (torch.rand(B, 512, generator=gen) < 0.02).float() * torch.rand(B, 512, generator=gen)
        X = codes @ feats + 0.01 * torch.randn(B, d, generator=gen)
        loss, aux = ens.step_batch(X.cuda())
        rloss, raux = ref.step_batch(X)
        for k in rloss:
            assert torch.allclose(loss[k].cpu(), rloss[k], rtol=1e-3, atol=1e-7), (step, k, loss[k], rloss[k])
    for k in ref.params:
        assert relnorm(ens.params[k], ref.params[k]) <= 2e-3, (k, relnorm(ens.params[k], ref.params[k]))
    tol = 1e-3 if arith == "bf16x3" else 3e-3
    assert relnorm(ens.optim_states["mu"]["encoder"], ref.mu["encoder"]) <= tol
    assert relnorm(ens.optim_states["nu"]["encoder"], ref.nu["encoder"]) <= tol


def test_topk_trajectory_matches_oracle():
    import sparse_coding_b200 as S
    torch.manual_seed(3)
    d, n, B = 64, 256, 128
    models = [S.TopKEncoder.init(d, n, k) for k in (4, 8, 16)]
    ens = S.FunctionalEnsemble(clone_models(models), S.TopKEncoder, S.adam, {"lr": 1e-3}, device="cuda", no_stacking=True)
    ref = O.RefPortEnsemble(clone_models(models), O.SIG_LOSSES["topk"], lr=1e-3, no_stacking=True)
    gen = torch.Generator().manual_seed(4)
    for step in range(10):
        X = torch.randn(B, d, generator=gen)
        loss, aux = ens.step_batch(X.cuda())
        rloss, raux = ref.step_batch(X)
        assert torch.allclose(loss["loss"].cpu(), rloss["loss"], rtol=1e-3), (step, loss["loss"], rloss["loss"])
    assert relnorm(ens.params["dict"], ref.params["dict"]) <= 2e-3


def test_config2_shape_properties():
    """BASELINE config 2 at full size (M=16, d=512, n=4096, B=8192): x̂ on ALL rows and the three loss terms against
    the oracle evaluated in fp64 on the GPU (three models across the L1 grid), the fused nnz counter against the dense
    code, loss == l_rec + l_l1, and 3 steps reduce every model's loss. (Full backward at this size:
    tests/test_scale_parity_gpu.py.)"""
    import sparse_coding_b200 as S
    M, d, n, B = 16, 512, 4096, 8192
    torch.manual_seed(0)
    models = [S.FunctionalTiedSAE.init(d, n, float(a)) for a in torch.logspace(-4, -2, M)]
    ens = S.FunctionalEnsemble(models, S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda")
    gen = torch.Generator().manual_seed(1)
    X = torch.randn(B, d, generator=gen).cuda()
    loss0, aux0, x_hat = ens.forward_batch(X, return_x_hat=True)
    for m in (0, 7, 15):
        f = O.tied_forward(ens.params["encoder"][m].double(), ens.params["encoder_bias"][m].double(), X.double(),
                           float(ens.buffers["l1_alpha"][m]))
        assert relnorm(x_hat[m], f["x_hat"]) <= REL
        for k in ("loss", "l_reconstruction", "l_l1"):
            assert abs(float(loss0[k][m]) - float(f[k])) <= REL * abs(float(f[k])), (m, k, float(loss0[k][m]), float(f[k]))
        del f
    c = aux0["c"].dense()
    assert torch.allclose(c.count_nonzero(dim=-1).float().mean(dim=-1), aux0["c"].count_nonzero(dim=-1).float().mean(dim=-1),
                          rtol=1e-6)
    assert torch.allclose(loss0["loss"], loss0["l_reconstruction"] + loss0["l_l1"], rtol=1e-6)
    del c, x_hat
    first = None
    for _ in range(3):
        loss, _ = ens.step_batch(X)
        first = loss["loss"].clone() if first is None else first
    assert bool((loss["loss"] < first).all())
    assert all(torch.isfinite(v).all() for v in ens.params.values())


@pytest.mark.parametrize("shape", [
    # (kind, M, d, n, B)  — the non-headline BASELINE configs at their real widths, reduced batch
    ("topk", 3, 768, 3072, 512),      # config 3: GPT-2-small residual, TopK k in {16, 32, 64}
    ("topk", 2, 768, 12288, 256),     # config 3: largest dictionary
    ("topk", 3, 128, 1040, 200),      # 32.5 chunks of 32 columns: one full warp of chunk maxima, a half chunk at the end
    ("topk", 1, 256, 32768, 128),     # rows too long for the candidate list in shared memory (keys-only select)
    ("tied", 1, 2048, 32768, 256),    # config 5: Pythia-1.4b MLP-out, dict_ratio 16
    ("untied", 2, 768, 3072, 384),    # untied at GPT-2 width
    ("tied", 1, 4096, 8192, 256),     # Pythia-6.9b residual width (row kernels with 8 float4 per thread)
    ("untied", 1, 5120, 1024, 128),   # Pythia-12b width: not a power of two, 16 float4 per thread
])
def test_other_config_shapes(shape):
    """Forward quantities (x̂, loss) on a row slice and one optimiser step at the widths of BASELINE configs 3/5."""
    import sparse_coding_b200 as S
    kind, M, d, n, B = shape
    torch.manual_seed(0)
    if kind == "topk":
        models = [S.TopKEncoder.init(d, n, k) for k in (16, 32, 64)[:M]]
        sig = S.TopKEncoder
    elif kind == "tied":
        models = [S.FunctionalTiedSAE.init(d, n, 1e-3) for _ in range(M)]
        sig = S.FunctionalTiedSAE
    else:
        models = [S.FunctionalSAE.init(d, n, a) for a in (1e-3, 1e-2)[:M]]
        sig = S.FunctionalSAE
    ens = S.FunctionalEnsemble(models, sig, S.adam, {"lr": 1e-3}, device="cuda", no_stacking=(kind == "topk"))
    X = torch.randn(B, d, generator=torch.Generator().manual_seed(1)).cuda()
    loss, aux, x_hat = ens.forward_batch(X, return_x_hat=True)
    rows = torch.arange(0, B, 7, device="cuda")
    code = aux["c"].dense() if kind == "topk" else None
    for m in range(M):
        p = {k: v[m].double() for k, v in ens.params.items()}
        if kind == "topk":
            # Near-ties at the k-th score may legitimately resolve differently in fp32-split and fp64 arithmetic
            # (Q8: torch.topk leaves ties unspecified), so: (i) the engine's support must be a valid top-k of the
            # fp64 scores up to rounding, (ii) x̂ / loss are compared on that support.
            k = int(ens.buffers["sparsity"][m])
            Wn, _ = O.unit_rows(p["dict"], floor=None)
            S = X.double() @ Wn.T
            support = code[m] > 0
            assert int(support.sum(-1).max()) <= k and int(support.sum(-1).min()) >= k - 1
            lowest_kept = torch.where(support, S, torch.full_like(S, float("inf"))).min(-1).values
            highest_dropped = torch.where(support, torch.full_like(S, -float("inf")), S).max(-1).values
            assert bool((lowest_kept >= highest_dropped - 1e-4).all())
            xh = (S.clamp(min=0) * support) @ Wn
            f = {"x_hat": xh[rows]}
            full = {"loss": (X.double() - xh).pow(2).mean()}
        elif kind == "tied":
            f = O.tied_forward(p["encoder"], p["encoder_bias"], X[rows].double(), float(ens.buffers["l1_alpha"][m]))
            full = O.tied_forward(p["encoder"], p["encoder_bias"], X.double(), float(ens.buffers["l1_alpha"][m]))
        else:
            f = O.untied_forward(p["encoder"], p["encoder_bias"], p["decoder"], X[rows].double(),
                                 float(ens.buffers["l1_alpha"][m]))
            full = O.untied_forward(p["encoder"], p["encoder_bias"], p["decoder"], X.double(),
                                    float(ens.buffers["l1_alpha"][m]))
        assert relnorm(x_hat[m][rows], f["x_hat"]) <= REL, (shape, m, relnorm(x_hat[m][rows], f["x_hat"]))
        assert abs(float(loss["loss"][m]) - float(full["loss"])) <= REL * float(full["loss"])
    before = loss["loss"].clone()
    for _ in range(3):
        after, _ = ens.step_batch(X)
    assert bool((after["loss"] < before).all()) and all(torch.isfinite(v).all() for v in ens.params.values())


@pytest.mark.parametrize("kind,d,n,B", [("tied", 4096, 1024, 192), ("untied", 5120, 512, 130)])
def test_wide_activation_widths_backward(kind, d, n, B):
    """d beyond BASELINE's 2048 (Pythia-6.9b / -12b residual widths): gradients against the fp64 oracle with the kink
    pinned, then three steps against the fp32 reference step (the Adam / renormalise / re-split row kernels hold 8 and
    16 float4 per thread at these widths)."""
    import sparse_coding_b200 as S
    torch.manual_seed(0)
    gen = torch.Generator().manual_seed(7)
    if kind == "tied":
        models = [S.FunctionalTiedSAE.init(d, n, 1e-3)]
        sig = S.FunctionalTiedSAE
    else:
        models = [S.FunctionalSAE.init(d, n, 1e-3, bias_decay=0.02)]
        sig = S.FunctionalSAE
    for p, _b in models:
        p["encoder_bias"] = 0.05 * torch.randn(n, generator=gen)
    ens = S.FunctionalEnsemble(clone_models(models), sig, S.adam, {"lr": 1e-3}, device="cuda")
    X = torch.randn(B, d, generator=gen)
    grads, (loss, aux) = ens.grads_batch(X.cuda())
    code = aux["c"].dense().cpu()
    pd = {k: v.double() for k, v in models[0][0].items()}
    alpha = float(models[0][1]["l1_alpha"])
    if kind == "tied":
        f0 = O.tied_forward(pd["encoder"], pd["encoder_bias"], X.double(), alpha)
        active = torch.where(f0["Z"].abs() < kink_window(f0["Z"]), code[0] > 0, f0["Z"] > 0)
        f = O.tied_grads(pd["encoder"], pd["encoder_bias"], X.double(), alpha, 0.0, None, active=active)
    else:
        bd = float(models[0][1]["bias_decay"])
        f0 = O.untied_forward(pd["encoder"], pd["encoder_bias"], pd["decoder"], X.double(), alpha, bd)
        active = torch.where(f0["Z"].abs() < kink_window(f0["Z"]), code[0] > 0, f0["Z"] > 0)
        f = O.untied_grads(pd["encoder"], pd["encoder_bias"], pd["decoder"], X.double(), alpha, bd, active=active)
    assert abs(float(loss["loss"][0]) - float(f0["loss"])) <= REL * float(f0["loss"])
    for k, g in f["grads"].items():
        assert relnorm(grads[k][0], g) <= 2e-4, (kind, k, relnorm(grads[k][0], g))
    ref = O.RefPortEnsemble(clone_models(models), O.SIG_LOSSES[kind], lr=1e-3)
    for _ in range(3):
        le, _ = ens.step_batch(X.cuda())
        lr_, _ = ref.step_batch(X)
    assert abs(float(le["loss"][0]) - float(lr_["loss"][0])) <= 1e-3 * float(lr_["loss"][0])
    for k in ens.params:
        assert relnorm(ens.params[k][0], ref.params[k][0]) <= 2e-3, (kind, k)


@pytest.mark.parametrize("bwd_passes", [3, 1])
def test_fvu_and_l0_match_reference_after_training(bwd_passes):
    """The quality half of the metric ("FVU vs ref"): train engine and oracle from the same initial state on the
    same 300 batches, export LearnedDicts, compare FVU (standard_metrics.py:310-314) and mean L0 (:305-308) on
    held-out data. Also run with single-pass bf16 backward GEMMs (the optional fast mode): the trained dictionaries
    must be just as good."""
    import sparse_coding_b200 as S
    from sparse_coding_b200.train_loop import unstacked_to_learned_dicts
    torch.manual_seed(0)
    d, n, B = 64, 256, 512
    models = [S.FunctionalTiedSAE.init(d, n, a) for a in (3e-4, 1e-3, 3e-3)]
    ens = S.FunctionalEnsemble(clone_models(models), S.FunctionalTiedSAE, S.adam, {"lr": 1e-3}, device="cuda",
                               bwd_passes=bwd_passes)
    ref = O.RefPortEnsemble(clone_models(models), O.SIG_LOSSES["tied"], lr=1e-3)
    gen = torch.Generator().manual_seed(1)
    feats = torch.randn(384, d, generator=gen)
    feats /= feats.norm(dim=-1, keepdim=True)

    def batch(rows):
        codes = (torch.rand(rows, 384, generator=gen) < 0.03).float() * torch.rand(rows, 384, generator=gen)
        return codes @ feats + 0.01 * torch.randn(rows, d, generator=gen)

    for _ in range(300):
        X = batch(B)
        ens.step_batch(X.cuda())
        ref.step_batch(X)
    held = batch(4096)
    mine = unstacked_to_learned_dicts(ens, {"dict_size": n}, ["dict_size"], ["l1_alpha"])
    for i, (ld, hp) in enumerate(mine):
        rp = {k: v[i] for k, v in ref.params.items()}
        rb = {k: v[i] for k, v in ref.buffers.items()}
        rld = S.FunctionalTiedSAE.to_learned_dict(rp, rb)
        fvu_e, fvu_r = float(O.fvu(held, ld.predict(held))), float(O.fvu(held, rld.predict(held)))
        l0_e = float((ld.encode(ld.center(held)) != 0).float().sum(-1).mean())
        l0_r = float((rld.encode(rld.center(held)) != 0).float().sum(-1).mean())
        assert abs(fvu_e - fvu_r) <= 0.01 * fvu_r + 1e-4, (i, fvu_e, fvu_r)
        assert abs(l0_e - l0_r) <= 0.01 * l0_r + 0.05, (i, l0_e, l0_r)
        assert fvu_r < 0.5                                      # it actually learned something


def test_topk_exact_ties_break_by_lowest_index():
    """Q8: torch.topk leaves ties unspecified; the engine keeps the lowest indices among keys equal to the k-th
    score. Duplicated dictionary rows make every score appear exactly twice, so an odd k cuts through a tie."""
    import sparse_coding_b200 as S
    torch.manual_seed(0)
    d, n, B, k = 32, 128, 64, 7
    half = torch.randn(n // 2, d)
    p = {"dict": torch.cat([half, half]).contiguous()}          # row j == row j + 64
    b = {"sparsity": torch.tensor(k, dtype=torch.long)}
    ens = S.FunctionalEnsemble([(p, b)], S.TopKEncoder, S.adam, {"lr": 1e-3}, device="cuda", no_stacking=True)
    X = torch.randn(B, d).cuda()
    loss, aux = ens.forward_batch(X)
    c = aux["c"].dense()[0].cpu()
    Wn = p["dict"] / p["dict"].norm(dim=-1, keepdim=True)
    S64 = (X.cpu().double() @ Wn.double().T)
    for r in range(B):
        row = c[r]
        assert torch.equal(row[:64] != 0, (row[:64] != 0))       # (shape sanity)
        top = torch.topk(S64[r, :64], 4).values                  # distinct values: the 4 largest, each duplicated
        assert bool((top > 0).all())
        nz = (row != 0).nonzero().flatten().tolist()
        assert len(nz) == k, (r, nz)
        lo = [j for j in nz if j < 64]
        hi = [j - 64 for j in nz if j >= 64]
        assert len(lo) == 4 and len(hi) == 3                     # the tied pair at the cut keeps its lower index
        assert set(hi) < set(lo)
        cut = (set(lo) - set(hi)).pop()
        assert abs(float(S64[r, cut]) - float(top[3])) < 1e-5    # ... and it is the 4th largest value


def test_random_shape_sweep():
    """Seeded sweep over odd shapes (every multiple-of-8 corner the plan accepts: tiny d / n, n < one tile, B = 1,
    B straddling 128/256-row tiles, single model, many models) for tied / untied / masked / top-k against the fp64
    oracle: loss within 1e-4, x̂ within 1e-4, gradients within 5e-4 with the ReLU kink pinned to the engine's side."""
    import random
    import sparse_coding_b200 as S
    rng = random.Random(1234)
    kinds = ["tied", "untied", "masked_tied", "topk"]
    cases = [(1, 8, 8, 1), (2, 8, 16, 5), (1, 16, 8, 130), (3, 24, 40, 257), (2, 136, 264, 129), (1, 8, 520, 64),
             (2, 264, 24, 300)]
    for _ in range(14):
        cases.append((rng.choice([1, 2, 3, 5]), 8 * rng.randint(1, 40), 8 * rng.randint(1, 70), rng.randint(1, 400)))
    for ci, (M, d, n, B) in enumerate(cases):
        kind = kinds[ci % len(kinds)]
        torch.manual_seed(ci)
        gen = torch.Generator().manual_seed(1000 + ci)
        if kind == "tied":
            models = [S.FunctionalTiedSAE.init(d, n, 10 ** rng.uniform(-4, -2)) for _ in range(M)]
            sig = S.FunctionalTiedSAE
        elif kind == "untied":
            models = [S.FunctionalSAE.init(d, n, 10 ** rng.uniform(-4, -2), bias_decay=rng.choice([0.0, 0.05])) for _ in range(M)]
            sig = S.FunctionalSAE
        elif kind == "masked_tied":
            models = [S.FunctionalMaskedTiedSAE.init(d, 8 * rng.randint(1, n // 8), n, 10 ** rng.uniform(-4, -2)) for _ in range(M)]
            sig = S.FunctionalMaskedTiedSAE
        else:
            models = [S.TopKEncoder.init(d, n, rng.randint(1, min(n, 24))) for _ in range(M)]
            sig = S.TopKEncoder
        for p, _b in models:
            if "encoder_bias" in p:
                p["encoder_bias"] = 0.05 * torch.randn(n, generator=gen)
        ens = S.FunctionalEnsemble([({k: v.clone() for k, v in p.items()}, b) for p, b in models], sig, S.adam,
                                   {"lr": 1e-3}, device="cuda", no_stacking=(kind == "topk"))
        X = torch.randn(B, d, generator=gen)
        grads, (loss, aux) = ens.grads_batch(X.cuda())
        code = aux["c"].dense().cpu()                      # before the next engine call reuses the code buffers
        _, _, x_hat = ens.forward_batch(X.cuda(), return_x_hat=True)
        tag = (ci, kind, M, d, n, B)
        for i, (p, b) in enumerate(models):
            pd = {k: v.double() for k, v in p.items()}
            Xd = X.double()
            if kind == "topk":
                k = int(b["sparsity"])
                Wn, _ = O.unit_rows(pd["dict"], floor=None)
                Sc = Xd @ Wn.T
                support = code[i] > 0
                kept = torch.where(support, Sc, torch.full_like(Sc, float("inf"))).min(-1).values
                dropped = torch.where(support, torch.full_like(Sc, -float("inf")), Sc).max(-1).values
                assert int(support.sum(-1).max()) <= k and bool((kept >= dropped.clamp(min=0) - 1e-5).all()), tag
                xh = (Sc.clamp(min=0) * support) @ Wn
                ref_loss = (Xd - xh).pow(2).mean()
                assert relnorm(x_hat[i], xh) <= REL, tag
                assert abs(float(loss["loss"][i]) - float(ref_loss)) <= REL * float(ref_loss), tag
                continue
            mask = b["coef_mask"] if kind == "masked_tied" else None
            alpha = float(b["l1_alpha"])
            if kind == "untied":
                f0 = O.untied_forward(pd["encoder"], pd["encoder_bias"], pd["decoder"], Xd, alpha, float(b["bias_decay"]))
            else:
                f0 = O.tied_forward(pd["encoder"], pd["encoder_bias"], Xd, alpha, 0.0, mask)
            assert relnorm(x_hat[i], f0["x_hat"]) <= REL, tag
            assert abs(float(loss["loss"][i]) - float(f0["loss"])) <= REL * abs(float(f0["loss"])) + 1e-12, tag
            if kind != "untied":
                active = torch.where(f0["Z"].abs() < kink_window(f0["Z"]), code[i] > 0, f0["Z"] > 0)
                f = O.tied_grads(pd["encoder"], pd["encoder_bias"], Xd, alpha, 0.0, mask, active=active)
                assert relnorm(grads["encoder"][i], f["grads"]["encoder"]) <= 5e-4, tag
                assert relnorm(grads["encoder_bias"][i], f["grads"]["encoder_bias"]) <= 5e-4, tag
        del ens


@pytest.mark.parametrize("kind", ["tied", "untied", "topk"])
def test_bitwise_determinism(kind):
    """Two runs from the same state on the same batches give bit-identical parameters, moments and losses: every
    reduction in the engine has a fixed order (per-warp partials reduced by a finalisation kernel, no floating-point
    atomics), unlike the reference's cuBLAS / atomics-based PyTorch path."""
    import sparse_coding_b200 as S
    d, n, B = 96, 320, 300
    torch.manual_seed(0)
    if kind == "tied":
        models, sig = [S.FunctionalTiedSAE.init(d, n, a) for a in (1e-3, 1e-2)], S.FunctionalTiedSAE
    elif kind == "untied":
        models, sig = [S.FunctionalSAE.init(d, n, a, bias_decay=0.01) for a in (1e-3, 1e-2)], S.FunctionalSAE
    else:
        models, sig = [S.TopKEncoder.init(d, n, k) for k in (8, 24)], S.TopKEncoder
    gen = torch.Generator().manual_seed(1)
    batches = [torch.randn(B, d, generator=gen).cuda() for _ in range(6)]
    runs = []
    for _ in range(2):
        ens = S.FunctionalEnsemble(clone_models(models), sig, S.adam, {"lr": 1e-3}, device="cuda")
        losses = [ens.step_batch(x)[0]["loss"].clone() for x in batches]
        runs.append((ens.params, ens.optim_states, losses))
    for k in runs[0][0]:
        assert torch.equal(runs[0][0][k], runs[1][0][k])
        assert torch.equal(runs[0][1]["nu"][k], runs[1][1]["nu"][k])
    assert all(torch.equal(a, b) for a, b in zip(runs[0][2], runs[1][2]))


def test_gemm_selftest(tmp_path):
    """The standalone check of the GEMM core (tests/csrc/gemm_selftest.cu): the seven configurations libsce launches
    against a double-precision product of the same planes, ragged edges included; the accuracy of the f16f8 cross-term
    accumulation (native and widened) at reduction lengths up to 16384; and the f16f8 weight gradient with mixed
    operand layouts, native against widened. Each configuration's `_persist` case (f16f8 MN x MN both native and
    widened) has more than two output tiles per SM, so persistent CTAs run second and partial tiles."""
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(root, "build", "gemm_selftest")
    if not os.path.exists(exe):   # build() makes it; a tree built with `make` alone may not have it
        exe = str(tmp_path / "gemm_selftest")
        subprocess.run(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-o", exe,
                        os.path.join(root, "tests", "csrc", "gemm_selftest.cu")], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1800)
    print(r.stdout)
    assert r.returncode == 0 and "ALL PASS" in r.stdout, r.stdout[-4000:] + r.stderr[-2000:]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    persist = re.findall(r"\[(\w+_persist(?:/\w+)?)\] PASS .* tiles=(\d+)", r.stdout)
    assert len(persist) == 7 and all(int(t) > 2 * sms for _, t in persist), (sms, persist)
