"""How each engine signature is wired into a plan, without a GPU: the descriptor and the buffer slots that
``_lib.plan_structs`` fills for every signature ``FunctionalEnsemble`` trains, and for every kind of dictionary the
evaluation passes of ``metrics`` plan. Each slot is matched to the tensor it must point at (NULL where none), and
every descriptor field to its value, for shared and per-model batches, FunctionalTiedSAE's centring, several top-k k
and padded / centred dictionary groups."""
import ctypes as C

import numpy as np
import pytest
import torch

import sparse_coding_b200 as S
from sparse_coding_b200 import _lib
from sparse_coding_b200 import metrics as MT
from sparse_coding_b200.ensemble import FunctionalEnsemble
from sparse_coding_b200.learned_dict import TiedSAE, UntiedSAE
from sparse_coding_b200.topk_encoder import TopKLearnedDict

D, N = 32, 64
FLOAT_FIELDS = {"lr", "beta1", "beta2", "eps", "eps_root", "norm_floor", "input_shift"}

# Per case: every SceDesc field, and the SceBuffers slots that are set (all others are NULL). Ensemble slots name a
# tensor of the ensemble ("params.encoder", "mu.encoder", ...) or a converted copy of a buffer ("buffers.name:dtype");
# evaluation slots name what the dictionary plan holds: the padded stacks "enc", "bias", "dec", the one placeholder
# "unused" for every Adam moment, the padding "mask", the "sparsity" ks and the centring "trans", "rot", "scale".
EXPECTED = {
    "tied_shared": (
        dict(variant=0, n_models=2, d=32, n=64, batch_max=64, x_per_model=0, lr=0.001, beta1=0.9, beta2=0.999,
             eps=1e-08, eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=0,
             topk_k_max=0, centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.encoder", "encoder_bias": "params.encoder_bias", "encoder_m": "mu.encoder", "encoder_v":
         "nu.encoder", "bias_m": "mu.encoder_bias", "bias_v": "nu.encoder_bias", "l1_alpha": "buffers.l1_alpha:float32",
         "bias_decay": "buffers.bias_decay:float32"}),
    "tied_per_model": (
        dict(variant=0, n_models=2, d=32, n=64, batch_max=48, x_per_model=1, lr=0.0003, beta1=0.8, beta2=0.99,
             eps=1e-06, eps_root=0.0, adam_count_mode=1, fwd_passes=1, bwd_passes=1, norm_floor=1e-08, arith=1,
             topk_k_max=0, centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.encoder", "encoder_bias": "params.encoder_bias", "encoder_m": "mu.encoder", "encoder_v":
         "nu.encoder", "bias_m": "mu.encoder_bias", "bias_v": "nu.encoder_bias", "l1_alpha": "buffers.l1_alpha:float32",
         "bias_decay": "buffers.bias_decay:float32"}),
    "tied_centred_shared": (
        dict(variant=0, n_models=2, d=32, n=64, batch_max=64, x_per_model=1, lr=0.001, beta1=0.9, beta2=0.999,
             eps=1e-08, eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=0,
             topk_k_max=0, centering=1, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.encoder", "encoder_bias": "params.encoder_bias", "encoder_m": "mu.encoder", "encoder_v":
         "nu.encoder", "bias_m": "mu.encoder_bias", "bias_v": "nu.encoder_bias", "l1_alpha": "buffers.l1_alpha:float32",
         "bias_decay": "buffers.bias_decay:float32", "center_trans": "buffers.center_trans:float32", "center_rot":
         "buffers.center_rot:float32", "center_scale": "buffers.center_scale:float32"}),
    "tied_centred_per_model": (
        dict(variant=0, n_models=2, d=32, n=64, batch_max=40, x_per_model=1, lr=0.001, beta1=0.9, beta2=0.999,
             eps=1e-08, eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=2,
             topk_k_max=0, centering=2, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.encoder", "encoder_bias": "params.encoder_bias", "encoder_m": "mu.encoder", "encoder_v":
         "nu.encoder", "bias_m": "mu.encoder_bias", "bias_v": "nu.encoder_bias", "l1_alpha": "buffers.l1_alpha:float32",
         "bias_decay": "buffers.bias_decay:float32", "center_trans": "buffers.center_trans:float32", "center_rot":
         "buffers.center_rot:float32", "center_scale": "buffers.center_scale:float32"}),
    "masked_tied_shared": (
        dict(variant=0, n_models=2, d=32, n=64, batch_max=64, x_per_model=0, lr=0.001, beta1=0.9, beta2=0.999,
             eps=1e-08, eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=0,
             topk_k_max=0, centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.encoder", "encoder_bias": "params.encoder_bias", "encoder_m": "mu.encoder", "encoder_v":
         "nu.encoder", "bias_m": "mu.encoder_bias", "bias_v": "nu.encoder_bias", "l1_alpha": "buffers.l1_alpha:float32",
         "coef_mask": "buffers.coef_mask:uint8"}),
    "masked_tied_per_model": (
        dict(variant=0, n_models=3, d=32, n=64, batch_max=32, x_per_model=1, lr=0.0003, beta1=0.8, beta2=0.99,
             eps=1e-06, eps_root=0.0, adam_count_mode=1, fwd_passes=1, bwd_passes=1, norm_floor=1e-08, arith=1,
             topk_k_max=0, centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.encoder", "encoder_bias": "params.encoder_bias", "encoder_m": "mu.encoder", "encoder_v":
         "nu.encoder", "bias_m": "mu.encoder_bias", "bias_v": "nu.encoder_bias", "l1_alpha": "buffers.l1_alpha:float32",
         "coef_mask": "buffers.coef_mask:uint8"}),
    "untied_shared": (
        dict(variant=1, n_models=2, d=32, n=64, batch_max=64, x_per_model=0, lr=0.001, beta1=0.9, beta2=0.999,
             eps=1e-08, eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=2,
             topk_k_max=0, centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.encoder", "encoder_bias": "params.encoder_bias", "decoder": "params.decoder", "encoder_m":
         "mu.encoder", "encoder_v": "nu.encoder", "bias_m": "mu.encoder_bias", "bias_v": "nu.encoder_bias", "decoder_m":
         "mu.decoder", "decoder_v": "nu.decoder", "l1_alpha": "buffers.l1_alpha:float32", "bias_decay":
         "buffers.bias_decay:float32"}),
    "untied_per_model": (
        dict(variant=1, n_models=2, d=32, n=64, batch_max=16, x_per_model=1, lr=0.0003, beta1=0.8, beta2=0.99,
             eps=1e-06, eps_root=0.0, adam_count_mode=1, fwd_passes=1, bwd_passes=1, norm_floor=1e-08, arith=1,
             topk_k_max=0, centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.encoder", "encoder_bias": "params.encoder_bias", "decoder": "params.decoder", "encoder_m":
         "mu.encoder", "encoder_v": "nu.encoder", "bias_m": "mu.encoder_bias", "bias_v": "nu.encoder_bias", "decoder_m":
         "mu.decoder", "decoder_v": "nu.decoder", "l1_alpha": "buffers.l1_alpha:float32", "bias_decay":
         "buffers.bias_decay:float32"}),
    "masked_untied_shared": (
        dict(variant=1, n_models=2, d=32, n=64, batch_max=64, x_per_model=0, lr=0.001, beta1=0.9, beta2=0.999,
             eps=1e-08, eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=0,
             topk_k_max=0, centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.encoder", "encoder_bias": "params.encoder_bias", "decoder": "params.decoder", "encoder_m":
         "mu.encoder", "encoder_v": "nu.encoder", "bias_m": "mu.encoder_bias", "bias_v": "nu.encoder_bias", "decoder_m":
         "mu.decoder", "decoder_v": "nu.decoder", "l1_alpha": "buffers.l1_alpha:float32", "coef_mask":
         "buffers.coef_mask:uint8"}),
    "masked_untied_per_model": (
        dict(variant=1, n_models=3, d=32, n=64, batch_max=24, x_per_model=1, lr=0.0003, beta1=0.8, beta2=0.99,
             eps=1e-06, eps_root=0.0, adam_count_mode=1, fwd_passes=1, bwd_passes=1, norm_floor=1e-08, arith=1,
             topk_k_max=0, centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.encoder", "encoder_bias": "params.encoder_bias", "decoder": "params.decoder", "encoder_m":
         "mu.encoder", "encoder_v": "nu.encoder", "bias_m": "mu.encoder_bias", "bias_v": "nu.encoder_bias", "decoder_m":
         "mu.decoder", "decoder_v": "nu.decoder", "l1_alpha": "buffers.l1_alpha:float32", "coef_mask":
         "buffers.coef_mask:uint8"}),
    "topk_shared": (
        dict(variant=2, n_models=2, d=32, n=64, batch_max=64, x_per_model=0, lr=0.001, beta1=0.9, beta2=0.999,
             eps=1e-08, eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=0.0, arith=0,
             topk_k_max=8, centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.dict", "encoder_m": "mu.dict", "encoder_v": "nu.dict", "sparsity":
         "buffers.sparsity:int64"}),
    "topk_per_model": (
        dict(variant=2, n_models=3, d=32, n=64, batch_max=32, x_per_model=1, lr=0.0003, beta1=0.8, beta2=0.99,
             eps=1e-06, eps_root=0.0, adam_count_mode=1, fwd_passes=1, bwd_passes=1, norm_floor=0.0, arith=1,
             topk_k_max=48, centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.dict", "encoder_m": "mu.dict", "encoder_v": "nu.dict", "sparsity":
         "buffers.sparsity:int64"}),
    "topk_large_k": (
        dict(variant=2, n_models=2, d=32, n=512, batch_max=64, x_per_model=0, lr=0.001, beta1=0.9, beta2=0.999,
             eps=1e-08, eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=0.0, arith=2,
             topk_k_max=300, centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.dict", "encoder_m": "mu.dict", "encoder_v": "nu.dict", "sparsity":
         "buffers.sparsity:int64"}),
    "learned_center_shared": (
        dict(variant=3, n_models=2, d=32, n=64, batch_max=64, x_per_model=0, lr=0.001, beta1=0.9, beta2=0.999,
             eps=1e-08, eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=0,
             topk_k_max=0, centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.encoder", "encoder_bias": "params.encoder_bias", "encoder_m": "mu.encoder", "encoder_v":
         "nu.encoder", "bias_m": "mu.encoder_bias", "bias_v": "nu.encoder_bias", "l1_alpha": "buffers.l1_alpha:float32",
         "center": "params.center", "center_m": "mu.center", "center_v": "nu.center"}),
    "learned_center_per_model": (
        dict(variant=3, n_models=2, d=32, n=64, batch_max=56, x_per_model=1, lr=0.0003, beta1=0.8, beta2=0.99,
             eps=1e-06, eps_root=0.0, adam_count_mode=1, fwd_passes=1, bwd_passes=1, norm_floor=1e-08, arith=1,
             topk_k_max=0, centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "params.encoder", "encoder_bias": "params.encoder_bias", "encoder_m": "mu.encoder", "encoder_v":
         "nu.encoder", "bias_m": "mu.encoder_bias", "bias_v": "nu.encoder_bias", "l1_alpha": "buffers.l1_alpha:float32",
         "center": "params.center", "center_m": "mu.center", "center_v": "nu.center"}),
    "positive_tied_shared": (
        dict(variant=0, n_models=2, d=32, n=64, batch_max=64, x_per_model=0, lr=0.001, beta1=0.9, beta2=0.999,
             eps=1e-08, eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=0,
             topk_k_max=0, centering=0, encoder_nonneg=1, input_shift=0.18),
        {"encoder": "params.encoder", "encoder_bias": "params.encoder_bias", "encoder_m": "mu.encoder", "encoder_v":
         "nu.encoder", "bias_m": "mu.encoder_bias", "bias_v": "nu.encoder_bias", "l1_alpha": "buffers.l1_alpha:float32",
         "bias_decay": "buffers.bias_decay:float32"}),
    "positive_tied_per_model": (
        dict(variant=0, n_models=2, d=32, n=64, batch_max=64, x_per_model=1, lr=0.001, beta1=0.9, beta2=0.999,
             eps=1e-08, eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=2,
             topk_k_max=0, centering=0, encoder_nonneg=1, input_shift=0.18),
        {"encoder": "params.encoder", "encoder_bias": "params.encoder_bias", "encoder_m": "mu.encoder", "encoder_v":
         "nu.encoder", "bias_m": "mu.encoder_bias", "bias_v": "nu.encoder_bias", "l1_alpha": "buffers.l1_alpha:float32",
         "bias_decay": "buffers.bias_decay:float32"}),
    "eval_tied": (
        dict(variant=0, n_models=2, d=32, n=64, batch_max=128, x_per_model=0, lr=0.0, beta1=0.9, beta2=0.999, eps=1e-08,
             eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=1, topk_k_max=0,
             centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "enc", "encoder_bias": "bias", "encoder_m": "unused", "encoder_v": "unused", "bias_m": "unused",
         "bias_v": "unused"}),
    "eval_tied_padded": (
        dict(variant=0, n_models=2, d=32, n=64, batch_max=96, x_per_model=0, lr=0.0, beta1=0.9, beta2=0.999, eps=1e-08,
             eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=1, topk_k_max=0,
             centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "enc", "encoder_bias": "bias", "encoder_m": "unused", "encoder_v": "unused", "bias_m": "unused",
         "bias_v": "unused", "coef_mask": "mask"}),
    "eval_tied_centred": (
        dict(variant=0, n_models=2, d=32, n=64, batch_max=128, x_per_model=1, lr=0.0, beta1=0.9, beta2=0.999, eps=1e-08,
             eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=2, topk_k_max=0,
             centering=1, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "enc", "encoder_bias": "bias", "encoder_m": "unused", "encoder_v": "unused", "bias_m": "unused",
         "bias_v": "unused", "center_trans": "trans", "center_rot": "rot", "center_scale": "scale"}),
    "eval_tied_centred_padded": (
        dict(variant=0, n_models=2, d=32, n=48, batch_max=64, x_per_model=1, lr=0.0, beta1=0.9, beta2=0.999, eps=1e-08,
             eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=1, topk_k_max=0,
             centering=1, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "enc", "encoder_bias": "bias", "encoder_m": "unused", "encoder_v": "unused", "bias_m": "unused",
         "bias_v": "unused", "coef_mask": "mask", "center_trans": "trans", "center_rot": "rot", "center_scale":
         "scale"}),
    "eval_untied": (
        dict(variant=1, n_models=1, d=32, n=64, batch_max=128, x_per_model=0, lr=0.0, beta1=0.9, beta2=0.999, eps=1e-08,
             eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=1, topk_k_max=0,
             centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "enc", "encoder_bias": "bias", "decoder": "dec", "encoder_m": "unused", "encoder_v": "unused",
         "bias_m": "unused", "bias_v": "unused", "decoder_m": "unused", "decoder_v": "unused"}),
    "eval_untied_padded": (
        dict(variant=1, n_models=2, d=32, n=64, batch_max=32, x_per_model=0, lr=0.0, beta1=0.9, beta2=0.999, eps=1e-08,
             eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=1e-08, arith=2, topk_k_max=0,
             centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "enc", "encoder_bias": "bias", "decoder": "dec", "encoder_m": "unused", "encoder_v": "unused",
         "bias_m": "unused", "bias_v": "unused", "decoder_m": "unused", "decoder_v": "unused", "coef_mask": "mask"}),
    "eval_topk": (
        dict(variant=2, n_models=2, d=32, n=64, batch_max=128, x_per_model=0, lr=0.0, beta1=0.9, beta2=0.999, eps=1e-08,
             eps_root=0.0, adam_count_mode=0, fwd_passes=3, bwd_passes=3, norm_floor=0.0, arith=1, topk_k_max=9,
             centering=0, encoder_nonneg=0, input_shift=0.0),
        {"encoder": "enc", "encoder_m": "unused", "encoder_v": "unused", "sparsity": "sparsity"}),
}


def _models(sig, M):
    torch.manual_seed(0)
    out = []
    for m in range(M):
        l1, bd = 1e-3 * (m + 1), 0.1 * m
        if sig is S.FunctionalSAE or sig is S.FunctionalPositiveTiedSAE:
            out.append(sig.init(D, N, l1, bd))
        elif sig is S.FunctionalTiedSAE:
            out.append(sig.init(D, N, l1, bias_decay=bd))
        elif sig is S.FunctionalTiedCenteredSAE:
            out.append(sig.init(D, N, l1))
        else:   # the masked signatures: model m uses N - 8 m of the N rows
            out.append(sig.init(D, N - 8 * m, N, l1, bd))
    return out


def _ens(sig, M=2, n=N, ks=None, centred=False, opt=None, **kw):
    if sig is S.TopKEncoder:
        torch.manual_seed(0)
        models = [sig.init(D, n, k) for k in ks]
    else:
        models = _models(sig, M)
    if centred:
        for m, (_, b) in enumerate(models):
            b["center_trans"] = torch.full((D,), 0.5 * (m + 1))
            b["center_scale"] = torch.full((D,), 2.0)
    return FunctionalEnsemble(models, sig, "adam", opt or {"lr": 1e-3}, device="cpu", **kw)


_STD = dict(adam_count_mode="standard", fwd_passes=1, bwd_passes=1, arith="bf16x3",
            opt={"lr": 3e-4, "betas": (0.8, 0.99), "eps": 1e-6})
_F8 = dict(arith="f16f8")
# name -> (ensemble, (batch_max, x_per_model, centering))
ENSEMBLE_CASES = {
    "tied_shared": (lambda: _ens(S.FunctionalTiedSAE), (64, False, 0)),
    "tied_per_model": (lambda: _ens(S.FunctionalTiedSAE, **_STD), (48, True, 0)),
    "tied_centred_shared": (lambda: _ens(S.FunctionalTiedSAE, centred=True), (64, True, 1)),
    "tied_centred_per_model": (lambda: _ens(S.FunctionalTiedSAE, centred=True, **_F8), (40, True, 2)),
    "masked_tied_shared": (lambda: _ens(S.FunctionalMaskedTiedSAE), (64, False, 0)),
    "masked_tied_per_model": (lambda: _ens(S.FunctionalMaskedTiedSAE, M=3, **_STD), (32, True, 0)),
    "untied_shared": (lambda: _ens(S.FunctionalSAE, **_F8), (64, False, 0)),
    "untied_per_model": (lambda: _ens(S.FunctionalSAE, **_STD), (16, True, 0)),
    "masked_untied_shared": (lambda: _ens(S.FunctionalMaskedSAE), (64, False, 0)),
    "masked_untied_per_model": (lambda: _ens(S.FunctionalMaskedSAE, M=3, **_STD), (24, True, 0)),
    "topk_shared": (lambda: _ens(S.TopKEncoder, ks=[4, 8]), (64, False, 0)),
    "topk_per_model": (lambda: _ens(S.TopKEncoder, ks=[1, 16, 48], **_STD), (32, True, 0)),
    "topk_large_k": (lambda: _ens(S.TopKEncoder, n=512, ks=[300, 7], **_F8), (64, False, 0)),
    "learned_center_shared": (lambda: _ens(S.FunctionalTiedCenteredSAE), (64, False, 0)),
    "learned_center_per_model": (lambda: _ens(S.FunctionalTiedCenteredSAE, **_STD), (56, True, 0)),
    "positive_tied_shared": (lambda: _ens(S.FunctionalPositiveTiedSAE), (64, False, 0)),
    "positive_tied_per_model": (lambda: _ens(S.FunctionalPositiveTiedSAE, **_F8), (64, True, 0)),
}


def _tied(n, trans=0.0):
    torch.manual_seed(n)
    c = (torch.full((D,), trans), torch.eye(D), torch.ones(D)) if trans else (None, None, None)
    return TiedSAE(torch.randn(n, D), torch.randn(n), centering=c)


def _untied(n):
    torch.manual_seed(n)
    return UntiedSAE(torch.randn(n, D), torch.randn(n, D), torch.randn(n))


def _topk(n, k):
    torch.manual_seed(n + k)
    return TopKLearnedDict(torch.randn(n, D), k)


# name -> (dictionaries, centre, arith, batch_max): each forms one evaluation group
METRICS_CASES = {
    "eval_tied": (lambda: [_tied(64), _tied(64)], True, "bf16x3", 128),
    "eval_tied_padded": (lambda: [_tied(64), _tied(60)], False, "bf16x3", 96),
    "eval_tied_centred": (lambda: [_tied(64, 0.25), _tied(64, 0.5)], True, "f16f8", 128),
    "eval_tied_centred_padded": (lambda: [_tied(48, 0.25), _tied(44, 0.5)], True, "auto", 64),
    "eval_untied": (lambda: [_untied(64)], True, "bf16x3", 128),
    "eval_untied_padded": (lambda: [_untied(64), _untied(60)], True, "f16f8", 32),
    "eval_topk": (lambda: [_topk(64, 4), _topk(64, 9)], True, "bf16x3", 128),
}


def _check_desc(desc, want):
    assert [f for f, _ in _lib.SceDesc._fields_] == list(want)
    for f, v in want.items():
        got = getattr(desc, f)
        if f in FLOAT_FIELDS:
            assert got == float(np.float32(v)), f
        else:
            assert got == v, f


def _slots(bufs):
    """{slot: address} of every set SceBuffers slot (the workspace is create_plan's)."""
    out = {f: getattr(bufs, f) for f, _ in _lib.SceBuffers._fields_ if f not in ("workspace", "workspace_bytes")}
    assert bufs.workspace is None and bufs.workspace_bytes == 0
    return {f: p for f, p in out.items() if p}


def _read(addr, like):
    """The memory at ``addr`` as a tensor shaped and typed like ``like``."""
    raw = (C.c_uint8 * (like.numel() * like.element_size())).from_address(addr)
    return torch.frombuffer(raw, dtype=like.dtype).reshape(like.shape).clone()


@pytest.mark.parametrize("name", list(ENSEMBLE_CASES))
def test_ensemble_plan_wiring(name):
    make, (batch_max, x_per_model, centering) = ENSEMBLE_CASES[name]
    want_desc, want_slots = EXPECTED[name]
    ens = make()
    desc, bufs, keep = _lib.plan_structs(
        _lib.SIGNATURES[ens.sig.variant], ens.params, ens.buffers, ens.optim_states["mu"], ens.optim_states["nu"],
        batch_max=batch_max, x_per_model=x_per_model, centering=centering, adam=ens.optimizer,
        adam_count_mode=ens.adam_count_mode, fwd_passes=ens.fwd_passes, bwd_passes=ens.bwd_passes, arith=ens.arith)
    _check_desc(desc, want_desc)
    slots = _slots(bufs)
    assert set(slots) == set(want_slots)
    trees = {"params": ens.params, "mu": ens.optim_states["mu"], "nu": ens.optim_states["nu"]}
    converted = set()
    for slot, label in want_slots.items():
        tree, key = label.split(".")
        if tree == "buffers":
            key, dtype = key.split(":")
            t = keep[key]
            assert t.dtype == getattr(torch, dtype) and t.is_contiguous()
            assert torch.equal(t, ens.buffers[key].to(t.dtype))
            converted.add(key)
        else:
            t = trees[tree][key]
        assert slots[slot] == t.data_ptr(), slot
    # FunctionalEnsemble.refresh refills exactly these copies
    assert set(keep) == converted


@pytest.mark.parametrize("name", list(METRICS_CASES))
def test_dictionary_plan_wiring(name, monkeypatch):
    make, centre, arith, batch_max = METRICS_CASES[name]
    want_desc, want_slots = EXPECTED[name]
    lds = make()
    _, groups, ar = MT._dict_inputs(lds, torch.zeros(4, D), arith, centre)
    (key, idx), = groups.items()
    assert idx == list(range(len(lds)))
    kind, n_pad, _, centred = key
    M = len(lds)

    def padded(ts):
        out = torch.zeros((M, n_pad) + tuple(ts[0].shape[1:]))
        for m, t in enumerate(ts):
            out[m, : t.shape[0]] = t
        return out

    expect = {"unused": torch.zeros(1)}
    if kind == "topk":
        expect["enc"] = padded([ld.dict for ld in lds])
        expect["sparsity"] = torch.tensor([ld.sparsity for ld in lds], dtype=torch.int64)
    else:
        expect["enc"] = padded([ld.encoder for ld in lds])
        expect["bias"] = padded([ld.encoder_bias for ld in lds])
        if kind == "untied":
            expect["dec"] = padded([ld.decoder for ld in lds])
        sizes = torch.tensor([ld.n_feats for ld in lds])
        expect["mask"] = (torch.arange(n_pad)[None, :] >= sizes[:, None]).to(torch.uint8)
    if centred:
        for k in ("trans", "rot", "scale"):
            expect[k] = torch.stack([getattr(ld, "center_" + k) for ld in lds])

    seen = {}

    class Captured(Exception):
        pass

    def create_plan(desc, bufs, device):   # reads the slots while the plan's tensors are alive
        _check_desc(desc, want_desc)
        slots = _slots(bufs)
        assert set(slots) == set(want_slots)
        for slot, label in want_slots.items():
            assert torch.equal(_read(slots[slot], expect[label]), expect[label]), slot
            seen.setdefault(label, set()).add(slots[slot])
        raise Captured

    monkeypatch.setattr(_lib, "create_plan", create_plan)
    with pytest.raises(Captured):
        MT._DictPlan(key, [lds[i] for i in idx], batch_max, ar, torch.device("cpu"))
    assert all(len(addrs) == 1 for addrs in seen.values())   # one placeholder for every moment
