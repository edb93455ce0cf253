"""SAE signatures on the accelerated hot path (reference: autoencoders/sae_ensemble.py).

    FunctionalSAE            untied encoder/decoder        sae_ensemble.py:13-78
    FunctionalTiedSAE        tied, optional centring       sae_ensemble.py:81-162
    FunctionalTiedCenteredSAE tied, learned centre         sae_ensemble.py:164-230
    FunctionalPositiveTiedSAE tied, clamped encoder        mlp_tests.py:68-125
    FunctionalMaskedTiedSAE  tied, per-model dict size     sae_ensemble.py:309-373
    FunctionalMaskedSAE      untied, per-model dict size   sae_ensemble.py:377-444

``init`` keeps the reference's positional orders and initialisers (xavier-uniform matrices, zero bias, 0-dim
hyper-parameter buffers) so that seeded initialisation is bit-identical; ``to_learned_dict`` builds the same export
objects. ``loss`` is evaluated by the CUDA engine. Differences from the reference, both deliberate:
  * FunctionalTiedSAE.init stores ``bias_decay`` in the buffers. The reference accepts the argument, drops it, and
    then reads ``buffers["bias_decay"]`` in ``loss`` (:150) — a KeyError at HEAD (SURVEY.md Q1).
  * the centring of FunctionalTiedSAE is applied once to the batch, the identity case is skipped, and the unused
    un-centred reconstruction (:146) is not computed (SURVEY.md Q6).
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .learned_dict import NORM_FLOOR, TiedSAE, UntiedSAE
from .signatures import DictSignature, engine_loss

_REF_MODULE = "autoencoders.sae_ensemble"


def _xavier(n, d, device, dtype):
    w = torch.empty((n, d), device=device, dtype=dtype)
    nn.init.xavier_uniform_(w)
    return w


class FunctionalSAE(DictSignature):
    variant = "untied"

    @staticmethod
    def init(activation_size, n_dict_components, l1_alpha, bias_decay=0.0, device=None, dtype=None):
        params = {}
        params["encoder"] = _xavier(n_dict_components, activation_size, device, dtype)
        params["encoder_bias"] = torch.zeros((n_dict_components,), device=device, dtype=dtype)
        params["decoder"] = _xavier(n_dict_components, activation_size, device, dtype)
        buffers = {
            "l1_alpha": torch.tensor(l1_alpha, device=device, dtype=dtype),
            "bias_decay": torch.tensor(bias_decay, device=device, dtype=dtype),
        }
        return params, buffers

    @staticmethod
    def to_learned_dict(params, buffers):
        return UntiedSAE(params["encoder"], params["decoder"], params["encoder_bias"])

    @staticmethod
    def learned_dict_stack(params, buffers):
        return params["decoder"], NORM_FLOOR, None

    @staticmethod
    def encode(params, buffers, batch):
        return (batch @ params["encoder"].T + params["encoder_bias"]).clamp(min=0.0)

    @staticmethod
    def loss(params, buffers, batch):
        return engine_loss(FunctionalSAE, params, buffers, batch)


class FunctionalTiedSAE(DictSignature):
    variant = "tied"

    @staticmethod
    def init(activation_size, n_dict_components, l1_alpha, device=None, dtype=None, bias_decay=0.0,
             translation=None, rotation=None, scaling=None):
        buffers = {}
        buffers["center_rot"] = (torch.eye(activation_size, device=device, dtype=dtype)
                                 if rotation is None else rotation)
        buffers["center_trans"] = (torch.zeros(activation_size, device=device, dtype=dtype)
                                   if translation is None else translation)
        buffers["center_scale"] = (torch.ones(activation_size, device=device, dtype=dtype)
                                   if scaling is None else scaling)
        params = {}
        params["encoder"] = _xavier(n_dict_components, activation_size, device, dtype)
        params["encoder_bias"] = torch.zeros((n_dict_components,), device=device, dtype=dtype)
        buffers["l1_alpha"] = torch.tensor(l1_alpha, device=device, dtype=dtype)
        buffers["bias_decay"] = torch.tensor(bias_decay, device=device, dtype=dtype)  # Q1, see module docstring
        return params, buffers

    @staticmethod
    def to_learned_dict(params, buffers):
        return TiedSAE(params["encoder"], params["encoder_bias"],
                       centering=(buffers["center_trans"], buffers["center_rot"], buffers["center_scale"]),
                       norm_encoder=True)

    @staticmethod
    def learned_dict_stack(params, buffers):
        return params["encoder"], NORM_FLOOR, None

    @staticmethod
    def center(buffers, batch):
        return ((batch - buffers["center_trans"][None, :]) @ buffers["center_rot"].T) * buffers["center_scale"][None, :]

    @staticmethod
    def uncenter(buffers, batch):
        return (batch / buffers["center_scale"][None, :]) @ buffers["center_rot"] + buffers["center_trans"][None, :]

    @staticmethod
    def loss(params, buffers, batch):
        return engine_loss(FunctionalTiedSAE, params, buffers, batch)


class FunctionalTiedCenteredSAE(DictSignature):
    """A tied SAE on ``x - center``, the centre a trained parameter (a learned pre-encoder bias): loss
    ``mean((x̂_c - x_c)^2) + l1_alpha * mean_b sum_n |c|`` with ``x_c = x - center``, no bias decay. The engine computes
    the centre's gradient ``sum_b g_b - db W`` and updates it with Adam like the other parameters."""
    variant = "tied_learned_center"

    @staticmethod
    def init(activation_size, n_dict_components, l1_alpha, center=None, device=None, dtype=None):
        params = {}
        buffers = {}
        # the reference's order (zero centre, then the xavier encoder, then the zero bias): seeded init is bitwise its own
        params["center"] = torch.zeros(activation_size, device=device, dtype=dtype) if center is None else center
        params["encoder"] = _xavier(n_dict_components, activation_size, device, dtype)
        params["encoder_bias"] = torch.zeros((n_dict_components,), device=device, dtype=dtype)
        buffers["l1_alpha"] = torch.tensor(l1_alpha, device=device, dtype=dtype)
        return params, buffers

    @staticmethod
    def to_learned_dict(params, buffers):
        return TiedSAE(params["encoder"], params["encoder_bias"], centering=(params["center"], None, None),
                       norm_encoder=True)

    @staticmethod
    def learned_dict_stack(params, buffers):
        return params["encoder"], NORM_FLOOR, None

    @staticmethod
    def center(params, batch):
        return batch - params["center"][None, :]

    @staticmethod
    def uncenter(params, batch):
        return batch + params["center"][None, :]

    @staticmethod
    def loss(params, buffers, batch):
        return engine_loss(FunctionalTiedCenteredSAE, params, buffers, batch)


class FunctionalPositiveTiedSAE(DictSignature):
    """A tied SAE on non-negative dictionary rows (reference: autoencoders/mlp_tests.py:68-125): the loss reads the
    encoder clamped at 0, ``W = max(E, 0) / max(||max(E, 0)||, 1e-8)``, encodes and reconstructs ``x + 0.18``, and adds
    bias decay: ``mean((x̂ - 0.18 - x)^2) + l1_alpha * mean_b sum_n |c| + bias_decay * ||b||``. As in the reference,
    the encoder's gradient is taken with respect to the clamped encoder and applied to the raw one (straight-through),
    so entries that went negative keep moving. The export is the reference's: a plain ``TiedSAE`` of the raw encoder,
    with neither the clamp nor the shift, so an exported dictionary's FVU is not the training loss."""
    variant = "positive_tied"

    @staticmethod
    def init(activation_size, n_dict_components, l1_alpha, bias_decay=0.0, device=None, dtype=None):
        params = {}
        buffers = {}
        params["encoder"] = _xavier(n_dict_components, activation_size, device, dtype).abs()
        params["encoder_bias"] = torch.full((n_dict_components,), -1.0, device=device, dtype=dtype)
        buffers["l1_alpha"] = torch.tensor(l1_alpha, device=device, dtype=dtype)
        buffers["bias_decay"] = torch.tensor(bias_decay, device=device, dtype=dtype)
        return params, buffers

    @staticmethod
    def to_learned_dict(params, buffers):
        return TiedSAE(params["encoder"], params["encoder_bias"], norm_encoder=True)

    @staticmethod
    def learned_dict_stack(params, buffers):
        return params["encoder"], NORM_FLOOR, None

    @staticmethod
    def loss(params, buffers, batch):
        return engine_loss(FunctionalPositiveTiedSAE, params, buffers, batch)


def _mask_buffers(n_dict_components, n_components_stack, l1_alpha, bias_decay, device, dtype):
    mask = torch.ones(n_components_stack, device=device, dtype=torch.bool)
    mask[:n_dict_components] = False
    return {
        "l1_alpha": torch.tensor(l1_alpha, device=device, dtype=dtype),
        "bias_decay": torch.tensor(bias_decay, device=device, dtype=dtype),
        "dict_size": torch.tensor(n_dict_components, device=device, dtype=torch.long),
        "coef_mask": mask,
    }


class FunctionalMaskedTiedSAE(DictSignature):
    """Models with different dictionary sizes share one [M, n_stack, d] stack; coefficients beyond a model's
    ``dict_size`` are forced to zero (sae_ensemble.py:331-333, :356). The bias-decay term is not part of this
    signature's loss (:347-373)."""
    variant = "masked_tied"

    @staticmethod
    def init(activation_size, n_dict_components, n_components_stack, l1_alpha, bias_decay=0.0, device=None,
             dtype=None):
        params = {
            "encoder": _xavier(n_components_stack, activation_size, device, dtype),
            "encoder_bias": torch.zeros((n_components_stack,), device=device, dtype=dtype),
        }
        return params, _mask_buffers(n_dict_components, n_components_stack, l1_alpha, bias_decay, device, dtype)

    @staticmethod
    def to_learned_dict(params, buffers):
        k = buffers["dict_size"].item()
        return TiedSAE(params["encoder"][:k], params["encoder_bias"][:k], norm_encoder=True)

    @staticmethod
    def learned_dict_stack(params, buffers):
        return params["encoder"], NORM_FLOOR, buffers["dict_size"]

    @staticmethod
    def loss(params, buffers, batch):
        return engine_loss(FunctionalMaskedTiedSAE, params, buffers, batch)


class FunctionalMaskedSAE(DictSignature):
    """Untied counterpart (sae_ensemble.py:377-444)."""
    variant = "masked_untied"

    @staticmethod
    def init(activation_size, n_dict_components, n_components_stack, l1_alpha, bias_decay=0.0, device=None,
             dtype=None):
        params = {
            "encoder": _xavier(n_components_stack, activation_size, device, dtype),
            "encoder_bias": torch.zeros((n_components_stack,), device=device, dtype=dtype),
            "decoder": _xavier(n_components_stack, activation_size, device, dtype),
        }
        return params, _mask_buffers(n_dict_components, n_components_stack, l1_alpha, bias_decay, device, dtype)

    @staticmethod
    def to_learned_dict(params, buffers):
        k = buffers["dict_size"].item()
        return UntiedSAE(params["encoder"][:k], params["decoder"][:k], params["encoder_bias"][:k])

    @staticmethod
    def learned_dict_stack(params, buffers):
        return params["decoder"], NORM_FLOOR, buffers["dict_size"]

    @staticmethod
    def loss(params, buffers, batch):
        return engine_loss(FunctionalMaskedSAE, params, buffers, batch)


for _cls in (FunctionalSAE, FunctionalTiedSAE, FunctionalTiedCenteredSAE, FunctionalMaskedTiedSAE, FunctionalMaskedSAE):
    _cls.__module__ = _REF_MODULE
FunctionalPositiveTiedSAE.__module__ = "autoencoders.mlp_tests"
