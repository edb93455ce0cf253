"""``DictSignature`` — the model protocol of the ensemble engine (reference: autoencoders/ensemble.py:15-22).

A signature is a namespace of static methods:
    init(...)                      -> (params: dict[str, Tensor], buffers: dict[str, Tensor])
    loss(params, buffers, batch)   -> (loss, (loss_data: dict[str, Tensor], aux: {"c": [B, n]}))
    to_learned_dict(params, buffers) -> LearnedDict
In the reference ``loss`` is a differentiable torch function that FunctionalEnsemble wraps in
``vmap(grad(...))``. Here the signatures the hot path covers carry a ``variant`` tag instead, and both
``FunctionalEnsemble.step_batch`` and a direct ``sig.loss(...)`` call execute in the CUDA engine (libsce.so).
"""
from __future__ import annotations

import torch


class DictSignature:
    variant = None  # engine-backed signatures: a key of _lib.SIGNATURES ("tied", "masked_tied", "untied", "masked_untied",
                    # "topk", "tied_learned_center", "positive_tied")

    @staticmethod
    def to_learned_dict(params, buffers):
        pass

    @staticmethod
    def loss(params, buffers, batch):
        pass

    @staticmethod
    def learned_dict_stack(params, buffers):
        """The stacked learned dictionaries of an ensemble as ``(matrix [M, n, d], norm_floor, rows)``: what
        ``to_learned_dict(...).get_learned_dict()`` returns per model is ``matrix[m, :rows[m]]`` with every row divided
        by ``max(||row||, norm_floor)`` (``norm_floor <= 0``: no clamp; ``None``: not normalised); ``rows`` is a [M]
        tensor, or None when every model uses all ``n`` rows. Read by ``metrics.dictionary_similarity``."""
        raise NotImplementedError("this signature does not describe its learned dictionary")


DictSignature.__module__ = "autoencoders.ensemble"


def engine_loss(sig, params, buffers, batch):
    """Single-model forward through the engine: what ``sig.loss(params, buffers, batch)`` returns in the
    reference — (loss, (loss_data, {"c": code})) — evaluated on the device of ``batch`` (must be CUDA)."""
    from .ensemble import FunctionalEnsemble  # local import: ensemble imports this module

    if not batch.is_cuda:
        raise RuntimeError(
            f"{sig.__name__}.loss runs in the sm_90a CUDA engine and needs CUDA tensors (got {batch.device}); "
            "there is no CPU implementation in the product path")
    dev = batch.device
    model = ({k: v.detach().to(dev) for k, v in params.items()}, {k: v.detach().to(dev) for k, v in buffers.items()})
    ens = FunctionalEnsemble([model], sig, "adam", {"lr": 0.0}, device=dev)
    loss_data, aux = ens.forward_batch(batch)
    loss_data = {k: v[0] for k, v in loss_data.items()}
    return loss_data["loss"], (loss_data, {"c": aux["c"].dense()[0]})
