"""Top-k dictionaries: the training-side signature and the exported inference object.

Behavioural contract (reference ``autoencoders/topk_encoder.py``): the dictionary is initialised from a standard
normal on the CPU and carries a per-model integer ``sparsity`` buffer (:10-17); a code keeps, per input row, the
``k`` largest *signed* scores against the row-normalised dictionary and then applies a ReLU, so a row can end up
with fewer than ``k`` non-zeros (:19-27); the loss is the plain MSE of the reconstruction, without bias or L1 term
(:29-40); export wraps the normalised dictionary together with ``k`` (:43-62).

Training-time ``loss`` runs in the CUDA engine: scores on the tensor cores, a per-row selection that bounds the k-th
largest score and ranks the few candidates above it (``topk_select2_kernel``), then a gather decode over the k selected
rows or the tied SAE's dense decode, and the same backward / Adam pipeline. Unlike the reference,
which has to fall back to a Python loop over models because ``torch.topk`` with a data-dependent ``k`` cannot be
vmapped (``no_stacking=True``), models with different ``k`` are batched in one launch sequence.
"""
from __future__ import annotations

import torch

from .learned_dict import LearnedDict
from .signatures import DictSignature, engine_loss

_REF_MODULE = "autoencoders.topk_encoder"


def _unit_norm_rows(mat: torch.Tensor) -> torch.Tensor:
    # no clamp on the norm here, unlike the SAE variants
    return mat / mat.norm(dim=-1)[:, None]


def sparse_code_from_scores(scores: torch.Tensor, k: int) -> torch.Tensor:
    """Keep each row's k largest entries (by signed value), zero the rest, clip negatives."""
    k = int(k)
    top = torch.topk(scores, k, dim=-1)
    kept = torch.zeros_like(scores).scatter_(-1, top.indices, top.values)
    return kept.clamp_(min=0.0)


class TopKLearnedDict(LearnedDict):
    """Inference object stored in ``learned_dicts.pt`` for top-k runs: attributes ``dict`` (already normalised),
    ``sparsity``, ``n_feats``, ``activation_size``."""

    def __init__(self, dict, sparsity):
        self.dict = dict
        self.sparsity = sparsity
        self.n_feats, self.activation_size = dict.shape

    def get_learned_dict(self):
        return self.dict

    def encode(self, x):
        return sparse_code_from_scores(x @ self.dict.T, self.sparsity)

    def to_device(self, device):
        self.dict = self.dict.to(device)


class TopKEncoder(DictSignature):
    variant = "topk"

    @staticmethod
    def init(d_activation, n_features, sparsity, dtype=torch.float32):
        if not 0 < int(sparsity) <= n_features:
            raise ValueError(f"sparsity must be in [1, {n_features}], got {sparsity}")
        dictionary = torch.randn(n_features, d_activation, dtype=dtype)
        return {"dict": dictionary}, {"sparsity": torch.tensor(sparsity, dtype=torch.long)}

    @staticmethod
    def encode(b, sparsity, normed_dict):
        return sparse_code_from_scores(b @ normed_dict.T, sparsity)

    @staticmethod
    def loss(params, buffers, batch):
        return engine_loss(TopKEncoder, params, buffers, batch)

    @staticmethod
    def to_learned_dict(params, buffers):
        return TopKLearnedDict(_unit_norm_rows(params["dict"]), buffers["sparsity"].item())

    @staticmethod
    def learned_dict_stack(params, buffers):
        return params["dict"], 0.0, None   # unit rows without a clamp (_unit_norm_rows)


for _cls in (TopKEncoder, TopKLearnedDict):
    _cls.__module__ = _REF_MODULE
