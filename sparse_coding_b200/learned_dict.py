"""Inference-side dictionary objects — the checkpoint schema of the sweep (``learned_dicts.pt``).

Mirrors the public surface of the reference's ``autoencoders/learned_dict.py`` (LearnedDict :16-53, UntiedSAE
:129-149, TiedSAE :152-215): attribute names, method names and arithmetic are the contract every consumer of a
checkpoint relies on (``.encode``, ``.predict``, ``.get_learned_dict``, ``.to_device``, ``.n_feats``,
``.activation_size``, ``.encoder``, ``.encoder_bias``, ``.decoder``, ``.center_*``, ``.norm_encoder``).

Instances pickle under the reference's qualified names (``autoencoders.learned_dict.TiedSAE`` …) so that files
written by this engine load inside the reference repo and vice versa; the top-level ``autoencoders`` shim package
makes those names resolve here. These objects are plain tensor containers: they are produced at the end of a chunk
and used for analysis, they are not on the training hot path.
"""
from __future__ import annotations

from abc import ABC, abstractmethod

import torch

NORM_FLOOR = 1e-8

_REF_MODULE = "autoencoders.learned_dict"


def _unit_rows(mat: torch.Tensor) -> torch.Tensor:
    return mat / mat.norm(dim=-1).clamp(min=NORM_FLOOR)[:, None]


class LearnedDict(ABC):
    """learned_dict.py:16-53."""
    n_feats: int
    activation_size: int

    @abstractmethod
    def get_learned_dict(self) -> torch.Tensor:
        ...

    @abstractmethod
    def encode(self, batch: torch.Tensor) -> torch.Tensor:
        ...

    @abstractmethod
    def to_device(self, device) -> None:
        ...

    def decode(self, code: torch.Tensor) -> torch.Tensor:
        return code @ self.get_learned_dict()

    def center(self, batch: torch.Tensor) -> torch.Tensor:
        return batch

    def uncenter(self, batch: torch.Tensor) -> torch.Tensor:
        return batch

    def predict(self, batch: torch.Tensor) -> torch.Tensor:
        return self.uncenter(self.decode(self.encode(self.center(batch))))

    def n_dict_components(self) -> int:
        return self.get_learned_dict().shape[0]


class UntiedSAE(LearnedDict):
    """learned_dict.py:129-149: separate encoder and (row-normalised) decoder."""

    def __init__(self, encoder, decoder, encoder_bias):
        self.encoder = encoder
        self.decoder = decoder
        self.encoder_bias = encoder_bias
        self.n_feats, self.activation_size = self.encoder.shape

    def get_learned_dict(self):
        return _unit_rows(self.decoder)

    def to_device(self, device):
        self.encoder = self.encoder.to(device)
        self.decoder = self.decoder.to(device)
        self.encoder_bias = self.encoder_bias.to(device)

    def encode(self, batch):
        return (batch @ self.encoder.T + self.encoder_bias).clamp(min=0.0)


class TiedSAE(LearnedDict):
    """learned_dict.py:152-215: one matrix, normalised on the fly when ``norm_encoder``; optional affine centring
    ``center(x) = ((x - trans) @ rot^T) * scale``."""

    def __init__(self, encoder, encoder_bias, centering=(None, None, None), norm_encoder=True):
        self.encoder = encoder
        self.encoder_bias = encoder_bias
        self.norm_encoder = norm_encoder
        self.n_feats, self.activation_size = self.encoder.shape
        trans, rot, scale = centering
        dev = self.encoder.device
        self.center_trans = torch.zeros(self.activation_size, device=dev) if trans is None else trans
        self.center_rot = torch.eye(self.activation_size, device=dev) if rot is None else rot
        self.center_scale = torch.ones(self.activation_size, device=dev) if scale is None else scale

    def initialize_missing(self):
        """Checkpoints written before centring existed lack the three attributes (learned_dict.py:176-184)."""
        dev = self.encoder.device
        if not hasattr(self, "center_trans"):
            self.center_trans = torch.zeros(self.activation_size, device=dev)
        if not hasattr(self, "center_rot"):
            self.center_rot = torch.eye(self.activation_size, device=dev)
        if not hasattr(self, "center_scale"):
            self.center_scale = torch.ones(self.activation_size, device=dev)

    def center(self, batch):
        return ((batch - self.center_trans[None, :]) @ self.center_rot.T) * self.center_scale[None, :]

    def uncenter(self, batch):
        return (batch / self.center_scale[None, :]) @ self.center_rot + self.center_trans[None, :]

    def get_learned_dict(self):
        return _unit_rows(self.encoder)

    def to_device(self, device):
        self.initialize_missing()
        for name in ("encoder", "encoder_bias", "center_trans", "center_rot", "center_scale"):
            setattr(self, name, getattr(self, name).to(device))

    def encode(self, batch):
        enc = _unit_rows(self.encoder) if self.norm_encoder else self.encoder
        return (batch @ enc.T + self.encoder_bias).clamp(min=0.0)


class IdentityReLU(LearnedDict):
    """learned_dict.py:86-104: the activations themselves as the code, ``relu(x + bias)``, with the identity as the
    dictionary. Keeps the reference's quirks: ``if bias:`` raises for a bias of more than one element (so only the
    default zero bias can be given), and ``get_learned_dict`` returns a CPU identity."""

    def __init__(self, activation_size, bias=None):
        self.n_feats = activation_size
        self.activation_size = activation_size
        if bias:
            self.bias = bias
        else:
            self.bias = torch.zeros(activation_size)
        assert self.bias.shape == (activation_size,)

    def get_learned_dict(self):
        return torch.eye(self.n_feats)

    def encode(self, batch):
        return torch.clamp(batch + self.bias, min=0.0)

    def to_device(self, device):
        self.bias = self.bias.to(device)


class RandomDict(LearnedDict):
    """learned_dict.py:107-127: a Gaussian matrix drawn with ``torch.randn`` from the global RNG at construction, used
    as the encoder, ``relu(x E^T + b)``, and as the dictionary, with its rows as drawn (not normalised)."""

    def __init__(self, activation_size, n_feats=None):
        if not n_feats:
            n_feats = activation_size
        self.n_feats = n_feats
        self.activation_size = activation_size
        self.encoder = torch.randn(n_feats, activation_size)
        self.encoder_bias = torch.zeros(n_feats)

    def get_learned_dict(self):
        return self.encoder

    def encode(self, batch):
        c = torch.einsum("nd,bd->bn", self.encoder, batch)
        c = c + self.encoder_bias
        return torch.clamp(c, min=0.0)

    def to_device(self, device):
        self.encoder = self.encoder.to(device)
        self.encoder_bias = self.encoder_bias.to(device)


class Rotation(LearnedDict):
    """learned_dict.py:277-293: a fixed matrix whose rows are the dictionary; the code is linear, ``batch @ matrix^T``.
    ``activation_size`` is the matrix's row count, as in the reference. The matrix is moved to ``device`` (the CPU by
    default) on construction."""

    def __init__(self, matrix, device=None):
        self.device = "cpu" if device is None else device
        self.matrix = matrix.to(self.device)
        self.activation_size = matrix.shape[0]

    def get_learned_dict(self):
        return self.matrix

    def to_device(self, device):
        self.device = device
        self.matrix = self.matrix.to(device)

    def encode(self, batch):
        return batch @ self.matrix.T


for _cls in (LearnedDict, UntiedSAE, TiedSAE, IdentityReLU, RandomDict, Rotation):
    _cls.__module__ = _REF_MODULE
