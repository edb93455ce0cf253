"""CPU oracle for FunctionalPositiveTiedSAE (autoencoders/mlp_tests.py:68-125): a tied SAE whose dictionary is the
clamped encoder E+ = max(E, 0), trained on the shifted input x + 0.18, with bias decay.

*** TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT PATH. *** (as oracle/sae_oracle.py, on whose tied pieces it builds)

Two formulations, cross-checked in tests/test_positive_tied_cpu.py and pinned there to the reference's own results
(tests/golden/positive_tied.pt, oracle/make_positive_tied_golden.py):
  * ``positive_tied_grads``: closed form — the tied gradients on x+ with W built from E+, the encoder gradient taken
    with respect to E+ and applied to E unmasked (straight-through), the bias gradient with its decay term;
  * ``sig_loss_positive_tied``: the restated loss in DictSignature form, for ``sae_oracle.RefPortEnsemble``
    (``vmap(grad)`` + Adam, fp32 or fp64), with the same straight-through encoder gradient.
"""
from __future__ import annotations

from typing import Dict

import torch

from .sae_oracle import tied_forward, tied_grads

Tensor = torch.Tensor
SHIFT = 0.18   # mlp_tests.py:104 `batch + 0.18`, :110 `x_hat - 0.18`


def positive_tied_grads(E, b, X, alpha, bias_decay=0.0, active=None) -> Dict[str, Tensor]:
    """Forward and gradients of one model on batch X. ``grads["encoder"]`` is dL/dE+, which is what the reference's
    ``grad`` returns for params["encoder"] (its loss rebinds the key to the clamped tensor, mlp_tests.py:100): no
    [E >= 0] mask. ``active``: as in ``sae_oracle.tied_grads`` (pins the ReLU activity pattern of near-kink
    coefficients)."""
    return tied_grads(E.clamp(min=0.0), b, X + SHIFT, alpha, bias_decay, None, active)


def masked_encoder_grad(E, b, X, alpha, bias_decay=0.0) -> Tensor:
    """dL/dE through the clamp, [E > 0] dL/dE+: what a masked clamp would give. The reference does NOT compute this;
    tests use it to show that a fixture tells the two apart."""
    g = positive_tied_grads(E, b, X, alpha, bias_decay)["grads"]["encoder"]
    return g * (E > 0).to(g.dtype)


def sig_loss_positive_tied(params, buffers, batch):
    """FunctionalPositiveTiedSAE.loss restated: (loss, ({"loss", "l_reconstruction", "l_l1", "l_bias_decay"},
    {"c": code})). The encoder enters as E + (max(E, 0) - E).detach(): the value of E+, the gradient of E+ passed to E
    unmasked, as the reference's rebinding of params["encoder"] gives."""
    E = params["encoder"]
    Ep = E + (E.clamp(min=0.0) - E).detach()
    f = tied_forward(Ep, params["encoder_bias"], batch + SHIFT, buffers["l1_alpha"], buffers["bias_decay"])
    data = {"loss": f["loss"], "l_reconstruction": f["l_reconstruction"], "l_l1": f["l_l1"],
            "l_bias_decay": f["l_bias_decay"]}
    return f["loss"], (data, {"c": f["c"]})
