"""CPU oracle for FunctionalTiedCenteredSAE (autoencoders/sae_ensemble.py:164-230): a tied SAE on x - center, the centre
a trained parameter, no bias decay.

*** TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT PATH. *** (as oracle/sae_oracle.py, on whose tied pieces it builds)

Two formulations, cross-checked in tests/test_learned_center_cpu.py and pinned there to the reference's own results
(tests/golden/tied_learned_center.pt, oracle/make_learned_center_golden.py):
  * ``tied_center_grads``: closed form — the tied gradients on x_c = x - center plus d_center = sum_b g_b - db W;
  * ``sig_loss_tied_learned_center``: the restated loss in DictSignature form, for ``sae_oracle.RefPortEnsemble``
    (``vmap(grad)`` + Adam, fp32 or fp64), which trains the centre like every other parameter.
"""
from __future__ import annotations

from typing import Dict

import torch

from .sae_oracle import tied_forward, tied_grads

Tensor = torch.Tensor


def tied_center_grads(E, b, center, X, alpha, active=None) -> Dict[str, Tensor]:
    """Forward and gradients of one model on batch X: the tied gradients on x_c = x - center (no bias decay), plus the
    centre's d_center = sum_b g_b - db W, g = dL/dx_hat. ``active``: as in ``sae_oracle.tied_grads`` (pins the ReLU
    activity pattern of near-kink coefficients)."""
    f = tied_grads(E, b, X - center[None, :], alpha, 0.0, None, active)
    f["grads"]["center"] = f["G"].sum(0) - f["grads"]["encoder_bias"] @ f["W"]
    f["loss"] = f["l_reconstruction"] + f["l_l1"]
    return f


def sig_loss_tied_learned_center(params, buffers, batch):
    """FunctionalTiedCenteredSAE.loss restated: (loss, ({"loss", "l_reconstruction", "l_l1"}, {"c": code}))."""
    f = tied_forward(params["encoder"], params["encoder_bias"], batch - params["center"][None, :], buffers["l1_alpha"])
    l = f["l_reconstruction"] + f["l_l1"]
    return l, ({"loss": l, "l_reconstruction": f["l_reconstruction"], "l_l1": f["l_l1"]}, {"c": f["c"]})
