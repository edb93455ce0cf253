"""Per-tile error bounds of the engine's training-step outputs against fp64.

*** TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT PATH. *** (as oracle/sae_oracle.py)

Every GEMM of the step writes its output in 128 x 128 tiles per model, and each fused epilogue works on one tile. A
defect there (the partial last row or column tile, the K tail, one model's slab, one operand set of the weight gradient,
the second tile a persistent CTA runs) usually touches part of one output: one norm-relative number per model dilutes
an error confined to one of T equal tiles by about 1/sqrt(T). So the error is measured per (model, tile), as

    ratio = ||got - want||_tile / ||S||_tile

where S is the absolute-product scale of the output: the same fp64 formula with every operand replaced by its absolute
value. It is the size the rounding of a split-operand product can reach, whatever the cancellation in the product
itself, so one bar serves every tile whether its values are large or cancel to almost nothing. The per-element
maximum of |got - want| / S is reported beside it.

The scales carry the absolute values through the whole chain from the step's inputs, so that a quantity that is itself
a cancelling sum is replaced by its own scale, not by its (possibly tiny) value: the pre-activation gradient
dz = (g W_d^T + alpha / B) [active] enters as its scale (|g| |W_d|^T + alpha / B) [active], and a centred batch
x_c = ((x - t) R^T) s as (|x - t| |R|^T) |s|. Measured on an H100: with |dz| in their place, single coefficients whose
reconstruction and L1 terms cancel (and the rotation's cancellation) put element ratios of a correct 3-pass gradient at
up to 1e-2. For a batch x (as the signature's loss sees it, or its scale), encoder W_e (unit rows where tied), decoder
W_d (unit rows), bias b, code c, reconstruction gradient g:
    code              S = |x| |W_e|^T + |b|              (relu is 1-Lipschitz: the error of c is at most that of z)
    x_hat             S = (|x| |W_e|^T + |b|) |W_d|
    dz                S_dz = (|g| |W_d|^T + alpha / B) [active]
    weight gradient   S = S_dz^T |x| + |c|^T |g|         (untied: the encoder has the first term, the decoder the second)
                      through the row-norm Jacobian (dW - w <w, dW>) / s:  |S| / s + |w| (|w| . |S|) / s
    bias gradient     S_db = sum_b S_dz  (+ |bias-decay term|)
    centre gradient   S = sum_b |g| + S_db |W|
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch

Tensor = torch.Tensor
TILE = 128


def code_scale(X: Tensor, W_enc: Tensor, b: Tensor) -> Tensor:
    return X.abs() @ W_enc.abs().T + b.abs()


def centered_input_scale(X: Tensor, trans: Tensor, rot: Tensor, scale: Tensor) -> Tensor:
    """Scale of FunctionalTiedSAE's centred batch ((x - t) R^T) s: (|x - t| |R|^T) |s|."""
    return ((X - trans[None, :]).abs() @ rot.abs().T) * scale.abs()[None, :]


def x_hat_scale(X: Tensor, W_enc: Tensor, b: Tensor, W_dec: Tensor) -> Tensor:
    return code_scale(X, W_enc, b) @ W_dec.abs()


def pre_activation_grad_scale(G: Tensor, W_dec: Tensor, alpha_over_B: float, gate: Tensor) -> Tensor:
    """Scale of dz = (g W_d^T + alpha / B [active]) [gate]: (|g| |W_d|^T + alpha / B) [gate] ([B, n])."""
    return (G.abs() @ W_dec.abs().T + abs(alpha_over_B)) * gate.to(G.dtype)


def weight_grad_scale(dZ: Optional[Tensor], X: Optional[Tensor], C: Optional[Tensor] = None,
                      G: Optional[Tensor] = None) -> Tensor:
    """|dz|^T |x| + |c|^T |g| ([n, d]); either operand set may be absent (None). Pass scales for operands that are
    themselves cancelling sums (S_dz for dz)."""
    S = dZ.abs().T @ X.abs() if dZ is not None else 0.0
    if C is not None:
        S = S + C.abs().T @ G.abs()
    return S


def row_norm_jacobian_scale(W: Tensor, s: Tensor, S: Tensor) -> Tensor:
    """The scale S of dW carried through d/dE of W = E / s: |S| / s + |w| (|w| . |S|) / s, row by row."""
    Wa, Sa = W.abs(), S.abs()
    return (Sa + Wa * (Wa * Sa).sum(-1, keepdim=True)) / s[:, None]


def bias_grad_scale(dZ: Tensor, decay_term: Optional[Tensor] = None) -> Tensor:
    S = dZ.abs().sum(0)
    return S + decay_term.abs() if decay_term is not None else S


def center_grad_scale(G: Tensor, db: Tensor, W: Tensor) -> Tensor:
    return G.abs().sum(0) + db.abs() @ W.abs()


def _grid(t: Tensor, tile: Tuple[int, int]) -> Tensor:
    """[M, R, C] -> [M, Tr, tr, Tc, tc], zero-padded up to whole tiles (the ragged last tiles keep their own elements)."""
    M, R, Cc = t.shape
    tr, tc = tile
    Tr, Tc = -(-R // tr), -(-Cc // tc)
    t = torch.nn.functional.pad(t, (0, Tc * tc - Cc, 0, Tr * tr - R))
    return t.reshape(M, Tr, tr, Tc, tc)


def tile_ratios(got: Tensor, want: Tensor, scale: Tensor, tile: Tuple[int, int] = (TILE, TILE)) -> Dict[str, object]:
    """Per-(model, tile) ratios ||got - want|| / ||S|| over the tile grid of an output, ragged edge tiles included.

    ``got``, ``want``, ``scale``: [M, R, C] (models, rows, columns), [R, C] (one model) or [L] (a vector, tiled in
    runs of ``tile[1]``). Computed in fp64 on ``want``'s device. Returns
      ratio   [M, Tr, Tc]  the per-tile ratios
      peak    [M, Tr, Tc]  the per-tile maxima of |got - want| / S (inf where S = 0 and got != want)
      worst   (ratio, (model, tile row, tile column)) of the largest ratio
      elem    the largest |got - want| / S over all elements"""
    want = want.double()
    got = got.to(want.device).double()
    scale = scale.to(want.device).double()
    if want.dim() == 1:
        got, want, scale = (t.reshape(1, 1, -1) for t in (got, want, scale))
        tile = (1, tile[1])
    elif want.dim() == 2:
        got, want, scale = (t.unsqueeze(0) for t in (got, want, scale))
    if not (got.shape == want.shape == scale.shape):
        raise ValueError(f"shapes differ: got {tuple(got.shape)}, want {tuple(want.shape)}, scale {tuple(scale.shape)}")
    err = (got - want).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, float("inf")), err)
    e, s = _grid(err, tile), _grid(scale.abs(), tile)
    num = e.pow(2).sum(dim=(2, 4)).sqrt()
    den = s.pow(2).sum(dim=(2, 4)).sqrt()
    ratio = torch.where(num == 0, torch.zeros_like(num), num / den)
    rel = torch.where(e == 0, torch.zeros_like(e), e / s)
    peak = rel.amax(dim=(2, 4))
    flat = int(ratio.argmax())
    Tr, Tc = ratio.shape[1:]
    where = (flat // (Tr * Tc), (flat // Tc) % Tr, flat % Tc)
    return {"ratio": ratio, "peak": peak, "worst": (float(ratio.max()), where), "elem": float(peak.max())}
