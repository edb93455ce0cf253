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


def kink_window(Z: Tensor) -> float:
    """Width of the band around a kink of the step (a ReLU's 0, a top-k's k-th score) inside which an engine and the
    fp64 oracle may decide differently: 1e-4 of the RMS pre-activation, at least 1e-5."""
    return max(1e-5, 1e-4 * float(Z.double().pow(2).mean().sqrt()))


class Worst:
    """The worst tile and element of each output over the models of one check."""

    def __init__(self):
        self.tile, self.elem, self.minimum = {}, {}, {}

    def add(self, name, m, r):
        ratio, (_, tr, tc) = r["worst"]
        if ratio >= self.tile.get(name, (-1.0,))[0]:
            self.tile[name] = (ratio, (m, tr, tc))
        self.elem[name] = max(self.elem.get(name, 0.0), r["elem"])
        lo = float(r["ratio"].min()), float(r["peak"].min())
        old = self.minimum.get(name, (float("inf"), float("inf")))
        self.minimum[name] = (min(old[0], lo[0]), min(old[1], lo[1]))

    def add_scalar(self, name, m, v):
        v = float("inf") if v != v else v          # a NaN is an infinite error, never dropped by the comparisons
        if v >= self.tile.get(name, (-1.0,))[0]:
            self.tile[name] = (v, (m,))
        self.elem[name] = max(self.elem.get(name, 0.0), v)
        self.minimum[name] = (min(self.minimum.get(name, (float("inf"),))[0], v),) * 2


def engine_activity(code, counts, near, Z):
    """[c > 0] as the engine gates the backward pass. The dense code is read back from the operand planes, where an f16f8
    code below about 4e-9 (under the fp16 plane's subnormals and the scaled residual's) reads as 0 although the engine's
    activity mask, the sign of its fp32 z, has it active: then the feature's mask count (``active_counts``) exceeds its
    count of non-zero codes. Those coefficients lie inside the kink window with a zero code; each such feature gets as
    many of them, the largest z first, back on the active side. A wrong pick could only fail the gradient check."""
    pos = code > 0
    missing = counts.long() - pos.sum(0)
    assert int(missing.min()) >= 0, int(missing.min())
    for j in torch.nonzero(missing).flatten().tolist():
        cand = near[:, j] & ~pos[:, j]
        k = int(missing[j])
        assert int(cand.sum()) >= k, (j, k, int(cand.sum()))
        zc = torch.where(cand, Z[:, j], torch.full_like(Z[:, j], -float("inf")))
        pos[torch.topk(zc, k).indices, j] = True
    return pos


# (tile ratio bar, element bar) of the dense variants' outputs per arithmetic, dictionary sign and output ("loss": one
# relative error per loss term), set from measurement in tests/test_tile_bounds_gpu.py (see its docstring).
# FunctionalPositiveTiedSAE ("nonneg") has its own: every product of its encode and decode has one sign, so the fp32
# accumulation of the tensor cores, not the operand split, sets its 3-pass error.
BARS = {
    "bf16x3": {
        "signed": {"code": (6.5e-7, 6.3e-6), "x_hat": (5.8e-8, 3.2e-7), "loss": (6.3e-5, 6.3e-5),
                   "encoder": (1.1e-5, 1.9e-4), "decoder": (6.5e-6, 2.6e-5), "encoder_bias": (5.3e-6, 5.6e-5),
                   "center": (7.6e-8, 2.1e-7)},
        "nonneg": {"code": (3.6e-6, 1.2e-5), "x_hat": (5.5e-6, 8.2e-6), "loss": (2.3e-5, 2.3e-5),
                   "encoder": (2.7e-5, 9.2e-5), "encoder_bias": (1.5e-5, 1.6e-5)},
    },
    "f16f8": {
        "signed": {"code": (2.8e-6, 2.5e-5), "x_hat": (1.6e-7, 8.8e-7), "loss": (1.7e-4, 1.7e-4),
                   "encoder": (1.4e-5, 3.8e-4), "decoder": (7.0e-5, 2.5e-4), "encoder_bias": (1.6e-5, 1.1e-4),
                   "center": (1.2e-7, 3.7e-7)},
        "nonneg": {"code": (1.7e-5, 5.2e-5), "x_hat": (1.7e-5, 2.5e-5), "loss": (6.9e-5, 6.9e-5),
                   "encoder": (5.4e-5, 1.7e-4), "encoder_bias": (3.9e-5, 4.3e-5)},
    },
}
# outputs whose tile bar sits at most half the smallest 1-pass tile ratio: the single-pass runs must clear it, and only
# these get a negative-control claim (the others are listed in tests/test_tile_bounds_gpu.py's docstring)
SEPARATED = {"bf16x3": {"signed": ("code", "x_hat", "decoder", "encoder_bias", "center"),
                        "nonneg": ("code", "x_hat", "encoder_bias")},
             "f16f8": {"signed": ("code", "x_hat"), "nonneg": ()}}


# ----------------------------------------------------------------------------------------------------------------------
# top-k (TopKEncoder): code c = relu(z) on the selected support, x_hat = c W, dict gradient through the row norm
# ----------------------------------------------------------------------------------------------------------------------
def topk_scales(X: Tensor, W: Tensor, s: Tensor, C: Tensor, G: Tensor, support: Tensor) -> Dict[str, Tensor]:
    """Scales of TopKEncoder's outputs for scores z = x W^T against the unit rows W (norms s) on ``support`` (bool
    [B, n], selected and positive), from the formulas above with no bias and no L1 term: the code's scale on the support
    (0 elsewhere, where code and oracle are both 0), x_hat's as that scale times |W|, and the dict gradient's from
    S_dz = |g| |W|^T on the support, through the row-norm Jacobian."""
    on = support.to(X.dtype)
    S_code = code_scale(X, W, torch.zeros(W.shape[0], dtype=X.dtype, device=X.device)) * on
    S_dz = pre_activation_grad_scale(G, W, 0.0, support)
    return {"code": S_code, "x_hat": S_code @ W.abs(),
            "dict": row_norm_jacobian_scale(W, s, weight_grad_scale(S_dz, X, C, G))}


def topk_support_check(Z: Tensor, support: Tensor, k: int, window: float) -> Dict[str, int]:
    """Whether ``support`` (bool [B, n]) is, row by row, the positive part of a top-k of the fp64 scores ``Z`` up to
    ``window``. Returns counts (rows, or entries for ``outside``):
      over_k     rows keeping more than k
      misranked  rows that keep a score below -window, or drop one above (k-th kept score, or 0 where fewer than k are
                 kept) + window
      differ     rows whose support is not Z's own (its k largest scores, the positive ones)
      outside    entries where the two differ farther than window from the row's boundary, max(k-th score, 0)"""
    inf = torch.full_like(Z, float("inf"))
    kept = support.sum(-1)
    kept_min = torch.where(support, Z, inf).amin(-1)
    dropped_max = torch.where(support, -inf, Z).amax(-1)
    thr = torch.where(kept >= k, kept_min, torch.zeros_like(kept_min))
    misranked = (kept_min < -window) | (dropped_max > thr + window)
    top = torch.topk(Z, k, dim=-1)
    own = torch.zeros_like(support).scatter_(-1, top.indices, True) & (Z > 0)
    diff = own != support
    boundary = top.values[:, -1:].clamp(min=0.0)
    return {"over_k": int((kept > k).sum()), "misranked": int(misranked.sum()), "differ": int(diff.any(-1).sum()),
            "outside": int((diff & ((Z - boundary).abs() > window)).sum())}


# (tile ratio bar, element bar) of TopKEncoder's outputs per arithmetic ("loss": one relative error per model), and the
# outputs whose bar separates 3-pass from 1-pass tiles: set from measurement in tests/test_topk_tile_bounds_gpu.py (see
# its docstring); tests/test_tile_bounds_cpu.py shows that they reject planted top-k defects
TOPK_BARS = {
    "bf16x3": {"code": (4.3e-6, 7.8e-6), "x_hat": (6.6e-7, 5.1e-6), "dict": (8.7e-7, 4.2e-5), "loss": (6.1e-6, 6.1e-6)},
    "f16f8": {"code": (1.6e-5, 3.2e-5), "x_hat": (2.8e-6, 1.9e-5), "dict": (3.9e-6, 2.1e-4), "loss": (2.6e-6, 2.6e-6)},
}
TOPK_SEPARATED = {"bf16x3": ("code", "x_hat", "dict"), "f16f8": ("x_hat",)}
