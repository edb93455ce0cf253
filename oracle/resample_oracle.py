"""fp64 oracle of dead-feature resampling (FunctionalEnsemble.track_dead_features / resample_dead_features; the
reference's process_reinit, experiments/huge_batch_size.py:120-254).

*** TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT PATH. *** (as oracle/sae_oracle.py, whose forward pieces it uses)

Per model, over a window of steps:
  * ``forward64``: the code and the row errors e_r = mean over d of (x_hat - x)^2 of one batch, in the space the
    signature reconstructs (FunctionalTiedSAE's centred batch, x - center, x + 0.18), in fp64;
  * ``Window``: the N rows with the largest e by (e descending, window serial ascending) with a copy of each row as
    it was fed (the reference's ``WorstIndices(n_features)`` fed ``mse_losses``, :120-146, :209-210), and each
    feature's active rows (``c_totals``, :206);
  * ``resample``: dead features (count 0, masked padding excluded) j_1 < j_2 < ... take the sorted rows v_1, v_2, ...
    scaled by ratio / mu, mu the mean row norm of the valid features before the change (:224-240, SURVEY.md Q11).
    The Adam moments of the replaced rows are zeroed (:242-250); the oracle reports which rows those are.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from .positive_tied_oracle import SHIFT
from .sae_oracle import center, tied_forward, topk_forward, untied_forward

Tensor = torch.Tensor


def forward64(variant: str, params: Dict[str, Tensor], buffers: Dict[str, Tensor], x: Tensor):
    """(code [B, n], e [B]) of one model on the batch x [B, d] as the caller fed it, in fp64."""
    p = {k: v.double() for k, v in params.items()}
    b = {k: v.double() if v.is_floating_point() else v for k, v in buffers.items()}
    x = x.double()
    mask = buffers["coef_mask"].bool() if "coef_mask" in buffers else None
    if variant == "topk":
        f = topk_forward(p["dict"], x, int(buffers["sparsity"]))
        xin = x
    elif variant in ("untied", "masked_untied"):
        xin = x
        f = untied_forward(p["encoder"], p["encoder_bias"], p["decoder"], xin, b["l1_alpha"], coef_mask=mask)
    else:
        E = p["encoder"]
        if variant == "tied_learned_center":
            xin = x - p["center"][None, :]
        elif variant == "positive_tied":
            xin, E = x + SHIFT, E.clamp(min=0.0)
        elif "center_rot" in b:
            xin = center(x, b["center_trans"], b["center_rot"], b["center_scale"])
        else:
            xin = x
        f = tied_forward(E, p["encoder_bias"], xin, b["l1_alpha"], coef_mask=mask)
    return f["c"], (f["x_hat"] - xin).pow(2).mean(dim=-1)


class Window:
    """One model's window: the list of the ``n_worst`` worst rows and the features' active-row counts."""

    def __init__(self, n_worst: int, n: int, d: int):
        self.n_worst = n_worst
        self.err = torch.zeros(0, dtype=torch.float64)
        self.serial = torch.zeros(0, dtype=torch.int64)
        self.rows = torch.zeros(0, d, dtype=torch.float32)
        self.counts = torch.zeros(n, dtype=torch.int64)
        self.next_serial = 0

    def add(self, e: Tensor, rows: Tensor, code: Tensor) -> None:
        B = e.shape[0]
        serial = self.next_serial + torch.arange(B, dtype=torch.int64)
        err = torch.cat([self.err, e.double().cpu()])
        ser = torch.cat([self.serial, serial])
        rws = torch.cat([self.rows, rows.float().cpu()])
        order = sorted_order(err, ser)[: self.n_worst]
        self.err, self.serial, self.rows = err[order], ser[order], rws[order]
        self.counts += (code.cpu() > 0).sum(dim=0)
        self.next_serial += B


def sorted_order(err: Tensor, serial: Tensor) -> Tensor:
    """Indices sorting the entries by (err descending, serial ascending)."""
    order = torch.sort(serial, stable=True).indices
    return order[torch.sort(err[order], descending=True, stable=True).indices]


def dead_features(counts: Tensor, coef_mask: Optional[Tensor] = None) -> Tensor:
    """Ascending indices of the features with no active row, masked padding (coef_mask = 1) excluded."""
    dead = counts == 0
    if coef_mask is not None:
        dead &= ~coef_mask.bool().cpu()
    return torch.nonzero(dead).flatten()


def resample(W: Tensor, rows_sorted: Tensor, dead: Tensor, ratio: float = 0.2,
             coef_mask: Optional[Tensor] = None) -> Dict[str, Tensor]:
    """The dictionary parameter W [n, d] after the replacement (fp64), the replaced indices, mu and the scale."""
    W = W.double().cpu()
    valid = torch.ones(W.shape[0], dtype=torch.bool) if coef_mask is None else ~coef_mask.bool().cpu()
    mu = W[valid].norm(dim=-1).mean()
    k = min(dead.numel(), rows_sorted.shape[0])
    out = W.clone()
    out[dead[:k]] = rows_sorted[:k].double() * ratio / mu
    return {"W": out, "replaced": dead[:k], "mu": mu, "scale": ratio / mu}
