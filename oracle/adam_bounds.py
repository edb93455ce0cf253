"""Per-element bounds on one Adam step of the engine (adam_apply in sparse_coding_b200/csrc/sce_kernels.cuh) against fp64.

*** TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT PATH. *** (as oracle/sae_oracle.py)

The engine updates every parameter element with

    m' = b1 m + (1 - b1) g
    v' = b2 v + (1 - b2) g g
    p' = p - lr (m' / bc1) / (sqrt(v' / bc2 + eps_root) + eps),      bc1 = 1 - b1^t, bc2 = 1 - b2^t

in fp32, where g is the element's gradient (the one ``grads_batch`` reports), ``lr, b1, b2, eps, eps_root`` are the fp32
values of the plan's descriptor and bc1, bc2 are formed in fp64 and rounded once to fp32 (hyper_for in sce_plan.cu).
``reference`` is the same step in fp64 (sae_oracle.adam_update) on the fp32 inputs and hyper-parameters, with the step
number t the engine should use: 1 under ``adam_count_mode="frozen_t1"``, steps taken + 1 under "standard".

The bars, with u = 2^-24 (the unit roundoff of fp32), count the roundings of adam_apply to first order. Whether the
compiler contracts a product and a sum into an FMA only removes roundings, so every bar holds for either order.

  m'  1 - b1 is exact (Sterbenz: 1/2 <= b1 <= 1); b1 m and (1 - b1) g round once each and their sum once:
      |m'_32 - m'| <= 2 u (b1 |m| + (1 - b1) |g|) = C_M u S_m. The scale S_m takes absolute values, so the bar holds
      when m and g cancel.
  v'  ((1 - b2) g) g rounds twice, b2 v once, the sum once, all terms >= 0: |v'_32 - v'| <= 3 u (b2 v + (1 - b2) g^2).
  p'  m'/bc1: m' error C_M u S_m, bc1's own rounding u, the division u: (C_M + 2) u S_m / bc1.
      v'/bc2 carries (C_V + 2) u relatively; + eps_root one more, sqrt halves it and adds u: (C_V + 5)/2 u = 4 u;
      + eps: 5 u on the denominator den = sqrt(v'/bc2 + eps_root) + eps. The quotient r = (m'/bc1) / den adds u, so
      |r_32 - r| <= (C_M + 2 + 5 + 1) u R = 10 u R with R = (S_m / bc1) / den (R >= |r|; R = |r| unless m and g
      cancel). lr r rounds once more (11 u lr R) and p - lr r once (u |p'|):
      |p'_32 - p'| <= u |p'| + C_P u lr R, C_P = 11.
  Subnormals: a result below 2^-126 is rounded to a multiple of 2^-149, which no relative bar covers; each of the
  (at most four) roundings of m' and v' adds at most 2^-150, hence FLOOR = 2^-148 added to both bars. Through v' it
  moves den by at most sqrt(FLOOR / bc2), which adds lr R sqrt(FLOOR / bc2) / den to the p' bar (below 1e-22 lr R at
  eps = 1e-8; it matters only for eps = 0 and a vanishing v').

Second-order terms (products of two roundings, below 2^-20 of each first-order term) are covered by the factor
SECOND_ORDER. None of the bars is loosened beyond this count.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle.sae_oracle import adam_update

U = 2.0 ** -24
C_M, C_V, C_P = 2.0, 3.0, 11.0
FLOOR = 2.0 ** -148
SECOND_ORDER = 1.0 + 2.0 ** -20


def fp32(x) -> float:
    return float(np.float32(x))


def fp32_hyper(h) -> dict:
    """The fp32 values the descriptor carries for ``h`` (an AdamConfig, or anything with lr, b1, b2, eps, eps_root)."""
    return {k: fp32(getattr(h, k)) for k in ("lr", "b1", "b2", "eps", "eps_root")}


def step_number(count_mode: str, steps_taken: int) -> int:
    """The t of the bias correction of the next step: always 1 under frozen_t1, steps taken + 1 under standard."""
    return 1 if count_mode == "frozen_t1" else steps_taken + 1


def reference(p, g, m, v, t, hyper):
    """The fp64 step from the fp32 inputs (any shape; tensors on any device) and the bars of the three outputs.
    ``hyper``: as fp32_hyper takes it. Returns {"p", "m", "v"} (fp64) and {"bar_p", "bar_m", "bar_v"}."""
    h = fp32_hyper(hyper)
    lr, b1, b2, eps, eps_root = h["lr"], h["b1"], h["b2"], h["eps"], h["eps_root"]
    p, g, m, v = (x.double().clone() for x in (p, g, m, v))
    S_m = b1 * m.abs() + (1.0 - b1) * g.abs()
    S_v = b2 * v + (1.0 - b2) * g * g
    adam_update(p, g, m, v, t, lr=lr, b1=b1, b2=b2, eps=eps, eps_root=eps_root)
    bc1, bc2 = 1.0 - b1 ** t, 1.0 - b2 ** t
    den = (v / bc2 + eps_root).sqrt() + eps
    R = S_m / bc1 / den
    bar_p = U * p.abs() + C_P * U * lr * R + lr * R * (FLOOR / bc2) ** 0.5 / den
    return {"p": p, "m": m, "v": v,
            "bar_p": SECOND_ORDER * bar_p,
            "bar_m": SECOND_ORDER * (C_M * U * S_m + FLOOR),
            "bar_v": SECOND_ORDER * (C_V * U * S_v + FLOOR)}


def ratios(got, want, bar):
    """|got - want| / bar per element; a NaN (or an error where the bar is 0) is an infinite error."""
    err = (got.double() - want).abs()
    r = torch.where(bar > 0, err / bar.clamp(min=1e-300), torch.where(err == 0, 0.0, float("inf")).to(err))
    return torch.where(r.isnan(), torch.full_like(r, float("inf")), r)


def worst(got, want, bar) -> float:
    """The largest ratio of ``ratios`` (0 for an empty tensor)."""
    r = ratios(got, want, bar)
    return float(r.max()) if r.numel() else 0.0


def check_step(got, ref):
    """The largest ratio of each output: ``got`` {"p", "m", "v"} of the engine against ``reference``'s result."""
    return {k: worst(got[k], ref[k], ref["bar_" + k]) for k in ("p", "m", "v")}
