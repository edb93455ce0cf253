"""fp64 restatement of the correlation of two dictionaries' codes over paired rows (inter_dict_connections.ipynb's
covariance cell, as its text intends: the population Pearson correlation; SURVEY Q16), and the error bounds of the
engine's cross sums.

*** TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT PATH. *** (as oracle/sae_oracle.py)

Cross sums. The engine forms S_ab = sum_r c_a,r c_b,r on the split-operand GEMM over slices of at most 2048 rows, each
slice accumulated in fp32 on the tensor cores and the slices added in fp64. Against the fp64 sum of the codes the
engine holds (its operand planes, read back with sce_read_code), each entry is bounded by

    |dS_ab| <= kappa_arith * sum_r |c_a,r| |c_b,r|

kappa covers the partial products the split drops (bf16x3: lo lo, 2^-16 relative; f16f8: the E5M2 cross terms, ~2^-13)
and the fp32 accumulation of a slice (the row passes' Gram bars for the same GEMM and slice length, 4.0e-5 / 2.6e-4,
tests/test_row_pass_tiles_gpu.py), with a factor of two to spare. Against codes c + e that differ from the engine's by
e (the reference's own fp32 codes; |e| <= bar * S per entry with the code scale S of oracle/tile_bounds.py), the
propagated term sum_r |e_a,r| |c_b,r| + |c_a,r| |e_b,r| + |e_a,r| |e_b,r| is added.

Correlation. With cov = S_ab / N - mu_a mu_b and the variances exact to their own (much smaller) bounds, an error dS
moves the correlation by |dS| / (N sigma_a sigma_b). By Cauchy-Schwarz sum_r |c_a||c_b| <= sqrt(sum c_a^2 sum c_b^2),
so the bound is at most kappa sqrt((sigma_a^2 + mu_a^2)(sigma_b^2 + mu_b^2)) / (sigma_a sigma_b): small in absolute
terms whatever the sign of the codes, unless a feature's mean is far above its spread."""
from __future__ import annotations

from typing import Dict

import torch

Tensor = torch.Tensor

KAPPA = {"bf16x3": 1.0e-4, "f16f8": 5.0e-4}


def moments(c: Tensor):
    """(mean, var) [n] of the code c [N, n] in fp64, population form."""
    c = c.double()
    mean = c.mean(0)
    return mean, (c * c).mean(0) - mean * mean


def best(corr: Tensor, dim: int):
    """(maximum, index) of ``corr`` along ``dim``, skipping NaN, equal values to the lower index; (NaN, -1) where no
    entry is defined."""
    c = corr.transpose(0, 1) if dim == 0 else corr
    filled = torch.where(torch.isnan(c), torch.full_like(c, float("-inf")), c)
    mx = filled.max(1).values
    hit = (filled == mx[:, None]) & ~torch.isnan(c)
    idx = torch.where(hit, torch.arange(c.shape[1])[None, :].expand_as(c), torch.full_like(c, c.shape[1], dtype=torch.long))
    arg = idx.min(1).values
    none = torch.isnan(c).all(1)
    return torch.where(none, torch.full_like(mx, float("nan")), mx), torch.where(none, torch.full_like(arg, -1), arg)


def cross_sums(ca: Tensor, cb: Tensor, rows: int = 64) -> Tensor:
    """sum_r ca[r, p] cb[r, q] in fp64, in the same order for every entry (a blocked matrix product is not), so that
    equal code columns give bitwise equal sums: an exact tie stays one."""
    ca, cb = ca.double(), cb.double()
    out = torch.zeros(ca.shape[1], cb.shape[1], dtype=torch.float64)
    for r in range(0, ca.shape[0], rows):
        out += (ca[r:r + rows, :, None] * cb[r:r + rows, None, :]).sum(0)
    return out


def correlation(ca: Tensor, cb: Tensor) -> Dict[str, Tensor]:
    """Every output of metrics.code_correlation for the codes ca [N, n_a] and cb [N, n_b], in fp64."""
    ca, cb = ca.double(), cb.double()
    N = ca.shape[0]
    ma, va = moments(ca)
    mb, vb = moments(cb)
    cov = cross_sums(ca, cb) / N - ma[:, None] * mb[None, :]
    ok = (va > 0)[:, None] & (vb > 0)[None, :]
    corr = torch.where(ok, cov / torch.sqrt((va[:, None] * vb[None, :]).clamp(min=0)), torch.full_like(cov, float("nan")))
    mx_ab, ag_ab = best(corr, 1)
    mx_ba, ag_ba = best(corr, 0)
    return {"mean_a": ma, "var_a": va, "mean_b": mb, "var_b": vb, "covariance": cov, "correlation": corr,
            "max_corr_ab": mx_ab, "argmax_ab": ag_ab, "max_corr_ba": mx_ba, "argmax_ba": ag_ba, "rows": N}


def cross_sum_bound(ca: Tensor, cb: Tensor, arith: str, ea: Tensor = None, eb: Tensor = None) -> Tensor:
    """[n_a, n_b] bound on |engine S_ab - fp64 sum_r ca cb|; ``ea`` / ``eb``: per-entry bounds on how far the codes the
    engine holds are from ``ca`` / ``cb`` (None: they are those codes)."""
    A, Bb = ca.double().abs(), cb.double().abs()
    bound = KAPPA[arith] * (A.T @ Bb)
    if ea is not None or eb is not None:
        Ea = ea.double().abs() if ea is not None else torch.zeros_like(A)
        Eb = eb.double().abs() if eb is not None else torch.zeros_like(Bb)
        bound = bound + Ea.T @ Bb + A.T @ Eb + Ea.T @ Eb
    return bound


def correlation_bound(ca: Tensor, cb: Tensor, sum_bound: Tensor) -> Tensor:
    """[n_a, n_b] bound on the correlation error that a cross-sum error ``sum_bound`` leaves (variances exact)."""
    _, va = moments(ca)
    _, vb = moments(cb)
    return sum_bound / (ca.shape[0] * torch.sqrt((va[:, None] * vb[None, :]).clamp(min=1e-300)))
