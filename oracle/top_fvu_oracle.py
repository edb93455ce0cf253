"""fp64 restatement of the reference's fraction_variance_unexplained_top_activating (standard_metrics.py:316-342), with
its quirk: both partial reconstructions go through ``center``, not ``uncenter``, before they are compared with the raw
batch (for every kind but a centred TiedSAE ``center`` is the identity). The features are ranked by their mean code,
equal means by the lower feature index (the reference's argsort is not stable).

A dictionary is a dict of fp64 tensors in the layout of oracle/eval_oracle.py (kinds "tied", "untied", "topk") or of
oracle/baselines_oracle.py (kinds "random", "identity_relu"). Device-agnostic: runs on the CPU against
tests/golden/top_fvu.pt and on the GPU at scale."""
import torch

from . import baselines_oracle as BO
from . import eval_oracle as EO

_BASELINES = ("random", "identity_relu")


def code(m, x):
    """The reference's code of the centred batch."""
    if m["kind"] in _BASELINES:
        return BO.encode(m, x)
    return EO.encode(m, EO.center(m, x))


def decoder(m):
    """The rows the reference's decode multiplies the code with."""
    return m["decoder"] if m["kind"] in _BASELINES else EO.learned(m)


def center(m, x):
    return x if m["kind"] in _BASELINES else EO.center(m, x)


def top_features(c, n_top):
    """The n_top columns of ``c`` [N, n] with the largest mean, descending, equal means by the lower index."""
    return torch.sort(c.mean(dim=0), descending=True, stable=True).indices[:n_top]


def mean_gap(c, n_top):
    """Mean code at rank n_top - 1 minus the one at rank n_top: how far the choice of the top features is from a tie."""
    means = torch.sort(c.mean(dim=0), descending=True).values
    return float(means[n_top - 1] - means[n_top])


def fraction_variance_unexplained_top_activating(m, x, n_top=2):
    """(fvu_top, fvu_rest, top features) of dictionary ``m`` on the rows ``x`` [N, d] (fp64)."""
    c = code(m, x)
    top = top_features(c, n_top)
    keep = torch.zeros(c.shape[1], dtype=torch.bool, device=c.device)
    keep[top] = True
    w = decoder(m)
    x_top = center(m, torch.where(keep, c, torch.zeros((), dtype=c.dtype, device=c.device)) @ w)
    x_rest = center(m, torch.where(keep, torch.zeros((), dtype=c.dtype, device=c.device), c) @ w)
    var = (x - x.mean(dim=0)).pow(2).mean()
    return (x - x_top).pow(2).mean() / var, (x - x_rest).pow(2).mean() / var, top


# the golden helpers: the rows of a case of tests/golden/top_fvu.pt (oracle/make_top_fvu_golden.py)
N_EVAL = 2500


def rows(d, seed):
    """[N_EVAL, d] fp32 rows with a per-column scale and offset, a function of (d, seed) alone."""
    g = torch.Generator().manual_seed(seed)
    scale, offset = 0.5 + torch.rand(d, generator=g), 0.3 * torch.randn(d, generator=g)
    return torch.randn(N_EVAL, d, generator=g) * scale + offset
