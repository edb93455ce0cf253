"""fp64 restatement of the reference's dictionary-similarity metrics (standard_metrics.py:270-303, 356-362).

TEST INFRASTRUCTURE: the yardstick for ``sparse_coding_b200.metrics`` (golden fixture, CPU) and for the at-scale GPU
tests (the same formulas on the device, in float64). Inputs are stored dictionaries described by a kind:
    "tied"   encoder rows / max(||row||, 1e-8)          (TiedSAE.get_learned_dict)
    "untied" decoder rows / max(||row||, 1e-8)          (UntiedSAE.get_learned_dict)
    "topk"   the stored, already normalised dict         (TopKLearnedDict.get_learned_dict)
    "raw"    the matrix as given                         (a ground-truth feature matrix)
"""
import torch

NORM_FLOOR = 1e-8


def learned(kind, w, dtype=torch.float64):
    w = w.to(dtype)
    if kind in ("tied", "untied"):
        return w / w.norm(dim=-1).clamp(min=NORM_FLOOR)[:, None]
    if kind == "topk_params":   # TopKEncoder params["dict"]: unit rows without a clamp
        return w / w.norm(dim=-1)[:, None]
    return w


def best_match(a, b):
    """For each row of ``a``, its largest inner product with a row of ``b``."""
    return (a @ b.T).max(dim=1).values


def mcs_duplicates(ground, model):
    return best_match(model, ground)


def mmcs(model, model2):
    return mcs_duplicates(model, model2).mean()


def mcs_to_fixed(model, truth):
    return best_match(model, truth)


def mmcs_to_fixed(model, truth):
    return mcs_to_fixed(model, truth).mean()


def mmcs_from_list(ls):
    n = len(ls)
    out = torch.eye(n, dtype=ls[0].dtype, device=ls[0].device)
    for i in range(n):
        for j in range(i):
            out[i, j] = out[j, i] = mmcs(ls[i], ls[j])
    return out


def representedness(features, model):
    return best_match(features, model)


def capacity_per_feature(model):
    s = (model @ model.T).pow(2)
    return torch.diag(s) / s.sum(dim=-1)


FUNCS = {f.__name__: f for f in (mcs_duplicates, mmcs, mcs_to_fixed, mmcs_to_fixed, mmcs_from_list, representedness,
                                 capacity_per_feature)}


def pair_maxima(a, b, block=8192):
    """(row maxima [na], column maxima [nb]) of a @ b.T in float64, ``block`` rows of ``a`` at a time (config 5's width
    would otherwise need an 8 GiB matrix)."""
    a, b = a.double(), b.double()
    rows, col = [], None
    for i in range(0, a.shape[0], block):
        s = a[i:i + block] @ b.T
        rows.append(s.max(dim=1).values)
        c = s.max(dim=0).values
        col = c if col is None else torch.maximum(col, c)
    return torch.cat(rows), col


def capacity_blocked(l, block=8192):
    """capacity_per_feature in float64, ``block`` rows at a time."""
    l = l.double()
    out = []
    for i in range(0, l.shape[0], block):
        s = (l[i:i + block] @ l.T).pow(2)
        out.append(s[torch.arange(s.shape[0]), torch.arange(i, i + s.shape[0])] / s.sum(dim=1))
    return torch.cat(out)
