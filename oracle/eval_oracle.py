"""fp64 restatement of the reference's dictionary scores on a set of activations (standard_metrics.py:305-314
mean_nonzero_activations / fraction_variance_unexplained, :344-345 r_squared, :446-454
batched_calc_feature_n_ever_active, :482-511 calc_moments_streaming), with the reference's quirks: FVU takes the
residual in the raw space (predict uncentres), mean_nonzero_activations encodes the centred batch, the two batched
functions encode the raw batch, times_active counts segments and the running averages weight the last partial segment
like a full one. Device-agnostic: runs on the CPU against tests/golden/dict_eval.pt and on the GPU at scale.

A dictionary is a dict of fp64 tensors: kind "tied" (encoder, encoder_bias, optional center_trans / center_rot /
center_scale), "untied" (encoder, encoder_bias, decoder) or "topk" (dict, sparsity)."""
import torch


def _unit(w, floor):
    nrm = w.norm(dim=-1)
    return w / (nrm.clamp(min=floor) if floor else nrm)[:, None]


def center(m, x):
    if m["kind"] != "tied" or "center_trans" not in m:
        return x
    return ((x - m["center_trans"][None]) @ m["center_rot"].T) * m["center_scale"][None]


def uncenter(m, x):
    if m["kind"] != "tied" or "center_trans" not in m:
        return x
    return (x / m["center_scale"][None]) @ m["center_rot"] + m["center_trans"][None]


def encode(m, x):
    if m["kind"] == "topk":
        s = x @ m["dict"].T
        top = torch.topk(s, int(m["sparsity"]), dim=-1)
        return torch.zeros_like(s).scatter_(-1, top.indices, top.values).clamp(min=0.0)
    w = _unit(m["encoder"], 1e-8) if m["kind"] == "tied" else m["encoder"]
    return (x @ w.T + m["encoder_bias"]).clamp(min=0.0)


def learned(m):
    if m["kind"] == "topk":
        return m["dict"]
    return _unit(m["encoder"] if m["kind"] == "tied" else m["decoder"], 1e-8)


def pre_activations(m, x):
    """z of every coefficient (top-k: the scores), for the kink window of a count comparison."""
    if m["kind"] == "topk":
        return x @ m["dict"].T
    w = _unit(m["encoder"], 1e-8) if m["kind"] == "tied" else m["encoder"]
    return x @ w.T + m["encoder_bias"]


def fraction_variance_unexplained(m, x):
    x_hat = uncenter(m, encode(m, center(m, x)) @ learned(m))
    return (x - x_hat).pow(2).mean() / (x - x.mean(dim=0)).pow(2).mean()


def r_squared(m, x):
    return 1.0 - fraction_variance_unexplained(m, x)


def mean_nonzero_activations(m, x):
    return (encode(m, center(m, x)) != 0).double().mean(dim=0)


def feature_counts(m, x, centred=False):
    return (encode(m, center(m, x) if centred else x) != 0).sum(dim=0)


def batched_calc_feature_n_ever_active(m, x, batch_size=1000, threshold=10):
    return int((feature_counts(m, x) > threshold).sum())


def moment_sums(m, x, batch_size=1000, centred=False):
    """(times_active, per-segment power sums [n_seg, n, 4], rows per segment)."""
    xs = center(m, x) if centred else x
    segs, rows, times = [], [], 0
    for i in range(0, x.shape[0], batch_size):
        c = encode(m, xs[i:i + batch_size])
        segs.append(torch.stack([c.sum(0), c.pow(2).sum(0), c.pow(3).sum(0), c.pow(4).sum(0)], dim=-1))
        rows.append(c.shape[0])
        times = times + (c.sum(0) != 0).double()
    return times, torch.stack(segs), rows


def calc_moments_streaming(m, x, batch_size=1000, centred=False):
    times, sums, rows = moment_sums(m, x, batch_size, centred)
    means = sums / torch.tensor(rows, dtype=sums.dtype, device=sums.device)[:, None, None]   # per-segment means
    mom = means.mean(dim=0)            # every segment weighted by batch_size, the last partial one included
    mean, m2, m3, m4 = mom.unbind(-1)
    var = m2 - mean ** 2
    skew = m3 / torch.clamp(var ** 1.5, min=1e-8)
    kurtosis = m4 / torch.clamp(var ** 2, min=1e-8)
    return times, mean, var, skew, kurtosis, m4


FUNCS = {
    "fraction_variance_unexplained": fraction_variance_unexplained,
    "r_squared": r_squared,
    "mean_nonzero_activations": mean_nonzero_activations,
    "batched_calc_feature_n_ever_active": batched_calc_feature_n_ever_active,
    "calc_moments_streaming": calc_moments_streaming,
}
