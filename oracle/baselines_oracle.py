"""fp64 oracle of the baseline dictionaries the engine scores with forward-only plans (ICAEncoder, RandomDict,
IdentityReLU): the reference's encode written out (autoencoders/ica.py:30-34 through sklearn's StandardScaler.transform and
FastICA.transform; learned_dict.py:86-127), and its metrics (standard_metrics.py:305-314, :446-454, :482-511) on that code.

A dictionary is a dict of fp64 tensors: ``kind`` ("ica", "random", "identity_relu"), ``encoder`` [n, d], ``encoder_bias``
[n], ``decoder`` [n, d] (the rows the reconstruction uses, as given) and ``trans`` [d] (subtracted before the encode).
The golden helpers at the end rebuild the cases of tests/golden/baselines.pt (oracle/make_baselines_golden.py)."""
import io
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "baselines.pt")


def ica(scaler_mean, scaler_scale, components, ica_mean):
    """((x - mean) / scale - ica_mean) C^T = (x - trans) (C / scale)^T, decoded by C's unit rows (get_learned_dict)."""
    f = lambda t: torch.as_tensor(t).double()
    comp, scale = f(components), f(scaler_scale)
    return {"kind": "ica", "encoder": comp / scale[None, :], "encoder_bias": torch.zeros(comp.shape[0], dtype=torch.float64),
            "decoder": comp / comp.norm(dim=-1, keepdim=True), "trans": f(scaler_mean) + scale * f(ica_mean)}


def random_dict(encoder, encoder_bias):
    e = encoder.double()
    return {"kind": "random", "encoder": e, "encoder_bias": encoder_bias.double(), "decoder": e,
            "trans": torch.zeros(e.shape[1], dtype=torch.float64)}


def identity_relu(bias):
    eye = torch.eye(bias.shape[0], dtype=torch.float64)
    return {"kind": "identity_relu", "encoder": eye, "encoder_bias": bias.double(), "decoder": eye,
            "trans": torch.zeros(bias.shape[0], dtype=torch.float64)}


def to(m, device):
    return {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in m.items()}


def pre_activations(m, x):
    return (x.double() - m["trans"]) @ m["encoder"].T + m["encoder_bias"]


def encode(m, x):
    z = pre_activations(m, x)
    return z if m["kind"] == "ica" else z.clamp(min=0.0)


def fraction_variance_unexplained(m, x):
    """NaN for ICA, whose reference decode raises; else the reference's formula."""
    x = x.double()
    if m["kind"] == "ica":
        return torch.tensor(float("nan"), dtype=torch.float64)
    r = (x - encode(m, x) @ m["decoder"]).pow(2).mean()
    return r / (x - x.mean(dim=0)).pow(2).mean()


def mean_nonzero_activations(m, x):
    return (encode(m, x) != 0).double().mean(dim=0)


def batched_calc_feature_n_ever_active(m, x, batch_size=1000, threshold=10):
    return int(((encode(m, x) != 0).sum(dim=0) > threshold).sum())


def calc_moments_streaming(m, x, batch_size=1000):
    """(times_active, mean, var, skew, kurtosis, m4) as the reference's running averages compute them, in fp64."""
    n_feats = m["encoder"].shape[0]
    z = lambda: torch.zeros(n_feats, dtype=torch.float64, device=x.device)
    times, mean, m2, m3, m4 = z(), z(), z(), z(), z()
    n = 0
    for i in range(0, x.shape[0], batch_size):
        c = encode(m, x[i:i + batch_size])
        bm = c.mean(dim=0)
        times += (bm != 0).double()
        upd = lambda old, new: (n * old + batch_size * new) / (n + batch_size)
        mean, m2, m3, m4 = upd(mean, bm), upd(m2, (c ** 2).mean(0)), upd(m3, (c ** 3).mean(0)), upd(m4, (c ** 4).mean(0))
        n += batch_size
    var = m2 - mean ** 2
    return times, mean, var, m3 / var.pow(1.5).clamp(min=1e-8), m4 / var.pow(2).clamp(min=1e-8), m4


# ---- the cases of tests/golden/baselines.pt
def load_golden():
    return torch.load(GOLDEN, weights_only=False)


def gaussian_rows(d, seed, n_rows=2500):
    """make_baselines_golden.py's evaluation rows: fp32 Gaussian rows with a per-column scale and offset."""
    g = torch.Generator().manual_seed(seed)
    scale, offset = 0.5 + torch.rand(d, generator=g), 0.3 * torch.randn(d, generator=g)
    return torch.randn(n_rows, d, generator=g) * scale + offset


def ica_from_golden(e):
    """The project's ICAEncoder holding the reference's fitted arrays of golden ICA case ``e``."""
    from sparse_coding_b200.ica import FittedFastICA, FittedScaler, ICAEncoder
    ica = ICAEncoder(e["d"])
    a = lambda t: t.numpy().astype(np.float64)
    ica.scaler = FittedScaler(a(e["scaler_mean"]), a(e["scaler_var"]), a(e["scaler_scale"]), e["rows"])
    ica.ica = FittedFastICA(a(e["components"]), a(e["mixing"]), a(e["ica_mean"]), None, None, 0)
    return ica


def ica_rows(e, n_rows=2500):
    from oracle.ica_oracle import mixed_sources
    x, _ = mixed_sources(e["d"], e["rows"], e["seed"])
    return x[:n_rows].float()


def golden_cases(golden):
    """(name, LearnedDict, oracle dictionary, evaluation rows, the reference's metrics) of every golden case; the
    RandomDict and IdentityReLU objects are unpickled from the reference's files."""
    n = golden["n_eval"]
    out = []
    for e in golden["ica"]:
        out.append((f"ica{e['d']}", ica_from_golden(e), ica(e["scaler_mean"], e["scaler_scale"], e["components"],
                                                            e["ica_mean"]), ica_rows(e, n), e["metrics"]))
    for e in golden["random"]:
        rd = torch.load(io.BytesIO(e["pickle"]), weights_only=False)
        out.append((f"random{e['n']}", rd, random_dict(rd.encoder, rd.encoder_bias), gaussian_rows(e["d"], e["x_seed"], n),
                    e["metrics"]))
    for e in golden["identity_relu"]:
        ir = torch.load(io.BytesIO(e["pickle"]), weights_only=False)
        out.append(("identity_relu", ir, identity_relu(ir.bias), gaussian_rows(e["d"], e["x_seed"], n), e["metrics"]))
    return out
