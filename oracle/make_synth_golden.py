"""Generate tests/golden/synthetic.pt by running the REFERENCE's own sc_datasets/random_dataset.py on the CPU.

TEST INFRASTRUCTURE. Run in the build container only (needs the reference tree):   python oracle/make_synth_golden.py

Recorded (fixtures only; the reference's random streams are torch's, which the GPU generator does not reproduce, so
what is compared is the numpy-drawn ground truth, bitwise, and sampling statistics):
  feats, corr        generate_rand_feats(64, 128) then generate_corr_matrix(128) after np.random.seed(0)
  "sparse_mix"       SparseMixDataset(64, 128, 4096, 5, 0.99, noise 0.1) built after np.random.seed(0) (its features and
                     covariance are the two matrices above), 64 sends of its own generate_correlated_dataset /
                     generate_noise_dataset
  "random"           RandomDatasetGenerator(64, 128, 4096, 5, 0.99, correlated=False) built after np.random.seed(0),
                     64 sends of its generate_rand_dataset
Per send (sends are independent, so the test takes the standard error of each statistic from their spread):
  freq [S, n_gt]     fraction of rows in which each component is non-zero
  nnz_hist [S, K]    fraction of rows with 0 .. K-2 non-zero components, and >= K-1
  fill [S]           fraction of rows the zero-row rule filled (a code of exactly 1.0)
  coef_mean, coef_var [S]   of the non-zero coefficients code * strength
  norm_mean, norm_var [S]   of ||x|| (x = the send, noise included)
  noise_var [S]      variance of the entries of the noise draw (sparse_mix only)
The strengths are not returned by the reference's functions; they are recorded by wrapping torch.rand for the call
(its third draw is the strength tensor)."""
import os
import sys
import types

import numpy as np
import torch

REF = os.environ.get("SCE_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "synthetic.pt")
D, N_GT, BATCH, NNZ, DECAY, NOISE, SENDS, K = 64, 128, 4096, 5, 0.99, 0.1, 64, 16


def import_reference():
    tt = types.ModuleType("torchtyping")

    class _TT:
        def __class_getitem__(cls, item):
            return cls

    tt.TensorType = _TT
    sys.modules.setdefault("torchtyping", tt)
    sys.path.insert(0, REF)
    import sc_datasets.random_dataset as rd  # noqa
    return rd


def recorded(fn, *args):
    """fn(*args) with every torch.rand result of the call recorded."""
    draws = []
    real = torch.rand

    def rand(*a, **k):
        t = real(*a, **k)
        draws.append(t)
        return t

    torch.rand = rand
    try:
        out = fn(*args)
    finally:
        torch.rand = real
    return out, draws


def send_stats(codes, strengths, x, noise=None):
    nz = codes != 0
    coef = (codes * strengths)[nz].double()
    nnz = nz.sum(1)
    hist = torch.stack([(nnz == k).double().mean() for k in range(K - 1)] + [(nnz >= K - 1).double().mean()])
    norm = x.double().norm(dim=1)
    s = {"freq": nz.double().mean(0), "nnz_hist": hist, "fill": (codes == 1.0).any(1).double().mean(),
         "coef_mean": coef.mean(), "coef_var": coef.var(), "norm_mean": norm.mean(), "norm_var": norm.var()}
    if noise is not None:
        s["noise_var"] = noise.double().var()
    return s


def stack(per_send):
    return {k: torch.stack([s[k] for s in per_send]) for k in per_send[0]}


def main():
    rd = import_reference()
    torch.manual_seed(0)
    np.random.seed(0)
    feats = rd.generate_rand_feats(D, N_GT, "cpu")
    corr = rd.generate_corr_matrix(N_GT, "cpu")

    np.random.seed(0)
    gen = rd.SparseMixDataset(D, N_GT, BATCH, NNZ, DECAY, NOISE, "cpu")
    assert torch.equal(gen.sparse_component_dict, feats) and torch.equal(gen.sparse_component_covariance, corr)
    per = []
    for _ in range(SENDS):     # SparseMixDataset.send, step by step (random_dataset.py:119-139)
        (_, codes, sparse), draws = recorded(rd.generate_correlated_dataset, N_GT, BATCH, gen.sparse_component_covariance,
                                             gen.sparse_component_dict, gen.frac_nonzero, gen.sparse_component_probs, "cpu")
        noise = rd.generate_noise_dataset(BATCH, gen.noise_covariance, gen.noise_magnitude_scale, "cpu")
        per.append(send_stats(codes, draws[2], (sparse + noise).to(gen.t_type), noise))
    sparse_mix = stack(per)

    np.random.seed(0)
    rgen = rd.RandomDatasetGenerator(D, N_GT, BATCH, NNZ, DECAY, False, "cpu")
    assert torch.equal(rgen.feats, feats)
    per = []
    for _ in range(SENDS):
        (_, codes, x), draws = recorded(rd.generate_rand_dataset, N_GT, BATCH, rgen.component_probs, rgen.feats, "cpu")
        per.append(send_stats(codes, draws[2], x))
    random = stack(per)

    torch.save({"feats": feats, "corr": corr, "sparse_mix": sparse_mix, "random": random,
                "config": {"d": D, "n_gt": N_GT, "batch": BATCH, "nnz": NNZ, "decay": DECAY, "noise": NOISE,
                           "sends": SENDS, "hist_bins": K, "np_seed": 0}}, OUT)
    print(f"wrote {os.path.normpath(OUT)}: sparse_mix fill {float(sparse_mix['fill'].mean()):.4f}, "
          f"coef mean {float(sparse_mix['coef_mean'].mean()):.4f}, random nnz mean "
          f"{float((random['freq'].sum(1)).mean()):.3f}")


if __name__ == "__main__":
    main()
